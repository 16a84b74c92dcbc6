"""Inputs shared by the frame-input sweeps (tests/test_oracle_prims.py, tests/test_oracle_frame_ref.py on the CPU and
tests/test_gpu_frame_input.py on the device): rectification maps that stress cv::remap's 1/32-px rounding, camera models that
stress Frame::UndistortKeyPoints / ComputeImageBounds, and depth values that stress ComputeStereoFromRGBD.  numpy only."""
import numpy as np

F32 = np.float32

# values whose *32 leaves int range, or is no number at all: cvRound gives INT_MIN, the pixel reads the border
SPECIAL_MAP_VALUES = np.array([np.nan, np.inf, -np.inf, 2.0 ** 26, -(2.0 ** 26), 2.0 ** 26 - 8, -(2.0 ** 26) + 8, 2.0 ** 26 + 16,
                               -(2.0 ** 26) - 16, 134217744.0, 2.0 ** 31, -(2.0 ** 31), 3.0e38, -3.0e38, 32767.5, -32768.5, 1.0e6],
                              np.float32)


def adversarial_remap_maps(src, dst, seed=0):
    """(map_x, map_y) pairs of shape (dst_h, dst_w) for a src_w x src_h source."""
    sw, sh = src
    dw, dh = dst
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:dh, 0:dw].astype(np.float64)
    sx, sy = (sw - 1) / max(dw - 1, 1), (sh - 1) / max(dh - 1, 1)
    out = []
    # 1. a smooth warp that leaves the source on every side, with a special value in every 7th entry of each map
    mx = (xx * sx * 1.1 - 2.5 + 3 * np.sin(yy / 5)).astype(F32)
    my = (yy * sy * 1.1 - 2.5 + 3 * np.cos(xx / 7)).astype(F32)
    flat_x, flat_y = mx.reshape(-1), my.reshape(-1)
    sp = SPECIAL_MAP_VALUES
    flat_x[::7] = sp[np.arange(len(flat_x[::7])) % len(sp)]
    flat_y[3::7] = sp[(np.arange(len(flat_y[3::7])) * 5) % len(sp)]
    out.append((mx, my))
    # 2. exact ties of the 1/32 grid: (k + 1/2)/32 for k around the whole source, both signs (round half to even)
    kx = rng.integers(-3 * 32, (sw + 2) * 32, (dh, dw))
    ky = rng.integers(-3 * 32, (sh + 2) * 32, (dh, dw))
    sgn = rng.choice([-1.0, 1.0], (dh, dw))
    out.append(((kx + 0.5 * sgn) / 32.0, (ky + 0.5 * sgn[::-1]) / 32.0))
    # 3. the taps at the source's edges: ix = -1 and ix = sw - 1 (one of the two bilinear taps outside), same for y
    fx = rng.integers(0, 32, (dh, dw)) / 32.0
    fy = rng.integers(0, 32, (dh, dw)) / 32.0
    ex = np.where(rng.random((dh, dw)) < 0.5, -1.0, sw - 1.0) + fx
    ey = np.where(rng.random((dh, dw)) < 0.5, -1.0, sh - 1.0) + fy
    iny = rng.uniform(0, sh - 1, (dh, dw))
    inx = rng.uniform(0, sw - 1, (dh, dw))
    out.append((np.where(xx % 2 == 0, ex, inx), np.where(xx % 2 == 0, iny, ey)))
    # 4. values one rounding step either side of the special band, and uniformly random floats over a wide range
    near = np.array([2.0 ** 26 - 8, 2.0 ** 26, -(2.0 ** 26), -(2.0 ** 26) - 8, -0.0, 0.0, -1 / 64, 1 / 64, -1.0, sw - 1 / 64.0,
                     sw + 0.0, -(1 / 32), 1e-30, -1e-30], np.float64)
    wx = np.where(rng.random((dh, dw)) < 0.3, near[rng.integers(0, len(near), (dh, dw))], rng.uniform(-2 * sw, 2 * sw, (dh, dw)))
    wy = np.where(rng.random((dh, dw)) < 0.3, near[rng.integers(0, len(near), (dh, dw))], rng.uniform(-2 * sh, 2 * sh, (dh, dw)))
    out.append((wx, wy))
    return [(np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)) for a, b in out]


def radial_rectify_maps(src, dst, k1=-0.28, k2=0.07, shift=(0.0, 0.0)):
    """A smooth rectification-like map (Brown radial model, no cv2) from a dst_w x dst_h image into a src_w x src_h frame."""
    sw, sh = src
    dw, dh = dst
    yy, xx = np.mgrid[0:dh, 0:dw].astype(np.float64)
    f = 0.6 * max(sw, sh)
    x = (xx - dw / 2 + shift[0]) / f
    y = (yy - dh / 2 + shift[1]) / f
    r2 = x * x + y * y
    d = 1 + k1 * r2 + k2 * r2 * r2
    return (x * d * f + sw / 2).astype(F32), (y * d * f + sh / 2).astype(F32)


# (K4, distortion) cases of the RGB-D / monocular Frame constructor: dist as Tracking builds mDistCoef (4 or 5 entries)
TUM1_K = (517.306408, 516.469215, 318.643040, 255.313989)
DIST_CASES = {
    "tum1_5": (TUM1_K, (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)),
    "tum1_4": (TUM1_K, (0.262383, -0.953104, -0.005358, 0.002628)),
    "k1_zero_rest_nonzero": (TUM1_K, (0.0, -0.953104, -0.005358, 0.002628, 1.163314)),   # k1 == 0: mvKeysUn = mvKeys
    "k1_neg_zero": (TUM1_K, (-0.0, 0.2, 0.001, -0.001, 0.1)),                            # -0.0 == 0.0: also a copy
    "barrel_4": ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)),
    "pincushion": ((300.0, 310.0, 330.0, 230.0), (0.9, 0.6, 0.002, -0.003, 0.4)),
    "icdist_negative": ((300.0, 300.0, 320.0, 240.0), (-0.9, 0.0, 0.0, 0.0)),            # 1/(1+k1 r^2) < 0 inside the image
    "none": (TUM1_K, (0.0, 0.0, 0.0, 0.0)),
}

DEPTH_FACTORS = (1.0 / 5000.0, 1.0 / 1000.0, 1.0)


def edge_depth_float(seed, w=640, h=480):
    """A float32 depth map (metres) seeded with 0, negative, NaN, +-inf and subnormal values among plausible depths."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.3, 8.0, (h, w)).astype(F32)
    special = np.array([0.0, -0.0, -1.0, np.nan, np.inf, -np.inf, 1e-45, 1e-40, -1e-45, 65535.0, 3.0e38], F32)
    m = rng.random((h, w)) < 0.3
    d[m] = special[rng.integers(0, len(special), int(m.sum()))]
    return d


def edge_depth_raw(seed, w=640, h=480):
    """A CV_16U depth map with holes (0), the largest raw value (65535) and the smallest nonzero ones."""
    rng = np.random.default_rng(seed)
    d = rng.integers(300, 40000, (h, w)).astype(np.uint16)
    special = np.array([0, 0, 1, 2, 65535, 65534], np.uint16)
    m = rng.random((h, w)) < 0.3
    d[m] = special[rng.integers(0, len(special), int(m.sum()))]
    return d


def keys_on_depth_specials(keys, depth):
    """How many keypoints look up a special depth (0 / negative / NaN / inf / subnormal): the sweep is only a sweep if many do."""
    d = depth[keys["y"].astype(np.int64), keys["x"].astype(np.int64)]
    return int((~np.isfinite(d) | (d <= 0) | ((d != 0) & (np.abs(d) < np.finfo(np.float32).tiny))).sum())
