"""Pins the oracle's OpenCV-primitive restatements (oracle/orb_prims.h) bit-exact against cv2 4.13.

The reference holds no tests or golden vectors for this path (SURVEY.md §4, §8c), and OpenCV is an
un-vendored dependency, so cv2 in this image is the only executable pin: parity target = reference
logic + OpenCV 4.13 primitive semantics.
"""
import ctypes as C

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from orb_slam2_b200 import synth
from tests.frame_input_cases import adversarial_remap_maps

u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)
f32p = C.POINTER(C.c_float)


@pytest.fixture(scope="module")
def lib(oracle):
    return C.CDLL(oracle.PORT_SO)


def _imgs(w, h):
    yield synth.mono_frame(3, 0, 0, w, h)
    yield synth.white_noise(5, w, h)
    g = np.tile(np.linspace(0, 255, w).astype(np.uint8), (h, 1))
    yield g


def level_sizes(w, h, n=8):
    s, inv = np.float32(1.0), []
    for _ in range(n):
        inv.append(np.float32(1.0) / s)
        s = np.float32(np.float64(s) * np.float64(np.float32(1.2)))
    return [(int(np.rint(np.float32(w) * i)), int(np.rint(np.float32(h) * i))) for i in inv]


@pytest.mark.parametrize("shape", [synth.KITTI, synth.TUM, synth.EUROC, (1241, 376), (333, 257)])
def test_resize_chain_matches_cv2(lib, shape):
    w, h = shape
    for img in _imgs(w, h):
        cur = img
        for (dw, dh) in level_sizes(w, h)[1:]:
            want = cv2.resize(cur, (dw, dh), interpolation=cv2.INTER_LINEAR)
            got = np.zeros((dh, dw), np.uint8)
            lib.orbport_resize_linear(cur.ctypes.data_as(u8p), cur.shape[1], cur.shape[0], cur.strides[0],
                                      got.ctypes.data_as(u8p), dw, dh, got.strides[0])
            assert np.array_equal(want, got), (shape, dw, dh, int((want != got).sum()))
            cur = want


@pytest.mark.parametrize("shape", [synth.KITTI, (640, 480), (347, 105), (179, 134), (64, 40), (9, 7)])
def test_gaussian_blur_matches_cv2(lib, shape):
    w, h = shape
    for img in _imgs(w, h):
        want = cv2.GaussianBlur(img, (7, 7), 2, None, 2, cv2.BORDER_REFLECT_101)
        got = np.zeros_like(img)
        lib.orbport_gaussian_blur7(img.ctypes.data_as(u8p), w, h, img.strides[0], got.ctypes.data_as(u8p), got.strides[0])
        assert np.array_equal(want, got), (shape, int((want != got).sum()))
        # in place (ORBextractor.cc:1086 blurs workingMat into itself)
        work = img.copy()
        lib.orbport_gaussian_blur7(work.ctypes.data_as(u8p), w, h, work.strides[0], work.ctypes.data_as(u8p), work.strides[0])
        assert np.array_equal(want, work)


def _cv_fast(img, th):
    det = cv2.FastFeatureDetector_create(threshold=th, nonmaxSuppression=True, type=cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
    return [(int(k.pt[0]), int(k.pt[1]), int(k.response)) for k in det.detect(img, None)]


@pytest.mark.parametrize("th", [20, 7, 12, 1])
def test_fast_matches_cv2(lib, th):
    for (w, h) in [(37, 38), (36, 35), (200, 120), (7, 7), (8, 30)]:
        for seed in range(3):
            base = synth.white_noise(seed, w, h) if seed else synth.mono_frame(9, 0, 0, max(w, 64), max(h, 64))[:h, :w].copy()
            want = _cv_fast(base, th)
            out = np.zeros((w * h + 1, 3), np.int32)
            n = lib.orbport_fast9(base.ctypes.data_as(u8p), w, h, base.strides[0], th, 1, out.ctypes.data_as(i32p), len(out))
            got = [tuple(r) for r in out[:n].tolist()]
            assert got == want, (w, h, seed, th, len(got), len(want))


def test_fast_atan2_matches_cv2(lib):
    rng = np.random.default_rng(0)
    n = 200000
    y = rng.integers(-2_900_000, 2_900_000, n).astype(np.float32)
    x = rng.integers(-2_900_000, 2_900_000, n).astype(np.float32)
    y[:10] = 0; x[5:15] = 0
    y[20:30] = x[20:30]
    # scalar cv::fastAtan2 is what ORBextractor.cc:103 calls (cv::phase's SIMD path contracts to FMA
    # and differs in the last ulp, so it is NOT the pin)
    want = np.array([cv2.fastAtan2(float(a), float(b)) for a, b in zip(y, x)], np.float32)
    got = np.zeros(n, np.float32)
    lib.orbport_fast_atan2(y.ctypes.data_as(f32p), x.ctypes.data_as(f32p), got.ctypes.data_as(f32p), n)
    assert np.array_equal(got, want)
    assert got.min() >= 0 and got.max() < 360


def test_reflect101(lib):
    for n in (1, 2, 5, 31):
        ref = cv2.copyMakeBorder(np.arange(n, dtype=np.uint8)[None, :], 0, 0, min(19, 3 * n), min(19, 3 * n), cv2.BORDER_REFLECT_101)[0]
        pad = min(19, 3 * n)
        got = [lib.orbport_reflect101(p, n) for p in range(-pad, n + pad)]
        assert got == ref.tolist()


@pytest.mark.parametrize("channels,rgb", [(3, True), (3, False), (4, True), (4, False)])
def test_cvtcolor_to_gray_matches_cv2(lib, channels, rgb):
    """Tracking::GrabImage* (src/Tracking.cc:172-197) convert colour frames with cv::cvtColor before extraction."""
    rng = np.random.default_rng(2)
    img = rng.integers(0, 256, (97, 131, channels), dtype=np.uint8)
    code = {(3, True): cv2.COLOR_RGB2GRAY, (3, False): cv2.COLOR_BGR2GRAY, (4, True): cv2.COLOR_RGBA2GRAY, (4, False): cv2.COLOR_BGRA2GRAY}[(channels, rgb)]
    want = cv2.cvtColor(img, code)
    got = np.zeros((97, 131), np.uint8)
    lib.orbport_cvt_color_to_gray(img.ctypes.data_as(u8p), 131, 97, img.strides[0], channels, int(rgb), got.ctypes.data_as(u8p), got.strides[0])
    assert np.array_equal(got, want)
    if channels == 3 and rgb:                                   # every colour once (2^24 pixels)
        r = np.arange(256, dtype=np.uint8)
        full = np.ascontiguousarray(np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(4096, 4096, 3))
        want = cv2.cvtColor(full, cv2.COLOR_RGB2GRAY)
        got = np.zeros((4096, 4096), np.uint8)
        lib.orbport_cvt_color_to_gray(full.ctypes.data_as(u8p), 4096, 4096, full.strides[0], 3, 1, got.ctypes.data_as(u8p), got.strides[0])
        assert np.array_equal(got, want)


def _euroc_maps(w, h, flip=1.0):
    K = np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1]])
    D = np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05]) * flip
    R = cv2.Rodrigues(np.array([0.003, -0.002, 0.001]) * flip)[0]
    P = np.array([[435.2, 0, 367.45], [0, 435.2, 252.2], [0, 0, 1]])
    return cv2.initUndistortRectifyMap(K, D, R, P, (w, h), cv2.CV_32F)


def test_remap_linear_matches_cv2(lib):
    """cv::remap(..., INTER_LINEAR) with CV_32FC1 maps (Examples/Stereo/stereo_euroc.cc:96-98,136-137)."""
    rng = np.random.default_rng(4)
    cases = []
    w, h = synth.EUROC
    cases.append((synth.mono_frame(6, 0, 0, w, h),) + tuple(_euroc_maps(w, h)))
    img = rng.integers(0, 256, (120, 160), dtype=np.uint8)
    yy, xx = np.mgrid[0:120, 0:160].astype(np.float32)
    mx = (xx + 6 * np.sin(yy / 17) + rng.normal(0, 0.3, (120, 160)) - 3).astype(np.float32)      # leaves the image on every side
    my = (yy + 5 * np.cos(xx / 23) + rng.normal(0, 0.3, (120, 160)) - 2).astype(np.float32)
    cases.append((img, mx, my))
    cases.append((img, (xx[:90, :100] * 1.5 + 0.25).astype(np.float32).copy(), (yy[:90, :100] * 1.25 - 0.5).astype(np.float32).copy()))   # dst != src size
    for im, m1, m2 in cases:
        want = cv2.remap(im, m1, m2, cv2.INTER_LINEAR)
        got = np.zeros(m1.shape, np.uint8)
        m1c, m2c = np.ascontiguousarray(m1), np.ascontiguousarray(m2)
        lib.orbport_remap_linear(im.ctypes.data_as(u8p), im.shape[1], im.shape[0], im.strides[0], m1c.ctypes.data_as(f32p),
                                 m2c.ctypes.data_as(f32p), got.ctypes.data_as(u8p), m1.shape[1], m1.shape[0], got.strides[0])
        assert np.array_equal(got, want), int((got != want).sum())


def _port_remap(lib, im, m1, m2):
    got = np.zeros(m1.shape, np.uint8)
    m1c, m2c = np.ascontiguousarray(m1, np.float32), np.ascontiguousarray(m2, np.float32)
    lib.orbport_remap_linear(im.ctypes.data_as(u8p), im.shape[1], im.shape[0], im.strides[0], m1c.ctypes.data_as(f32p),
                             m2c.ctypes.data_as(f32p), got.ctypes.data_as(u8p), m1.shape[1], m1.shape[0], got.strides[0])
    return got


@pytest.mark.parametrize("src,dst", [((64, 48), (61, 45)), ((64, 48), (130, 97)), ((37, 29), (23, 17)), ((160, 120), (159, 121))])
def test_remap_linear_adversarial_maps_match_cv2(lib, src, dst):
    """Map values where the 1/32-px rounding goes wrong: NaN, +-inf, finite values whose *32 leaves int range (cvRound saturates to
    INT_MIN: the pixel reads the border), k/32 +- 1/64 ties (round half to even), taps at ix = -1 and ix = src_w - 1, destinations
    larger and smaller than the source with dst_w % 4 in {1, 2, 3}."""
    for mx, my in adversarial_remap_maps(src, dst, seed=sum(src) + sum(dst)):
        im = np.random.default_rng(dst[0]).integers(1, 256, (src[1], src[0]), dtype=np.uint8)     # no zero pixel: border reads show
        want = cv2.remap(im, mx, my, cv2.INTER_LINEAR)
        got = _port_remap(lib, im, mx, my)
        bad = np.argwhere(got != want)
        assert len(bad) == 0, (len(bad), [(float(mx[tuple(b)]), float(my[tuple(b)])) for b in bad[:5]])


def test_remap_linear_out_of_range_values_read_the_border(lib):
    """The cases that separate a saturating cvRound from a wrapping one, pixel by pixel."""
    im = np.full((40, 50), 200, np.uint8)
    for v in (134217744.0, 2.0 ** 31, 2.0 ** 26, -(2.0 ** 26) - 64, np.inf, -np.inf, np.nan, 3.0e38):
        mx = np.full((3, 5), 10.0, np.float32); my = np.full((3, 5), 10.0, np.float32)
        mx[1, 2] = v
        my[2, 3] = v
        want = cv2.remap(im, mx, my, cv2.INTER_LINEAR)
        assert want[1, 2] == 0 and want[2, 3] == 0 and want[0, 0] == 200, v
        assert np.array_equal(_port_remap(lib, im, mx, my), want), v


def test_small_float_gemm_order_matches_cv2():
    """The cv::Mat products of the matcher / frame code (Rcw*p3Dw+tcw, -Rcw.t()*tcw, ...) are OpenCV gemm calls on 3x3 / 3x1
    CV_32F matrices.  oracle/cvmini (used by the verbatim builds of ORBmatcher.cc / Frame.cc), the restatements and the CUDA
    kernels all evaluate them as ((a0*b0 + a1*b1) + a2*b2) + c in float32, no FMA; cv2 agrees on every sample."""
    rng = np.random.default_rng(0)
    f32 = np.float32
    for _ in range(5000):
        R = rng.normal(0, 1, (3, 3)).astype(f32); p = rng.normal(0, 5, (3, 1)).astype(f32); t = rng.normal(0, 2, (3, 1)).astype(f32)
        mine = np.array([[f32(f32(f32(R[i, 0] * p[0, 0]) + f32(R[i, 1] * p[1, 0])) + f32(R[i, 2] * p[2, 0])) + t[i, 0]] for i in range(3)], f32)
        assert np.array_equal(cv2.gemm(R, p, 1.0, t, 1.0), mine)
        assert np.array_equal(cv2.gemm(R, p, 1.0, None, 0.0) + t, mine)
        M = rng.normal(0, 1, (3, 3)).astype(f32)
        mm = np.array([[f32(f32(f32(R[i, 0] * M[0, j]) + f32(R[i, 1] * M[1, j])) + f32(R[i, 2] * M[2, j])) for j in range(3)] for i in range(3)], f32)
        assert np.array_equal(cv2.gemm(R, M, 1.0, None, 0.0), mm)
