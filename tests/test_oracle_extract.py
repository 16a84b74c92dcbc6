"""Oracle self-consistency: the independent restatement (oracle/orb_port_extract.cpp) against the
reference's own ORBextractor.cc compiled verbatim (oracle/_ref), and against cv2 4.13 run the way
ORBextractor.cc:789-829 runs it (one cv::FAST call per cell)."""
import math

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import extract_config as XC

SHAPES = [(synth.KITTI, 2000), (synth.TUM, 1000), (synth.EUROC, 1200)]


@pytest.mark.parametrize("shape,nf", SHAPES)
@pytest.mark.parametrize("seed", [1, 2])
def test_port_equals_verbatim_reference(oracle_ref, shape, nf, seed):
    w, h = shape
    img = synth.mono_frame(seed, 0, 0, w, h)
    R, P = oracle_ref.RefExtractor(nf), oracle_ref.PortExtractor(nf)
    for name in ("scale", "inv_scale", "sigma2", "inv_sigma2", "per_level", "umax"):
        assert np.array_equal(getattr(R, name), getattr(P, name)), name
    kr, dr = R(img)
    kp, dp = P(img)
    assert len(kr) == len(kp) >= nf
    assert np.array_equal(kr, kp)          # all 7 KeyPoint fields, same order
    assert np.array_equal(dr, dp)
    for l in range(8):
        assert np.array_equal(R.level(l), P.level(l))


@pytest.mark.parametrize("nf", [500, 2000, 4000])
def test_port_equals_reference_white_noise(oracle_ref, nf):
    img = synth.white_noise(11, 640, 360)
    R, P = oracle_ref.RefExtractor(nf), oracle_ref.PortExtractor(nf)
    kr, dr = R(img)
    kp, dp = P(img)
    assert np.array_equal(kr, kp) and np.array_equal(dr, dp)


def test_reference_call_is_repeatable(oracle_ref):
    """The monotonic allocator makes the address-ordered quadtree tie-break deterministic."""
    img = synth.mono_frame(4, 0, 0, *synth.KITTI)
    R = oracle_ref.RefExtractor(2000)
    k1, d1 = R(img)
    other = synth.white_noise(1, 400, 300)
    R(other)
    k2, d2 = R(img)
    assert np.array_equal(k1, k2) and np.array_equal(d1, d2)


def test_edge_cases(oracle_ref):
    R, P = oracle_ref.RefExtractor(1000), oracle_ref.PortExtractor(1000)
    blank = np.full((240, 320), 128, np.uint8)
    for E in (R, P):
        k, d = E(blank)
        assert len(k) == 0 and d.shape == (0, 32)
    one = blank.copy()
    one[100:140, 150:200] = 220            # a single bright rectangle: 4 corners per level
    kr, dr = R(one)
    kp, dp = P(one)
    assert len(kr) > 0 and np.array_equal(kr, kp) and np.array_equal(dr, dp)
    weak = blank.copy()
    weak[60:120, 70:150] = 140             # contrast 12: only reachable through the minThFAST=7 fallback
    kr, dr = R(weak)
    kp, dp = P(weak)
    assert len(kr) > 0 and kr["response"].max() < 20
    assert np.array_equal(kr, kp) and np.array_equal(dr, dp)
    plateau = blank.copy()
    plateau[::2, ::2] = 200                # dense equal-score ties: strict NMS keeps none of a tie pair
    kr, dr = R(plateau)
    kp, dp = P(plateau)
    assert np.array_equal(kr, kp) and np.array_equal(dr, dp)


def _cells_cv2(level_img, ini_th=20, min_th=7):
    """ORBextractor.cc:765-829 with the real cv2.FAST, one call per cell."""
    cv2 = pytest.importorskip("cv2")
    H, W = level_img.shape
    minB, maxBX, maxBY = 16, W - 16, H - 16
    width, height = float(maxBX - minB), float(maxBY - minB)
    nCols, nRows = int(width / 30), int(height / 30)
    wCell, hCell = math.ceil(width / nCols), math.ceil(height / nRows)
    det = {t: cv2.FastFeatureDetector_create(threshold=t, nonmaxSuppression=True) for t in (ini_th, min_th)}
    out = []
    for i in range(nRows):
        iniY = minB + i * hCell
        maxY = iniY + hCell + 6
        if iniY >= maxBY - 3:
            continue
        maxY = min(maxY, maxBY)
        for j in range(nCols):
            iniX = minB + j * wCell
            maxX = iniX + wCell + 6
            if iniX >= maxBX - 6:
                continue
            maxX = min(maxX, maxBX)
            sub = np.ascontiguousarray(level_img[iniY:maxY, iniX:maxX])
            k = det[ini_th].detect(sub, None)
            if len(k) == 0:
                k = det[min_th].detect(sub, None)
            for kp in k:
                out.append((int(kp.pt[0]) + iniX, int(kp.pt[1]) + iniY, int(kp.response)))
    return out


@pytest.mark.parametrize("shape", [synth.KITTI, synth.TUM, (179, 134), (719, 217)])
def test_whole_level_candidates_equal_per_cell_cv2(oracle, shape):
    """At the default thresholds and at every pair of tests/extract_config.py (0, 127/128, 255, ini == min, ini < min); at
    the TUM shape also on that module's exact-score dot images."""
    w, h = shape
    imgs = (synth.mono_frame(6, 0, 0, w, h), synth.white_noise(2, w, h),
            (synth.mono_frame(7, 0, 0, w, h) // 8 + 100).astype(np.uint8))   # low contrast: fallback cells
    for ini, mn in [(20, 7)] + XC.THRESHOLD_PAIRS:
        dots = [XC.threshold_dots(ini, mn, b)[0] for b in (True, False)] if shape == XC.THRESHOLD_SIZE else []
        for img in list(imgs) + dots:
            P = oracle.PortExtractor(1000, 1.2, 8, ini, mn)
            P(img)
            got = [tuple(r) for r in P.candidates(0).tolist()]
            want = _cells_cv2(img, ini, mn)
            assert got == want, (ini, mn)


@pytest.mark.parametrize("N", [5, 60, 434, 869])
def test_quadtree_port_equals_reference(oracle_ref, N):
    rng = np.random.default_rng(N)
    R = oracle_ref.RefExtractor(2000)
    for width, height in [(1210, 343), (608, 448), (147, 102), (315, 73)]:
        for n in (1, 2, 7, 300, 5000):
            n = min(n, (width - 6) * (height - 6) // 4)
            flat = rng.choice((width - 6) * (height - 6), size=n, replace=False)
            xs, ys = 3 + flat % (width - 6), 3 + flat // (width - 6)
            sc = rng.integers(7, 60, n)           # few distinct responses: exercises first-wins ties
            order = np.lexsort((xs, ys))
            xys = np.stack([xs[order], ys[order], sc[order]], 1).astype(np.int32)
            want = R.distribute(xys.astype(np.float32), width, height, N).astype(np.int32)
            got = oracle_ref.port_distribute(xys, width, height, N)
            assert np.array_equal(want, got), (width, height, n, N)
