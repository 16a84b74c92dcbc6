"""GPU: the device maths functions themselves (borb_debug_eval_math runs the very __device__ functions the kernels inline,
compiled with them) against their references on every input they can receive, compared bit for bit.

  sinf / cosf   k_describe.cu glibc_sincosf, the rBRIEF rotation: every float in [0, 2*pi] and 100 past it, vs the host glibc
  logf          k_match.cu glibc_logf, inside PredictScale: every positive normal float, vs the host glibc
  PredictScale  k_match.cu predict_scale: every non-negative float ratio and a few NaNs, vs the port (whose logf is the same
                host glibc) and, on a stride, vs the verbatim MapPoint.cc
  fastAtan2     k_describe.cu fast_atan2_deg, the keypoint angle: every c in [0, 1] for both branches, the other sign quadrants
                on a stride, and the integer moments IC_Angle can form, vs orbport_fast_atan2 (pinned to cv2)

The descriptor and matcher fixtures barely notice a last-ulp error in these functions (DESIGN.md section 2), so these sweeps
are what ties the device ports to the functions the reference calls.  glibc >= 2.28 is required of the host: older releases
use other sinf/cosf/logf algorithms."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_b200 import _lib

pytestmark = pytest.mark.gpu

SIN, COS, ATAN2, LOGF, PREDICT = range(5)     # borb_debug_eval_math's fn
CHUNK = 1 << 26
TWO_PI_LAST = 0x40C90FDB + 100                # (float)(2*pi), then 100 floats more
POS_INF, ONE = 0x7F800000, 0x3F800000
NANS = np.array([0x7FC00000, 0x7F800001, 0x7FA00000, 0x7FFFFFFF, 0xFFC00000], np.uint32)
MOMENT_MAX = 624240                           # |m01|, |m10| <= 255 * (sum of the positive u over the 749-pixel disc)


@pytest.fixture(scope="module")
def glibc():
    try:
        libc = C.CDLL("libc.so.6")
        libc.gnu_get_libc_version.restype = C.c_char_p
        version = libc.gnu_get_libc_version().decode()
    except (OSError, AttributeError):
        pytest.skip("the host C library is not glibc")
    if tuple(int(p) for p in version.split(".")[:2]) < (2, 28):
        pytest.skip(f"glibc {version} < 2.28 uses other sinf/cosf/logf algorithms than the device ports")
    return version


def libm_logf(x):
    libm = C.CDLL("libm.so.6")
    libm.logf.restype, libm.logf.argtypes = C.c_float, [C.c_float]
    return np.float32(libm.logf(float(np.float32(x))))


def device(fn, a, b=None, log_scale=0.0, n_levels=0):
    out = np.empty(len(a), np.int32 if fn == PREDICT else np.float32)
    _lib.check(_lib.load().borb_debug_eval_math(fn, _lib.ptr(a), _lib.ptr(b), len(a), float(log_scale), n_levels,
                                                out.ctypes.data), "borb_debug_eval_math")
    return out


def floats(lo, hi):
    """The floats with bit patterns lo .. hi - 1."""
    return np.arange(lo, hi, dtype=np.uint32).view(np.float32)


def strided_ratios(stride):
    """Every stride-th non-negative float pattern, +inf and the NaNs."""
    return np.concatenate([np.arange(0, POS_INF, stride, dtype=np.uint32), np.array([POS_INF], np.uint32), NANS]).view(np.float32)


def _show(v):
    if isinstance(v, (np.floating, float)):
        v = np.float32(v)
        return f"{int(v.view(np.uint32)):#010x} ({float(v)!r})"
    return str(int(v))


class Sweep:
    """Bitwise comparison of device and reference outputs over many chunks; fails with the mismatch count and the first few
    inputs in hex, the device value next to the reference value."""

    def __init__(self, what):
        self.what, self.n, self.bad, self.first = what, 0, 0, []

    def add(self, got, want, *inputs):
        assert got.shape == want.shape and got.dtype == want.dtype
        g, w = (got.view(np.uint32), want.view(np.uint32)) if got.dtype == np.float32 else (got, want)
        diff = np.flatnonzero(g != w)
        self.n += len(g)
        self.bad += len(diff)
        for i in diff[: max(0, 8 - len(self.first))]:
            self.first.append(f"({', '.join(_show(x[i]) for x in inputs)}): device {_show(got[i])}, reference {_show(want[i])}")

    def check(self):
        assert self.bad == 0, f"{self.what}: {self.bad} of {self.n} values differ; first: " + "; ".join(self.first)
        print(f"{self.what}: {self.n} values, 0 mismatches")


@pytest.mark.parametrize("fn", [SIN, COS], ids=["sinf", "cosf"])
def test_sincosf_every_float_to_two_pi(glibc, oracle, fn):
    # describe_kernel's t = angle * (float)(pi/180) with angle < 360 (test_fast_atan2_reachable_moments) stays in the range
    assert np.float32(360) * np.float32(np.pi / 180) <= np.uint32(TWO_PI_LAST).view(np.float32)
    ref = oracle.LIBM_SINF if fn == SIN else oracle.LIBM_COSF
    sweep = Sweep(["sinf", "cosf"][fn])
    for lo in range(0, TWO_PI_LAST + 1, CHUNK):
        x = floats(lo, min(lo + CHUNK, TWO_PI_LAST + 1))
        sweep.add(device(fn, x), oracle.port_libm(ref, x), x)
    assert sweep.n == TWO_PI_LAST + 1
    sweep.check()


def test_logf_every_positive_normal_float(glibc, oracle):
    sweep = Sweep("logf")
    for lo in range(0x00800000, POS_INF, CHUNK):
        x = floats(lo, min(lo + CHUNK, POS_INF))
        sweep.add(device(LOGF, x), oracle.port_libm(oracle.LIBM_LOGF, x), x)
    assert sweep.n == 2_130_706_432
    sweep.check()


def test_predict_scale_every_ratio(glibc, oracle):
    """ORB-SLAM2's pyramid (scale 1.2, 8 levels); max_distance = x, dist = 1 makes the ratio exactly x: +0, the subnormals,
    every normal float, +inf and NaNs."""
    log_scale = libm_logf(1.2)
    sweep, levels = Sweep("PredictScale(1.2, 8)"), np.zeros(8, np.int64)
    ones = np.ones(CHUNK, np.float32)
    for lo in range(0, POS_INF + 1, CHUNK):
        x = floats(lo, min(lo + CHUNK, POS_INF + 1))
        got = device(PREDICT, x, ones[: len(x)], log_scale, 8)
        sweep.add(got, oracle.port_predict_scale(x, ones[: len(x)], log_scale, 8), x)
        levels += np.bincount(got, minlength=8)[:8]
    x = NANS.view(np.float32)
    sweep.add(device(PREDICT, x, ones[: len(x)], log_scale, 8), oracle.port_predict_scale(x, ones[: len(x)], log_scale, 8), x)
    assert sweep.n == POS_INF + 1 + len(NANS)
    sweep.check()
    assert (levels > 0).all(), levels


@pytest.mark.parametrize("n_levels", [1, 8, 12])
@pytest.mark.parametrize("scale", [1.1, 1.5, 2.0])
def test_predict_scale_pyramids_on_a_stride(glibc, oracle, scale, n_levels):
    log_scale = libm_logf(scale)
    x = strided_ratios(97)
    ones = np.ones(len(x), np.float32)
    sweep = Sweep(f"PredictScale({scale}, {n_levels})")
    got = device(PREDICT, x, ones, log_scale, n_levels)
    sweep.add(got, oracle.port_predict_scale(x, ones, log_scale, n_levels), x)
    sweep.check()
    assert set(np.unique(got).tolist()) == set(range(n_levels))


def test_predict_scale_matches_the_mappoint_source(glibc, oracle_ref):
    """Every 64th ratio of the sweep against MapPoint::PredictScale compiled from the reference source, both overloads."""
    if not oracle_ref.have_mapref():
        pytest.skip("oracle/_ref/libmapref.so not built (reference tree absent)")
    log_scale = libm_logf(1.2)
    x = strided_ratios(64)
    ones = np.ones(len(x), np.float32)
    got = device(PREDICT, x, ones, log_scale, 8)
    for use_frame in (False, True):
        sweep = Sweep(f"PredictScale vs MapPoint.cc ({'Frame' if use_frame else 'KeyFrame'} overload)")
        sweep.add(got, oracle_ref.ref_predict_scale(x, ones, log_scale, 8, use_frame=use_frame).astype(np.int32), x)
        sweep.check()


def _atan2_sweep(oracle, sweep, y, x):
    got = device(ATAN2, y, x)
    sweep.add(got, oracle.port_fast_atan2(y, x), y, x)
    return got


def test_fast_atan2_whole_polynomial_domain(oracle):
    """fast_atan2_deg sees (x, y) only through c = ay / (ax + eps) or its mirror; with the other coordinate 1 the division
    returns c exactly, so (y, x) = (c, 1) and (1, c) run each branch's polynomial on every c in [0, 1]."""
    below, above = Sweep("fastAtan2(c, 1)"), Sweep("fastAtan2(1, c)")
    ones = np.ones(CHUNK, np.float32)
    for lo in range(0, ONE + 1, CHUNK):
        c = floats(lo, min(lo + CHUNK, ONE + 1))
        _atan2_sweep(oracle, below, c, ones[: len(c)])
        _atan2_sweep(oracle, above, ones[: len(c)], c)
    assert below.n == above.n == 1_065_353_217
    below.check()
    above.check()


def test_fast_atan2_other_quadrants_on_a_stride(oracle):
    c = np.arange(0, ONE + 1, 61, dtype=np.uint32).view(np.float32)
    ones = np.ones(len(c), np.float32)
    for sy, sx in ((1, -1), (-1, 1), (-1, -1)):
        sweep = Sweep(f"fastAtan2 quadrant ({sy:+d}, {sx:+d})")
        _atan2_sweep(oracle, sweep, np.float32(sy) * c, np.float32(sx) * ones)
        _atan2_sweep(oracle, sweep, np.float32(sy) * ones, np.float32(sx) * c)
        sweep.check()


def test_fast_atan2_reachable_moments(oracle):
    """IC_Angle's moments are integers with |m01|, |m10| <= MOMENT_MAX.  Every pair within +-1024, 10^8 seeded pairs over the
    whole range, every pair with |m01| == |m10| or a zero moment, and the extremes: bit-exact, and every angle below 360, so the
    bin clamp of describe_kernel only guards."""
    umax = oracle.PortExtractor(1000).umax.astype(np.int64)
    half = umax[np.abs(np.arange(-15, 16))]
    assert (2 * half + 1).sum() == 749 and 255 * (half * (half + 1) // 2).sum() == MOMENT_MAX

    sweep, hi = Sweep("fastAtan2(m01, m10)"), np.float32(0)

    def run(m01, m10):
        nonlocal hi
        y, x = m01.astype(np.float32), m10.astype(np.float32)
        got = _atan2_sweep(oracle, sweep, y, x)
        assert got.min() >= 0
        hi = max(hi, got.max())

    small = np.arange(-1024, 1025)
    run(*[g.ravel() for g in np.meshgrid(small, small)])
    rng = np.random.default_rng(20261017)
    for n in (1 << 25, 1 << 25, 100_000_000 - (1 << 26)):
        run(rng.integers(-MOMENT_MAX, MOMENT_MAX + 1, n), rng.integers(-MOMENT_MAX, MOMENT_MAX + 1, n))
    m = np.arange(-MOMENT_MAX, MOMENT_MAX + 1)
    zero = np.zeros_like(m)
    run(np.concatenate([m, m, zero, m]), np.concatenate([m, -m, m, zero]))
    edge = np.array([-MOMENT_MAX, -MOMENT_MAX + 1, -1, 0, 1, MOMENT_MAX - 1, MOMENT_MAX])
    run(*[g.ravel() for g in np.meshgrid(edge, edge)])
    sweep.check()
    print(f"largest angle {float(hi)!r}")
    assert hi < 360


def test_eval_math_refusals(oracle):
    so = _lib.load()
    x = np.array([0.5, 1.0, 2.0], np.float32)
    out = np.zeros(3, np.float32)
    p, o = _lib.ptr(x), out.ctypes.data
    for fn, a, b, n, dst in ((-1, p, p, 3, o), (5, p, p, 3, o), (LOGF, p, None, -1, o), (LOGF, None, None, 3, o),
                             (LOGF, p, None, 3, None), (ATAN2, p, None, 3, o), (PREDICT, p, None, 3, o)):
        assert so.borb_debug_eval_math(fn, a, b, n, 0.0, 8, dst) == 1, (fn, n)      # BORB_ERR_INVALID_ARG
        assert so.borb_last_error()
    assert so.borb_debug_eval_math(LOGF, p, None, 0, 0.0, 0, o) == 0
    assert not out.any()
    # still usable: logf(1) = 0, cosf(0) = 1, fastAtan2(1, 1) as cv::fastAtan2 (44.99...), PredictScale(2 / 1) at scale 2 = level 1
    assert device(LOGF, x)[1] == 0 and device(COS, np.zeros(1, np.float32))[0] == 1
    assert device(ATAN2, x[1:2], x[1:2])[0] == oracle.port_fast_atan2(x[1:2], x[1:2])[0]
    assert device(PREDICT, x[2:], x[1:2], libm_logf(2.0), 8)[0] == 1
