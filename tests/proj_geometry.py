"""Matcher inputs placed on the float decision boundaries of the projection searches: Frame::isInFrustum, the SearchByProjection
overloads, both Fuse overloads and the epipolar gates of SearchForTriangulation.  Test tooling: tests/test_oracle_proj_geometry.py
pins the port to the verbatim Frame.cc / ORBmatcher.cc on every case and checks that both members of every boundary pair are
decided differently by the verbatim build; tests/test_gpu_proj_geometry.py pins the CUDA library to the port.

Every case is a small call (one boundary point or keypoint, a few ordinary ones) whose outcome is readable.  A pair is two
cases that differ in one free input by one float32 step, found by bisecting over that input's bit patterns with the gate
restated here in numpy float32 / float64, in the reference's operation order.  Each gate is restated next to the kernel line
it exists for.  Nothing in this module calls the CUDA library.

The LastFrame search runs with the forward / backward flags of its two poses (level_*: each mode's level window at
nLastOctave 0, 3 and 7; fwd_bwd_mb_*: tlc.z on mb), PredictScale is decided by the level window of every search that calls it
(predict_scale_*), and SearchBySim3 runs under a scaled, rotated similarity whose chained camera-frame point carries the
depth and distance gates (sim3_*).  With checkOrientation on, a contested histogram of ten matches decides the
rotation bin at rot = -0.0 / -2^-149 and at rot*(1/30) = 0.5 (rot_*); the key a search's square keeps at its outermost float lies
in the edge cell of the grid window, clamped or not (area_edge_*); and every world-point class is also run inside a natural
~1000-point call (dense_case).

No case separates the two flavours of 1/z the kernels use (1.0f/z and (float)(1.0/(double)z)): they are identical, because a
double quotient rounded to float is the correctly rounded float quotient (53 >= 2*24 + 2, double rounding is innocuous for
division)."""
import ctypes
import functools
import zlib

import numpy as np

from orb_slam2_b200.matcher import FeatureVector, FrameView, KeyFrameView, LastFrameView, MapPointsView, WorldPointsView
from orb_slam2_b200._lib import KP_DTYPE

f32, f64 = np.float32, np.float64
K_CAM = (500.0, 500.0, 320.0, 240.0)
BOUNDS = (0.0, 0.0, 640.0, 480.0)
T_CW = np.array([[1, 0, 0, 0.25], [0, 1, 0, -0.5], [0, 0, 1, 1.0]], np.float32)     # [I | t]: every product below is exact
OW = np.array([-0.25, 0.5, -1.0], np.float32)                                     # -Rcw^T tcw
BF = 40.0
N_LEVELS = 8


def _scale_factors():
    s = np.ones(N_LEVELS, np.float32)
    for i in range(1, N_LEVELS):                    # ORBextractor: mvScaleFactor[i] = mvScaleFactor[i-1] * scaleFactor, in float
        s[i] = f32(s[i - 1] * f32(1.2))
    return s


SCALE = _scale_factors()
SIGMA2 = (SCALE * SCALE).astype(np.float32)

# coverage classes -> the kernel line each exists for
CLASSES = {
    "frustum_max_x": "k_match.cu:119 u > maxX (inclusive bound) in Frame::isInFrustum",
    "frustum_min_x": "k_match.cu:119 u < minX (inclusive bound) in Frame::isInFrustum",
    "frustum_min_dist": "k_match.cu:152-153 dist < 0.8f*mfMinDistance, dist from cv::norm in double",
    "frustum_max_y": "k_match.cu:119 v > maxY (inclusive bound) in Frame::isInFrustum",
    "frustum_min_y": "k_match.cu:119 v < minY (inclusive bound) in Frame::isInFrustum",
    "frustum_max_dist": "k_match.cu:152-153 dist > 1.2f*mfMaxDistance",
    "frustum_view_cos": "k_match.cu:163-164 viewCos < viewingCosLimit",
    "camera_centre": "k_match.cu:113-119 PcZ == 0: NaN projection and NaN viewCos are in view, as the reference stores them",
    "pcz_sign": "k_match.cu:113 PcZ < 0: PcZ == -0 passes (NaN projection, in view), -(smallest subnormal) does not",
    "last_max_x": "k_match.cu:134 u > maxX in SearchByProjection(CurrentFrame, LastFrame)",
    "kf_max_x": "k_match.cu:134 u > maxX in SearchByProjection(CurrentFrame, KeyFrame)",
    "image_max_x": "k_match.cu:127 KeyFrame::IsInImage u < maxX (half-open) in both Fuse overloads",
    "image_min_x": "k_match.cu:127 KeyFrame::IsInImage u >= minX: the left bound is inside",
    "kf_behind_camera": "k_match.cu:131 the keyframe overload has no depth test: a point behind the camera is found",
    "fuse_normal_dot": "k_match.cu:156-157 PO.dot(Pn) < 0.5*dist in double, both Fuse overloads",
    "fuse_chi2_stereo": "k_proj.cu:200 e2*invSigma2 > 7.8 in double",
    "fuse_chi2_mono": "k_proj.cu:203 e2*invSigma2 > 5.99 in double",
    "fuse_kr_zero": "k_proj.cu:197 kpr >= 0 takes the stereo gate at kpr == +0",
    "proj_dx_eq_rs": "k_proj.cu:57 |dx| < rs (strict)",
    "proj_dy_eq_rs": "k_proj.cu:57 |dy| < rs (strict)",
    "proj_er_eq_rs": "k_proj.cu:61-62 |xr - ur| > rs rejects; equality is kept",
    "proj_ur_zero": "k_proj.cu:60 ur > 0: no stereo test at ur == 0",
    "proj_view_cos_0998": "k_proj.cu:92 mTrackViewCos > 0.998 in double: 0.998f takes radius 2.5",
    "proj_th_one": "k_proj.cu:93 th != 1 scales the radius; th == 1 does not",
    "tri_epipole": "k_match.cu:528-529 distance to the epipole < 100*scale (strict) rejects",
    "tri_dsqr": "k_match.cu:534 dsqr < 3.84*mvLevelSigma2 in double",
    "tri_den_zero": "k_match.cu:532 den == 0 rejects before the division",
    "level_fwd_0": "k_match.cu:141 forward from nLastOctave 0: minLevel 0, maxLevel -1, so area_passes (k_proj.cu:52) tests no level",
    "level_fwd_3": "k_match.cu:141 forward window [o, inf): octave o - 1 is outside",
    "level_fwd_7": "k_match.cu:141 forward window [7, inf): octave 6 is outside",
    "level_bwd_0": "k_match.cu:142 backward window [0, 0]: maxLevel 0 >= 0 still checks levels (k_proj.cu:52)",
    "level_bwd_3": "k_match.cu:142 backward window [0, o]: octave o + 1 is outside",
    "level_bwd_7": "k_match.cu:142 backward window [0, 7] keeps octave 0, which the mono window [6, 8] drops",
    "level_none_0": "k_match.cu:143 window [o - 1, o + 1] at o = 0: octave 2 is outside",
    "level_none_3_lo": "k_match.cu:143 window [o - 1, o + 1]: octave o - 2 is outside",
    "level_none_3_hi": "k_match.cu:143 window [o - 1, o + 1]: octave o + 2 is outside",
    "level_none_7": "k_match.cu:143 window [6, 8] at o = 7: octave 5 is outside",
    "fwd_bwd_mb_fwd": "ORBmatcher_borb.cc:128-135 bForward = tlc.z > mb (strict): tlc.z == mb searches the mono window",
    "fwd_bwd_mb_bwd": "ORBmatcher_borb.cc:128-135 bBackward = -tlc.z > mb (strict): -tlc.z == mb searches the mono window",
    "predict_scale_kf": "k_match.cu:63-74 PredictScale at ratio = sf^2, in the keyframe overload's window [L - 1, L + 1]",
    "predict_scale_local": "k_match.cu:63-74 isInFrustum's mnTrackScaleLevel at ratio = sf^2, in SearchByProjection's window",
    "predict_scale_sim3proj": "k_match.cu:63-74 PredictScale at ratio = sf^2 in SearchByProjection(pKF, Scw)",
    "predict_scale_fuse_kf": "k_match.cu:63-74 PredictScale at ratio = sf^2 in Fuse(pKF, vpMapPoints)",
    "predict_scale_fuse": "k_match.cu:63-74 PredictScale at ratio = sf^2 in Fuse(pKF, Scw)",
    "predict_scale_sim3": "k_match.cu:63-74 PredictScale at ratio = sf^2 in SearchBySim3",
    "predict_scale_ratio_inf": "k_match.cu:67-70 a ratio that overflows to +inf predicts level 0, the largest finite one level 7",
    "sim3_min_dist_12": "k_match.cu:147-153 dist3D = norm(p3Dc2) < 0.8f*mfMinDistance, KF1's points into KF2",
    "sim3_max_dist_12": "k_match.cu:147-153 dist3D = norm(p3Dc2) > 1.2f*mfMaxDistance, KF1's points into KF2",
    "sim3_min_dist_21": "k_match.cu:147-153 dist3D = norm(p3Dc1) < 0.8f*mfMinDistance, KF2's points into KF1",
    "sim3_max_dist_21": "k_match.cu:147-153 dist3D = norm(p3Dc1) > 1.2f*mfMaxDistance, KF2's points into KF1",
    "sim3_depth_12": "k_match.cu:107-111,122 p3Dc2.z < 0 on the chained point, while p3Dc1.z > 0",
    "sim3_depth_21": "k_match.cu:107-111,122 p3Dc1.z < 0 on the chained point, while p3Dc2.z > 0",
    "rot_zero_last": "match_rules.cuh:29-35 rot = -0.0 is bin 0; rot = -2^-149 becomes 360.0f, bin 12 (no wrap), culled; LastFrame overload",
    "rot_zero_kf": "match_rules.cuh:29-35 rot = -0.0 against -2^-149 in the KeyFrame overload's histogram",
    "rot_zero_tri": "match_rules.cuh:29-35 rot = -0.0 against -2^-149 in SearchForTriangulation's histogram",
    "rot_half_last": "match_rules.cuh:32 rot*(1/30) == 0.5 rounds half away to bin 1; one step below is bin 0, culled; LastFrame overload",
    "rot_half_kf": "match_rules.cuh:32 rot*(1/30) at 0.5 against one step below in the KeyFrame overload's histogram",
    "rot_half_tri": "match_rules.cuh:32 rot*(1/30) at 0.5 against one step below in SearchForTriangulation's histogram",
    "area_edge_left": "k_proj.cu:41 floor((x - minX - r)*invW): the key the square keeps lies in the window's first column",
    "area_edge_right": "k_proj.cu:42 ceil((x - minX + r)*invW): the key the square keeps lies in the window's last column",
    "area_edge_col0": "k_proj.cu:41 max(0, floor(-0.2)): the clamped first column holds the kept key",
    "area_edge_col63": "k_proj.cu:42 min(63, ceil(63.2)): the clamped last column holds the kept key",
    "area_edge_row0": "k_proj.cu:43 max(0, floor(-0.2)): the clamped first row holds the kept key",
    "area_edge_row47": "k_proj.cu:44 min(47, ceil(47.2)): the clamped last row holds the kept key",
    "area_edge_minx": "k_proj.cu:41 a frame with minX = 100 and a key at x == minX, in column 0",
}

# rows of the gate table these cases do not reach, each with the reason; test_every_class_is_reached keeps CLASSES and this
# table together, so a gate cannot silently fall out of both
NOT_COVERED = {
    "predict_scale_ratio_subnormal": "PredictScale's ratio <= 0 or subnormal (k_match.cu:66-67): no pair can exist.  The ratio "
                                     "mfMaxDistance/dist is below the smallest normal float only when dist > 2^126*mfMaxDistance, "
                                     "and every search drops such a point at dist > 1.2f*mfMaxDistance (k_match.cu:152-153) before "
                                     "it predicts a level.  dist == 0 (ratio +inf or NaN) is the camera-centre point, whose level 0 "
                                     "camera_centre pins and whose NaN projection has no search window",
    "dense_variants_other_kinds": "the dense variants (dense_cases) embed the world-point classes.  The rot_* classes are left "
                                  "out because no pair can exist there: a natural background fills the rotation histogram, so "
                                  "the three surviving bins are chosen by the background and not by the boundary match.  The "
                                  "proj_*, area_edge_*, tri_* and sim3_* cases take no world points to embed them in",
}


# ---------------------------------------------------------------------------------------------------------------------------
# float32 steps and bisection over bit patterns
def step(x, n=1):
    """x moved by n float32 steps (n < 0: towards -inf)."""
    x = f32(x)
    for _ in range(abs(n)):
        x = np.nextafter(x, f32(np.inf if n > 0 else -np.inf), dtype=np.float32)
    return f32(x)


def _key(x):
    i = int(np.array(x, np.float32).view(np.int32))
    return i if i >= 0 else -(i & 0x7FFFFFFF)


def _unkey(k):
    return np.array(k if k >= 0 else ((-k) | 0x80000000), np.uint32).view(np.float32)[()]


def first_separating(pair_of, candidates):
    """(*candidate, pair) for the first candidate whose pair_of(*candidate) is not None: the first base input whose boundary pair
    a float restatement of a double test would decide differently."""
    for cand in candidates:
        pair = pair_of(*cand)
        if pair is not None:
            return (*cand, pair)
    raise AssertionError("no candidate separates the double and float forms of the test")


def bisect(pred, lo, hi):
    """(a, b): adjacent float32 values between lo and hi on which pred (monotone on [lo, hi]) differs."""
    a, b = _key(lo), _key(hi)
    pa = pred(_unkey(a))
    assert pa != pred(_unkey(b)), (lo, hi)
    while b - a > 1:
        m = (a + b) // 2
        if pred(_unkey(m)) == pa:
            a = m
        else:
            b = m
    return f32(_unkey(a)), f32(_unkey(b))


# ---------------------------------------------------------------------------------------------------------------------------
# the reference's float arithmetic, restated
def cam_point(T, P):
    """cv::Mat 3x3 * 3x1 + 3x1 in float32: ((r0*p0 + r1*p1) + r2*p2) + t (k_match.cu:103-105)."""
    T, P = np.asarray(T, np.float32), np.asarray(P, np.float32)
    return np.array([f32(f32(f32(T[r, 0] * P[0]) + f32(T[r, 1] * P[1])) + f32(T[r, 2] * P[2])) + T[r, 3] for r in range(3)], np.float32)


def camera_centre(T):
    """mOw = -mRcw.t()*mtcw as cv::Mat evaluates it: the negated transpose times t, ((a0*t0 + a1*t1) + a2*t2) in float, which
    decides the sign of a zero component."""
    A = (-np.asarray(T, np.float32)[:, :3].T).astype(np.float32)
    t = np.asarray(T, np.float32)[:, 3]
    return np.array([f32(f32(f32(A[r, 0] * t[0]) + f32(A[r, 1] * t[1])) + f32(A[r, 2] * t[2])) for r in range(3)], np.float32)


def project_frustum(Pc, K=K_CAM):
    """u, v of Frame::isInFrustum: fx*PcX*invz + cx, invz = 1.0f/PcZ (k_match.cu:114-116)."""
    fx, fy, cx, cy = [f32(k) for k in K]
    invz = f32(f32(1.0) / Pc[2])
    return f32(f32(f32(fx * Pc[0]) * invz) + cx), f32(f32(f32(fy * Pc[1]) * invz) + cy)


def norm_po(P, Ow=OW):
    """(PO, dist): PO = P - Ow in float, dist = cv::norm(PO), squares accumulated in double (k_match.cu:148-150)."""
    PO = (np.asarray(P, np.float32) - np.asarray(Ow, np.float32)).astype(np.float32)
    d = PO.astype(np.float64)
    return PO, f32(np.sqrt(f64(f64(d[0] * d[0]) + f64(d[1] * d[1])) + f64(d[2] * d[2])))


def dot64(PO, N):
    d, n = np.asarray(PO, np.float64), np.asarray(N, np.float32).astype(np.float64)
    return f64(f64(d[0] * n[0]) + f64(d[1] * n[1])) + f64(d[2] * n[2])


def dot32(PO, N):
    """The same dot product in float: what a float restatement of the 0.5*dist test would compare."""
    PO, N = np.asarray(PO, np.float32), np.asarray(N, np.float32)
    return f32(f32(f32(PO[0] * N[0]) + f32(PO[1] * N[1])) + f32(PO[2] * N[2]))


# ---------------------------------------------------------------------------------------------------------------------------
# building blocks
def _desc(seed, n):
    return np.random.default_rng(seed).integers(0, 256, (n, 32), dtype=np.uint8)


def _keys(xy, octave=0, angle=0.0):
    k = np.zeros(len(xy), KP_DTYPE)
    k["x"] = [p[0] for p in xy]
    k["y"] = [p[1] for p in xy]
    k["octave"], k["size"], k["response"], k["angle"] = octave, 31.0, 1.0, angle
    return k


# the ordinary points that go with every world-point case: comfortably inside every gate, each with its own keypoint
_ORDINARY_CAM = [(-0.25, -0.125, 2.0), (0.125, 0.5, 4.0)]


def _world_case(cls, member, cam, key_xy, bounds=BOUNDS, mx=None, mn=None, normal=None, ur=-1.0, inv=None, T=T_CW, world0=None, key_oct=0,
                **kw):
    """One boundary point (index 0, camera coordinates `cam` under the pose T = [I | t], or world position world0) and the
    ordinary points; keypoint f sits at key_xy (octave key_oct) for point 0 and at its projection + (0.5, 0) for the others.
    Descriptors: point i equals keypoint i."""
    cams = [tuple(cam)] + _ORDINARY_CAM
    P = np.array([[c[0] - T[0, 3], c[1] - T[1, 3], c[2] - T[2, 3]] for c in cams], np.float32)
    if world0 is not None:
        P[0] = world0
    Ow = camera_centre(T)
    n = len(P)
    xy = [key_xy]
    for c in _ORDINARY_CAM:
        u, v = project_frustum(np.array(c, np.float32))
        xy.append((float(u) + 0.5, float(v)))
    keys = _keys(xy)
    keys["octave"][0] = key_oct
    desc = _desc(zlib.crc32(cls.encode()) % 1000 + 7, n)
    dists = np.array([norm_po(p, Ow)[1] for p in P], np.float32)
    mxs = dists.copy(); mns = (dists * f32(0.5)).astype(np.float32)
    if mx is not None:
        mxs[0] = mx
    if mn is not None:
        mns[0] = mn
    nrm = np.array([norm_po(p, Ow)[0] / d if d > 0 else (0, 0, 1) for p, d in zip(P, dists)], np.float32)
    if normal is not None:
        nrm[0] = normal
    urs = np.full(n, -1.0, np.float32); urs[0] = ur
    F = FrameView(mvKeysUn=keys, mDescriptors=desc, mvScaleFactors=SCALE, bounds=tuple(float(b) for b in bounds), mvuRight=urs,
                  mvInvLevelSigma2=(inv if inv is not None else (f32(1.0) / SIGMA2).astype(np.float32)))
    Pv = WorldPointsView(world_pos=P, descriptors=desc.copy(), max_distance=mxs, min_distance=mns, normal=nrm,
                         angle=np.zeros(n, np.float32), valid=np.ones(n, np.uint8))
    c = dict(cls=cls, member=member, F=F, P=Pv, Tcw=T, Ow=Ow, K=K_CAM, bf=BF, th=3.0, vcl=0.5, has_obs=np.ones(n, np.uint8))
    c.update(kw)
    return c


U0_CAM = (0.5, 0.25, 2.0)             # projects to u = 445, v = 302.5 exactly in every overload (powers of two throughout)
U0, V0 = 445.0, 302.5


def _pairs_frustum():
    out = []
    # inclusive bounds (:176): maxX == u keeps the point, one step below drops it; minX == u keeps it, one step above drops it.
    # The bounds are narrow so that a grid cell is under a pixel and the keypoint half a pixel from u lands in the grid.
    for m, mx in enumerate((U0, step(U0, -1))):
        out.append(_world_case("frustum_max_x", m, U0_CAM, (U0 - 0.5, V0), bounds=(400.0, 0.0, mx, 480.0)))
    for m, mn in enumerate((U0, step(U0, 1))):
        out.append(_world_case("frustum_min_x", m, U0_CAM, (U0 + 0.5, V0), bounds=(mn, 0.0, 490.0, 480.0)))
    for m, my in enumerate((V0, step(V0, -1))):
        out.append(_world_case("frustum_max_y", m, U0_CAM, (U0 + 0.5, V0 - 0.5), bounds=(0.0, 270.0, 640.0, my)))
    for m, my in enumerate((V0, step(V0, 1))):
        out.append(_world_case("frustum_min_y", m, U0_CAM, (U0 + 0.5, V0 + 0.5), bounds=(0.0, my, 640.0, 335.0)))
    # dist against 0.8f*mfMinDistance / 1.2f*mfMaxDistance (:210-211): bisect the distance over its float steps, and keep a
    # point whose kept member sits exactly on the bound (so that < versus <= is decided by the pair)
    P0 = np.array(U0_CAM, np.float32) - T_CW[:, 3]
    _, dist = norm_po(P0)
    a, b = bisect(lambda mn: not (dist < f32(f32(0.8) * mn)), dist, f32(dist * 2))
    assert f32(f32(0.8) * a) == dist
    for m, mn in enumerate((a, b)):
        out.append(_world_case("frustum_min_dist", m, U0_CAM, (U0 + 0.5, V0), mn=mn))
    a, b = bisect(lambda mx: not (dist > f32(f32(1.2) * mx)), f32(dist / 2), dist)
    assert f32(f32(1.2) * b) == dist
    for m, mx in enumerate((b, a)):
        out.append(_world_case("frustum_max_dist", m, U0_CAM, (U0 + 0.5, V0), mx=mx))
    # viewCos = PO.dot(Pn)/dist in double, rounded to float (:218-222), against the limit
    PO, _ = norm_po(P0)
    N = np.array([0.25, 0.75, 0.5], np.float32)
    vc = f32(dot64(PO, N) / f64(dist))
    for m, lim in enumerate((vc, step(vc, 1))):
        out.append(_world_case("frustum_view_cos", m, U0_CAM, (U0 + 0.5, V0), normal=N, vcl=float(lim)))
    # a point at the camera centre with mfMinDistance == 0: PcZ == +0, u = v = NaN, dist = 0, viewCos = 0/0 — the reference
    # keeps it (NaN passes every comparison) at level 0; the smallest positive mfMinDistance drops it
    for m, mn in enumerate((f32(0.0), step(0.0, 1))):
        out.append(_world_case("camera_centre", m, (0.0, 0.0, 0.0), (U0 + 0.5, V0), mn=mn, mx=f32(1.0)))
    # PcZ < 0 (:172) at the sign of zero: with t = (0.25, 0.5, -0) and P = (-0.25, -0.5, -0) every term of PcZ is -0, so PcZ ==
    # -0 passes (not < 0) and the point is the camera-centre NaN point again; P.z = -(smallest subnormal) gives PcZ < 0
    Tn = np.array([[1, 0, 0, 0.25], [0, 1, 0, 0.5], [0, 0, 1, -0.0]], np.float32)
    for m, z in enumerate((f32(-0.0), -step(0.0, 1))):
        out.append(_world_case("pcz_sign", m, (0.0, 0.0, 0.0), (U0 + 0.5, V0), mn=f32(0.0), mx=f32(1.0), T=Tn,
                               world0=(-0.25, -0.5, z)))
    return out


def _pairs_other_world():
    out = []
    # SearchByProjection(CurrentFrame, LastFrame) and (CurrentFrame, KeyFrame): the same inclusive bound on :192
    for m, mx in enumerate((U0, step(U0, -1))):
        out.append(dict(_world_case("last_max_x", m, U0_CAM, (U0 - 0.5, V0), bounds=(400.0, 0.0, mx, 480.0)), th=7.5))
        out.append(dict(_world_case("kf_max_x", m, U0_CAM, (U0 - 0.5, V0), bounds=(400.0, 0.0, mx, 480.0)), th=7.5))
    # KeyFrame::IsInImage (:185): one step above u is inside, u == maxX is outside
    for m, mx in enumerate((step(U0, 1), U0)):
        out.append(_world_case("image_max_x", m, U0_CAM, (U0 - 0.5, V0), bounds=(400.0, 0.0, mx, 480.0)))
    for m, mn in enumerate((U0, step(U0, 1))):                   # u == minX is inside
        out.append(_world_case("image_min_x", m, U0_CAM, (U0 + 0.5, V0), bounds=(mn, 0.0, 490.0, 480.0)))
    # the keyframe overload has no depth test: a point behind the camera projecting onto the same pixel (u = 445) is found,
    # and the inclusive bound decides it as for a point in front
    for m, mx in enumerate((U0, step(U0, -1))):
        out.append(dict(_world_case("kf_behind_camera", m, tuple(-x for x in U0_CAM), (U0 - 0.5, V0), bounds=(400.0, 0.0, mx, 480.0),
                                    mn=f32(1.0)), th=7.5))
    # the viewing-angle test of both Fuse overloads (:214-215): bisect the normal's last component; keep the first base normal
    # for which the same test in float decides one member of the pair differently (the pair then tells the two apart)
    P0 = np.array(U0_CAM, np.float32) - T_CW[:, 3]
    PO, dist = norm_po(P0)
    half = f64(0.5) * f64(dist)

    def normal_pair(n0, n1):
        a, b = bisect(lambda z: not (dot64(PO, (n0, n1, z)) < half), f32(-4.0), f32(4.0))
        in_float = [not (dot32(PO, (n0, n1, z)) < f32(f32(0.5) * dist)) for z in (a, b)]
        return (a, b) if in_float != [False, True] else None
    n0, n1, (a, b) = first_separating(normal_pair, [(n0, n1) for n0 in np.linspace(0.1, 0.9, 33, dtype=np.float32)
                                                    for n1 in (f32(0.3), f32(-0.7), f32(0.55))])
    for m, z in enumerate((b, a)):
        out.append(_world_case("fuse_normal_dot", m, U0_CAM, (U0 - 0.5, V0), normal=(n0, n1, z)))
    # Fuse(pKF, vpMapPoints) reprojection gates (:907-931): e2 = 1 (keypoint one pixel left of u, on v, kpr on ur), so
    # e2*invSigma2 == invSigma2[0]: the free input is mvInvLevelSigma2[0] itself
    ur0 = f32(f32(U0) - f32(f32(BF) * f32(0.5)))
    for m, inv0 in enumerate((step(7.8, -1), f32(7.8))):        # 7.8f > 7.8 in double: rejected
        inv = (f32(1.0) / SIGMA2).astype(np.float32); inv[0] = inv0
        out.append(_world_case("fuse_chi2_stereo", m, U0_CAM, (U0 - 1.0, V0), ur=ur0, inv=inv))
    for m, inv0 in enumerate((f32(5.99), step(5.99, 1))):       # 5.99f < 5.99 in double: kept
        inv = (f32(1.0) / SIGMA2).astype(np.float32); inv[0] = inv0
        out.append(_world_case("fuse_chi2_mono", m, U0_CAM, (U0 - 1.0, V0), ur=-1.0, inv=inv))
    # kpr == +0 takes the stereo gate (er = 425 px: rejected); the largest negative value takes the monocular one (kept)
    for m, kr in enumerate((step(0.0, -1), f32(0.0))):
        out.append(_world_case("fuse_kr_zero", m, U0_CAM, (U0 - 1.0, V0), ur=kr))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchByProjection(CurrentFrame, LastFrame, th, bMono = false): the forward / backward decision and the level windows
MB = f32(f32(BF) / f32(K_CAM[0]))                 # Frame::mb = mbf/fx
T_FB = np.array([[1, 0, 0, 0.25], [0, 1, 0, -0.5], [0, 0, 1, 0.0]], np.float32)     # tcw.z = 0: twc.z is +0 exactly


def last_pose(tz):
    """The last frame's pose [I | (0.25, -0.5, tz)]: with the current pose T_FB, tlc.z == tz exactly."""
    return np.array([[1, 0, 0, 0.25], [0, 1, 0, -0.5], [0, 0, 1, tz]], np.float32)


def forward_backward(Tcur, Tlast, mb=MB):
    """(bForward, bBackward) of ORBmatcher.cc:1338-1349: twc = -Rcw^T*tcw, tlc = Rlw*twc + tlw, tlc.z > mb / -tlc.z > mb, both
    strict.  The kernels take the two flags from the host (integration/ORBmatcher_borb.cc:128-135, borb.h:315)."""
    tlc = cam_point(Tlast, camera_centre(Tcur))
    return bool(tlc[2] > mb), bool(-tlc[2] > mb)


MODE_TZ = {"fwd": f32(0.5), "bwd": f32(-0.5), "none": f32(0.0)}

# GetFeaturesInArea's level window per mode (ORBmatcher.cc:1385-1390, k_match.cu:141-143, bCheckLevels in area_passes):
# forward [o, inf), backward [0, o], neither [o - 1, o + 1], o = nLastOctave.  class: ((mode, o, key octave) of the kept
# member, (mode, o, key octave) of the rejected one); the key octaves sit just inside and just outside the window
LEVEL_PAIRS = {
    "level_fwd_0": (("fwd", 0, 7), ("none", 0, 7)),      # forward from 0: bCheckLevels is false, no level test at all
    "level_fwd_3": (("fwd", 3, 3), ("fwd", 3, 2)),
    "level_fwd_7": (("fwd", 7, 7), ("fwd", 7, 6)),
    "level_bwd_0": (("bwd", 0, 0), ("bwd", 0, 1)),       # backward from 0: maxLevel 0 >= 0 checks levels, octave 0 only
    "level_bwd_3": (("bwd", 3, 3), ("bwd", 3, 4)),
    "level_bwd_7": (("bwd", 7, 0), ("none", 7, 0)),      # backward from 7 keeps every octave of the pyramid
    "level_none_0": (("none", 0, 1), ("none", 0, 2)),
    "level_none_3_lo": (("none", 3, 2), ("none", 3, 1)),
    "level_none_3_hi": (("none", 3, 4), ("none", 3, 5)),
    "level_none_7": (("none", 7, 6), ("none", 7, 5)),
}


def _last_case(cls, member, tz, last_oct, key_oct):
    """The boundary point seen by a last-frame keypoint at octave last_oct and by the current keypoint (octave key_oct) half a
    pixel from its projection; the last frame's pose puts tlc.z at tz."""
    Tl = last_pose(tz)
    fwd, bwd = forward_backward(T_FB, Tl)
    return _world_case(cls, member, U0_CAM, (U0 + 0.5, V0), T=T_FB, key_oct=key_oct, Tlast=Tl, fwd=fwd, bwd=bwd, last_oct=last_oct)


def _pairs_last_levels():
    out = []
    for cls, members in LEVEL_PAIRS.items():
        for m, (mode, o, ko) in enumerate(members):
            out.append(_last_case(cls, m, MODE_TZ[mode], o, ko))
    # tlc.z == mb is neither forward nor backward (strict >); one step beyond it is.  With nLastOctave 3 the key at octave 5 lies
    # in the forward window [3, inf) only and the key at octave 1 in the backward window [0, 3] only (neither: [2, 4])
    for cls, tzs, ko in (("fwd_bwd_mb_fwd", (step(MB, 1), MB), 5), ("fwd_bwd_mb_bwd", (-step(MB, 1), -MB), 1)):
        for m, tz in enumerate(tzs):
            out.append(_last_case(cls, m, tz, 3, ko))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# MapPoint::PredictScale decided by a search's level window
_LIBM = ctypes.CDLL("libm.so.6")
_LIBM.logf.restype, _LIBM.logf.argtypes = ctypes.c_float, [ctypes.c_float]


def logf(x):
    """glibc logf, the function std::log(float) calls on x86 (k_match.cu restates it as glibc_logf)."""
    return f32(_LIBM.logf(float(f32(x))))


LOG_SCALE = logf(SCALE[1])                       # Frame::mfLogScaleFactor = log(mfScaleFactor) (Frame.cc:71)


def predict_scale(mx, dist):
    """MapPoint::PredictScale (MapPoint.cc:385-417, k_match.cu:63-74) for a positive normal ratio: ceil(logf(mfMaxDistance /
    dist) / mfLogScaleFactor) in float, clamped to the pyramid."""
    ratio = f32(f32(mx) / f32(dist))
    assert np.isfinite(ratio) and ratio >= np.finfo(np.float32).tiny
    return int(np.clip(np.ceil(f32(logf(ratio) / LOG_SCALE)), 0, N_LEVELS - 1))


PS_LEVEL = 2
# class: (deciding method, key octave).  Level PS_LEVEL + 1 against PS_LEVEL: the keyframe overload's window [L - 1, L + 1]
# holds octave PS_LEVEL + 2 only at the higher level; the windows [L - 1, L] of the others hold octave PS_LEVEL + 1 only there
PREDICT_SCALE = {
    "predict_scale_kf": ("kf", PS_LEVEL + 2),                  # ORBmatcher.cc:1520-1523
    "predict_scale_local": ("local_match", PS_LEVEL + 1),      # isInFrustum's mnTrackScaleLevel (Frame.cc:312), :100-103
    "predict_scale_sim3proj": ("sim3proj", PS_LEVEL + 1),      # :348-357, :376-378
    "predict_scale_fuse_kf": ("fuse_kf", PS_LEVEL + 1),        # :878-887, :907
    "predict_scale_fuse": ("fuse", PS_LEVEL + 1),              # :1036-1046, :1062
    "predict_scale_sim3": ("sim3", PS_LEVEL + 1),              # :1186, :1266 (identity Sim3: both directions alike)
}


def predict_scale_pair():
    """(mx_low, mx_high): adjacent mfMaxDistance values around dist * sf^PS_LEVEL whose predicted levels are PS_LEVEL and
    PS_LEVEL + 1 for the boundary point's distance."""
    _, dist = norm_po(np.array(U0_CAM, np.float32) - T_CW[:, 3])
    r = f32(dist * f32(1.2) ** PS_LEVEL)
    return bisect(lambda mx: predict_scale(mx, dist) > PS_LEVEL, f32(r * f32(0.99)), f32(r * f32(1.01)))


def _pairs_predict_scale():
    out = []
    a, b = predict_scale_pair()
    for cls, (_, ko) in PREDICT_SCALE.items():
        for m, mx in enumerate((b, a)):
            out.append(_world_case(cls, m, U0_CAM, (U0 + 0.5, V0), mx=mx, key_oct=ko))
    # mfMaxDistance/dist overflowing to +inf: logf(inf) = inf, and the reference's (int)ceil(inf) is INT_MIN, clamped to level 0;
    # one step below, the ratio is finite and the level 7.  Converting +inf to int is undefined in C++: INT_MIN is what x86's
    # cvttss2si returns, so this pair pins the kernel to the reference as built on x86; a toolchain or platform that converts
    # differently flips the reference's member 0, not a kernel bug.  The point at a quarter of U0_CAM's depth has dist < 1, so a finite
    # mfMaxDistance (with 1.2f*mfMaxDistance finite) overflows the ratio; the key at octave 0 is in level 0's windows only
    for m, mx in enumerate(reversed(ratio_inf_pair())):
        out.append(_world_case("predict_scale_ratio_inf", m, NEAR_CAM, (U0 + 0.5, V0), mx=mx, mn=f32(0.0)))
    return out


NEAR_CAM = (0.125, 0.0625, 0.5)                 # projects to (445, 302.5) like U0_CAM


def ratio_inf_pair():
    """(mx_finite, mx_inf): adjacent mfMaxDistance values, the upper one the first whose ratio to NEAR_CAM's dist overflows."""
    _, dist = norm_po(np.array(NEAR_CAM, np.float32) - T_CW[:, 3])
    big = np.finfo(np.float32).max
    with np.errstate(over="ignore"):
        return bisect(lambda mx: bool(np.isinf(f32(f32(mx) / dist))), f32(big * f32(dist) * f32(0.5)), f32(big * f32(dist) * f32(1.5)))


def _proj_case(cls, member, key_xy, ur=-1.0, vc=0.9, th=1.0, xr=46.0, bounds=BOUNDS, q0=(100.0, 100.0)):
    """SearchByProjection(F, vpMapPoints, th) with query 0 at q0, level 0, and its keypoint at key_xy; two ordinary queries
    with keypoints right on their projections."""
    xy = [key_xy, (300.0, 200.0), (500.0, 400.0)]
    keys = _keys(xy)
    desc = _desc(zlib.crc32(cls.encode()) % 1000 + 11, 3)
    urs = np.array([ur, -1.0, 250.0], np.float32)
    F = FrameView(mvKeysUn=keys, mDescriptors=desc, mvScaleFactors=SCALE, bounds=bounds, mvuRight=urs)
    mps = MapPointsView(mTrackProjX=np.array([q0[0], 300.0, 500.0], np.float32), mTrackProjY=np.array([q0[1], 200.0, 400.0], np.float32),
                        mTrackProjXR=np.array([xr, 250.0, 250.0], np.float32), mnTrackScaleLevel=np.zeros(3, np.int32),
                        mTrackViewCos=np.array([vc, 0.9, 0.999], np.float32), descriptors=desc.copy(), valid=np.ones(3, np.uint8),
                        has_obs=np.ones(3, np.uint8))
    return dict(cls=cls, member=member, kind="proj", F=F, mps=mps, th=th, ratio=0.8)


def _pairs_proj():
    out = []
    # radius 4 (mTrackViewCos 0.9, th 1, level 0): |dx| == 4 is outside, one step less inside
    for m, x in enumerate((step(104.0, -1), f32(104.0))):
        out.append(_proj_case("proj_dx_eq_rs", m, (float(x), 100.0)))
    for m, y in enumerate((step(104.0, -1), f32(104.0))):
        out.append(_proj_case("proj_dy_eq_rs", m, (100.0, float(y))))
    # |xr - ur| == rs is kept, one step more is rejected
    for m, ur in enumerate((f32(50.0), step(50.0, 1))):
        out.append(_proj_case("proj_er_eq_rs", m, (101.0, 100.0), ur=ur))
    # ur == 0: no stereo test (er = 46 would reject); the smallest positive ur has one
    for m, ur in enumerate((f32(0.0), step(0.0, 1))):
        out.append(_proj_case("proj_ur_zero", m, (101.0, 100.0), ur=ur))
    # 0.998f > 0.998 in double: radius 2.5 (dx = 3 outside); one step below: radius 4 (inside)
    for m, vc in enumerate((step(0.998, -1), f32(0.998))):
        out.append(_proj_case("proj_view_cos_0998", m, (103.0, 100.0), vc=vc))
    # th == 1 leaves r = 4 (dx = 4 outside); th one step above 1 gives rs = 4*(1 + 2^-23) (inside)
    for m, th in enumerate((step(1.0, 1), f32(1.0))):
        out.append(_proj_case("proj_th_one", m, (104.0, 100.0), th=float(th)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchForTriangulation: F12 makes the epipolar line of kp1 the row y = kp1.y (a = 0, b = -1, c = y1, den = 1)
TRI_F12 = np.array([[0, 0, 0], [0, 0, 1], [0, -1, 0]], np.float32)
TRI_OW1 = np.array([0.5, 0.25, 2.0], np.float32)        # with T2w = I the epipole is (445, 302.5) exactly
TRI_T2W = np.eye(4, dtype=np.float32)[:3]


def epipole():
    """C2 = R2w*Cw + t2w, ex = fx*C2x*invz + cx (src/ORBmatcher.cc:663-670)."""
    C2 = cam_point(TRI_T2W, TRI_OW1)
    fx, fy, cx, cy = [f32(k) for k in K_CAM]
    invz = f32(f32(1.0) / C2[2])
    return float(f32(f32(f32(fx * C2[0]) * invz) + cx)), float(f32(f32(f32(fy * C2[1]) * invz) + cy))


def _tri_case(cls, member, kp1, kp2, ur1, ur2, oct2=0):
    k1 = _keys([kp1, (50.0, 20.0)])
    k2 = _keys([kp2, (60.0, 400.0)])
    k2["octave"][0] = oct2
    d = _desc(zlib.crc32(cls.encode()) % 1000 + 13, 2)
    mk = lambda k, ur: KeyFrameView(mvKeysUn=k, mDescriptors=d.copy(), mFeatVec=FeatureVector.from_nodes(np.zeros(2, np.int64)),
                                    has_mp=np.zeros(2, np.uint8), mvuRight=np.array([ur, 5.0], np.float32), mvScaleFactors=SCALE,
                                    mvLevelSigma2=SIGMA2)
    return dict(cls=cls, member=member, kind="tri", kf1=mk(k1, ur1), kf2=mk(k2, ur2), F12=TRI_F12, Ow1=TRI_OW1, T2w=TRI_T2W,
                ep=epipole(), only_stereo=False, ori=False)


def _pairs_tri():
    out = []
    ex, ey = epipole()
    # both monocular: (ex - x2)^2 == 100*scale[0] is kept; one step closer is rejected.  num = 0, so the line test passes
    for m, x2 in enumerate((f32(ex + 10.0), step(ex + 10.0, -1))):
        out.append(_tri_case("tri_epipole", m, (200.0, ey), (float(x2), ey), -1.0, -1.0))
    # kp1 stereo (no epipole test); kp2 on row 0, so num = y1 and dsqr = y1*y1: bisect y1, keeping the first octave whose
    # pair a float restatement of the 3.84 test would decide differently
    def dsqr_pair(o):
        a, b = bisect(lambda y: not (f64(f32(y * y)) < 3.84 * f64(SIGMA2[o])), f32(0.5), f32(20.0))
        in_float = [not (f32(y * y) < f32(f32(3.84) * SIGMA2[o])) for y in (a, b)]
        return (a, b) if in_float != [False, True] else None
    o, (a, b) = first_separating(dsqr_pair, [(o,) for o in range(N_LEVELS)])
    for m, y1 in enumerate((a, b)):
        out.append(_tri_case("tri_dsqr", m, (200.0, float(y1)), (300.0, 0.0), 10.0, -1.0, oct2=o))
    # den == 0 (:690): F12 = [[0, 0, 0], [0, 0, 0], [0, g, 0]] gives a = c = 0, b = g, den = g*g and num = 0 at y2 = 0; the
    # largest g whose square underflows to 0 is rejected, the next one (den > 0, dsqr = 0) is kept
    g0, g1 = bisect(lambda g: f32(g * g) > 0, f32(0.0), f32(1.0))
    for m, g in enumerate((g1, g0)):
        F12 = np.zeros((3, 3), np.float32); F12[2, 1] = g
        out.append(dict(_tri_case("tri_den_zero", m, (200.0, 0.0), (300.0, 0.0), 10.0, -1.0), F12=F12))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchBySim3 under a similarity with scale 2 and a rotation of 90 degrees about z: every product below is exact, and the
# chained camera-frame point is about half (1 -> 2) or twice (2 -> 1) as far from its camera as the first point of the chain
# is from the other, so a distance gate evaluated on the wrong point of the chain decides both members alike
R90 = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], np.float32)
SIM_A = (f32(2.0), R90, np.array([0.25, -0.5, 0.125], np.float32))
SIM_B = (f32(2.0), R90, np.array([0.25, -0.5, -0.125], np.float32))         # t21.z > 0: p3Dc2.z > 0 for p3Dc1 = (0, 0, +-z)
S3_T1 = T_CW
S3_T2 = np.array([[1, 0, 0, -0.125], [0, 1, 0, 0.25], [0, 0, 1, 0.5]], np.float32)
S3_ORDINARY = (-0.25, -0.125, 2.0)              # camera point of the ordinary mutual match (index 1), in both directions
S3_C0 = (0.5, 0.25, 2.0)                        # camera point of the boundary match; projects to (445, 302.5)


def sim3_mats(s12, R12, t12):
    """S12 = [s12*R12 | t12] and S21 = [(1.0/s12)*R12^T | -sR21*t12] (ORBmatcher.cc:1118-1122), in the float arithmetic cv::Mat
    evaluates them with."""
    R12 = np.asarray(R12, np.float32)
    sR12 = (f32(s12) * R12).astype(np.float32)
    sR21 = (f32(f64(1.0) / f64(s12)) * R12.T).astype(np.float32)
    neg = (-sR21).astype(np.float32)
    t21 = np.array([f32(f32(f32(neg[r, 0] * t12[0]) + f32(neg[r, 1] * t12[1])) + f32(neg[r, 2] * t12[2])) for r in range(3)], np.float32)
    return (np.concatenate([sR12, np.asarray(t12, np.float32).reshape(3, 1)], 1).astype(np.float32),
            np.concatenate([sR21, t21.reshape(3, 1)], 1).astype(np.float32))


def sim3_chain(Tw, S, P):
    """p3Dc2 = sR21*(R1w*p3Dw + t1w) + t21 (:1157-1158; :1237-1238 with the roles swapped), k_match.cu:103-111."""
    return cam_point(S, cam_point(Tw, P))


def project_sim3(p, K=K_CAM):
    """u, v of SearchBySim3: invz = 1.0/z in double rounded to float, u = fx*(x*invz) + cx (:1164-1170)."""
    fx, fy, cx, cy = [f32(k) for k in K]
    invz = f32(f64(1.0) / f64(p[2]))
    return f32(f32(fx * f32(p[0] * invz)) + cx), f32(f32(fy * f32(p[1] * invz)) + cy)


def norm3(p):
    """cv::norm of a float 3-vector: squares accumulated in double, rounded to float."""
    d = np.asarray(p, np.float32).astype(np.float64)
    return f32(np.sqrt(f64(f64(d[0] * d[0]) + f64(d[1] * d[1])) + f64(d[2] * d[2])))


def _sim3_case(cls, member, sim, d12, d21, side=None, mx=None, mn=None, oct0=0):
    """SearchBySim3(KF1, KF2) under sim = (s12, R12, t12), keyframe poses S3_T1 / S3_T2.  KF1's point 0 lands at d12 in camera
    2 and KF2's point 0 at d21 in camera 1, each half a pixel from keypoint 0 of the other keyframe; point 1 of each is an
    ordinary mutual match.  On `side` (12: KF1's point 0, 21: KF2's) mx / mn replace mfMaxDistance / mfMinDistance and the
    keypoint it is searched for has octave oct0."""
    S12, S21 = sim3_mats(*sim)
    desc = _desc(zlib.crc32(cls.encode()) % 1000 + 17, 2)
    keys, pts = {}, {}
    for s, Tw, S_to, S_from, d0 in ((12, S3_T1, S21, S12, d12), (21, S3_T2, S12, S21, d21)):
        P = []
        for d in (d0, S3_ORDINARY):
            d = np.asarray(d, np.float32)
            Pw = (cam_point(S_from, d) - Tw[:, 3]).astype(np.float32)        # the world point whose chain ends at d, exactly
            assert np.array_equal(sim3_chain(Tw, S_to, Pw), d), (cls, s, d)
            P.append(Pw)
        xy = [project_sim3(np.asarray(d, np.float32)) for d in (d0, S3_ORDINARY)]
        k = _keys([(float(u) + 0.5, float(v)) for u, v in xy])
        dists = np.array([norm3(d) for d in (d0, S3_ORDINARY)], np.float32)
        mxs, mns = dists.copy(), (dists * f32(0.5)).astype(np.float32)
        if s == side:
            k["octave"][0] = oct0
            mxs[0] = mxs[0] if mx is None else mx
            mns[0] = mns[0] if mn is None else mn
        keys[s] = k
        pts[s] = WorldPointsView(world_pos=np.array(P, np.float32), descriptors=desc.copy(), max_distance=mxs, min_distance=mns,
                                 normal=np.zeros((2, 3), np.float32), angle=np.zeros(2, np.float32), valid=np.ones(2, np.uint8))
    mk = lambda k: FrameView(mvKeysUn=k, mDescriptors=desc.copy(), mvScaleFactors=SCALE, bounds=BOUNDS)
    # KF1's keypoints are where KF2's points land (direction 2 -> 1) and KF2's where KF1's land (1 -> 2)
    return dict(cls=cls, member=member, kind="sim3", KF1=mk(keys[21]), KF2=mk(keys[12]), P1=pts[12], P2=pts[21], T1w=S3_T1, T2w=S3_T2,
                sim=sim, S12=S12, S21=S21, K=K_CAM, th=7.5)


def sim3_dist_pairs():
    """(dist, (a, b) on 0.8f*mfMinDistance, (a, b) on 1.2f*mfMaxDistance) for the camera-frame point S3_C0."""
    dist = norm3(S3_C0)
    return (dist, bisect(lambda mn: not (dist < f32(f32(0.8) * mn)), dist, f32(dist * 2)),
            bisect(lambda mx: not (dist > f32(f32(1.2) * mx)), f32(dist / 2), dist))


def _pairs_sim3():
    out = []
    # dist3D = cv::norm(p3Dc2) (:1177, :1257) against 0.8f*mfMinDistance / 1.2f*mfMaxDistance, kept member on the bound
    _, (a, b), (c, d) = sim3_dist_pairs()
    for side in (12, 21):
        for m, mn in enumerate((a, b)):
            out.append(_sim3_case(f"sim3_min_dist_{side}", m, SIM_A, S3_C0, S3_C0, side=side, mn=mn))
        for m, mx in enumerate((d, c)):
            out.append(_sim3_case(f"sim3_max_dist_{side}", m, SIM_A, S3_C0, S3_C0, side=side, mx=mx))
    # p3Dc2.z < 0 (:1161, :1241): the chained point at (0, 0, +-z) projects onto (cx, cy) with either sign (x*invz = +-0), while
    # the point in the other camera has positive depth in both members; mfMaxDistance 1 puts the predicted level at 7
    for m, z in enumerate((f32(0.03125), f32(-0.03125))):
        out.append(_sim3_case("sim3_depth_12", m, SIM_A, (0.0, 0.0, z), S3_C0, side=12, mx=f32(1.0), mn=f32(0.0), oct0=7))
    for m, z in enumerate((f32(0.0625), f32(-0.0625))):
        out.append(_sim3_case("sim3_depth_21", m, SIM_B, S3_C0, (0.0, 0.0, z), side=21, mx=f32(1.0), mn=f32(0.0), oct0=7))
    # These pairs are not one float step apart, and no such pair can exist at z = +-0: there 1/z is infinite, so x*invz is NaN
    # (x == 0) or +-inf, and IsInImage drops the point whichever way the depth test went.  A < / <= slip at 0 therefore changes
    # no outcome; what the pairs pin is that the test exists and is taken on the chained point.
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# The rotation histogram (checkOrientation = true) of the LastFrame and KeyFrame overloads and of SearchForTriangulation:
# rot = a1 - a2, rot + 360.0f below 0, bin = round(rot*(1.0f/30)) rounded half away from zero (match_rules.cuh:29-35);
# after the search only the three fullest bins survive (ComputeThreeMaxima).  Nine ordinary matches fill bins 3/3/2/1; the
# boundary match joins the first bin in the kept member and lands in an empty bin, culled as the fourth, in the other.
FACTOR = f32(f32(1.0) / f32(30.0))
ROT_BINS = {"zero": (0, 0, 0, 5, 5, 5, 20, 20, 25), "half": (1, 1, 1, 10, 10, 10, 20, 20, 25)}


def rot_bin(a1, a2):
    """The reference's bin of rot = a1 - a2 (ORBmatcher.cc:1430-1436): std::round of the float product, half away from zero."""
    rot = f32(f32(a1) - f32(a2))
    if rot < 0.0:
        rot = f32(rot + f32(360.0))
    x = f32(rot * FACTOR)
    b = int(np.copysign(np.floor(abs(f64(x)) + 0.5), x))
    return 0 if b == 30 else b


def rot_half_pair():
    """(rot_low, rot_high): adjacent floats, rot_high the first whose product with 1/30 rounds to bin 1 (product exactly 0.5)."""
    return bisect(lambda r: rot_bin(r, 0.0) >= 1, f32(14.0), f32(16.0))


def rot_boundaries():
    """class suffix -> ((a1, a2) of the kept member, (a1, a2) of the culled one)."""
    lo, hi = rot_half_pair()
    return {"zero": ((f32(-0.0), f32(0.0)), (f32(0.0), step(0.0, 1))),    # rot = -0.0: bin 0; rot = -2^-149: 360.0f, bin 12
            "half": ((hi, f32(0.0)), (lo, f32(0.0)))}                     # 0.5 rounds up to bin 1; one step below is bin 0


_ROT_CAMS = [(x, y, 2.0) for y in (-0.375, 0.0) for x in (-0.75, -0.5, -0.25, 0.0, 0.25)][:9]


def _rot_world_case(cls, member, kind, bins, a0):
    """The boundary point U0_CAM (keypoint 0) and nine ordinary points, each matched by the keypoint half a pixel from its
    projection; the source angle (the last frame's keypoint, or the keyframe's mvKeysUn[i].angle) is 30*bin for the ordinary
    matches, and (a1, a2) = a0 for the boundary one."""
    cams = [U0_CAM] + _ROT_CAMS
    P = np.array([[c[0] - T_CW[0, 3], c[1] - T_CW[1, 3], c[2] - T_CW[2, 3]] for c in cams], np.float32)
    n = len(P)
    xy = [(float(u) + 0.5, float(v)) for u, v in (project_frustum(np.array(c, np.float32)) for c in cams)]
    keys = _keys(xy)
    src = np.array([a0[0]] + [f32(30.0) * f32(b) for b in bins], np.float32)
    keys["angle"] = np.array([a0[1]] + [0.0] * len(bins), np.float32)
    desc = _desc(zlib.crc32(cls.encode()) % 1000 + 19, n)
    dists = np.array([norm_po(p)[1] for p in P], np.float32)
    F = FrameView(mvKeysUn=keys, mDescriptors=desc, mvScaleFactors=SCALE, bounds=BOUNDS, mvuRight=np.full(n, -1.0, np.float32))
    Pv = WorldPointsView(world_pos=P, descriptors=desc.copy(), max_distance=dists, min_distance=(dists * f32(0.5)).astype(np.float32),
                         normal=np.array([norm_po(p)[0] / d for p, d in zip(P, dists)], np.float32), angle=src, valid=np.ones(n, np.uint8))
    return dict(cls=cls, member=member, kind=kind, F=F, P=Pv, Tcw=T_CW, Ow=OW, K=K_CAM, bf=BF, th=3.0, vcl=0.5, has_obs=np.ones(n, np.uint8),
                ori=True, last_angle=src)


def _rot_tri_case(cls, member, bins, a0):
    """SearchForTriangulation with ten keypoint pairs on rows 50, 70, ... (the epipolar line of kp1 is its row): pair 0 is the
    boundary match with (kp1.angle, kp2.angle) = a0, pair i the ordinary one with kp1.angle = 30*bin."""
    n = len(bins) + 1
    k1 = _keys([(200.0, 50.0 + 20.0 * i) for i in range(n)])
    k2 = _keys([(300.0, 50.0 + 20.0 * i) for i in range(n)])
    k1["angle"] = np.array([a0[0]] + [f32(30.0) * f32(b) for b in bins], np.float32)
    k2["angle"] = np.array([a0[1]] + [0.0] * len(bins), np.float32)
    d = _desc(zlib.crc32(cls.encode()) % 1000 + 23, n)
    mk = lambda k: KeyFrameView(mvKeysUn=k, mDescriptors=d.copy(), mFeatVec=FeatureVector.from_nodes(np.zeros(n, np.int64)),
                                has_mp=np.zeros(n, np.uint8), mvuRight=np.full(n, -1.0, np.float32), mvScaleFactors=SCALE,
                                mvLevelSigma2=SIGMA2)
    return dict(cls=cls, member=member, kind="tri", kf1=mk(k1), kf2=mk(k2), F12=TRI_F12, Ow1=TRI_OW1, T2w=TRI_T2W, ep=epipole(),
                only_stereo=False, ori=True)


def _pairs_rot():
    out = []
    for which, members in rot_boundaries().items():
        bins = ROT_BINS[which]
        for m, a0 in enumerate(members):
            for kind in ("last", "kf"):
                out.append(_rot_world_case(f"rot_{which}_{kind}", m, kind, bins, a0))
            out.append(_rot_tri_case(f"rot_{which}_tri", m, bins, a0))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# GetFeaturesInArea's cell window (Frame.cc:332-344, area_window in k_proj.cu): the key that the square |dx| < r keeps at its
# outermost float lies in the window's edge cell, so a window one cell narrower on that side loses the match.  SearchByProjection
# with query 0 at (qx, qy) and radius 9 (th 2.25 * 4): the kept member's key is the outermost float the square keeps, the other's
# the next float out (rejected).  With the grid cell 10 px wide, (q -+ 9)/10 = 9.1 / 10.9 leaves the edge key in the edge cell by
# PosInGrid's rounding; near the borders the window is clamped to column 0 / 63 and row 0 / 47.
AREA_EDGES = {                         # class: (bounds, (qx, qy), axis, side)
    "area_edge_left": (BOUNDS, (100.0, 100.0), 0, -1),
    "area_edge_right": (BOUNDS, (100.0, 100.0), 0, 1),
    "area_edge_col0": (BOUNDS, (7.0, 100.0), 0, -1),             # floor(-0.2) = -1, clamped to 0
    "area_edge_col63": (BOUNDS, (623.0, 100.0), 0, 1),           # ceil(63.2) = 64, clamped to 63
    "area_edge_row0": (BOUNDS, (100.0, 7.0), 1, -1),
    "area_edge_row47": (BOUNDS, (100.0, 463.0), 1, 1),
    "area_edge_minx": ((100.0, 0.0, 740.0, 480.0), (109.0, 100.0), 0, -1),   # the key at x == minX > 0
}
AREA_R = f32(9.0)


def grid_cell(F, x, y):
    """Frame::PosInGrid (Frame.cc:386-395): round((x - mnMinX)*mfGridElementWidthInv), likewise for y; None outside the grid."""
    minX, minY, maxX, maxY = [f32(b) for b in F.bounds]
    invW, invH = f32(f32(64) / f32(maxX - minX)), f32(f32(48) / f32(maxY - minY))
    cx, cy = [int(np.copysign(np.floor(abs(f64(t)) + 0.5), t)) for t in (f32(f32(f32(x) - minX) * invW), f32(f32(f32(y) - minY) * invH))]
    return (cx, cy) if 0 <= cx < 64 and 0 <= cy < 48 else None


def area_window(F, x, y, r):
    """The cell window of GetFeaturesInArea(x, y, r) (Frame.cc:332-344): (c0x, c1x, c0y, c1y), clamped to the grid."""
    minX, minY, maxX, maxY = [f32(b) for b in F.bounds]
    invW, invH = f32(f32(64) / f32(maxX - minX)), f32(f32(48) / f32(maxY - minY))
    x, y, r = f32(x), f32(y), f32(r)
    return (max(0, int(np.floor(f32(f32(f32(x - minX) - r) * invW)))), min(63, int(np.ceil(f32(f32(f32(x - minX) + r) * invW)))),
            max(0, int(np.floor(f32(f32(f32(y - minY) - r) * invH)))), min(47, int(np.ceil(f32(f32(f32(y - minY) + r) * invH)))))


def _pairs_area_edges():
    out = []
    for cls, (bounds, q, axis, side) in AREA_EDGES.items():
        # the outermost key the square keeps, |f32(key - q)| < r, and the next float out (kx - q rounds, so this is a bisection)
        inside = lambda k, q=f32(q[axis]): bool(abs(f32(f32(k) - q)) < AREA_R)
        if side > 0:
            kept, out_ = bisect(inside, f32(q[axis]), f32(q[axis] + 2 * AREA_R))
        else:
            out_, kept = bisect(inside, f32(q[axis] - 2 * AREA_R), f32(q[axis]))
        for m, e in enumerate((kept, out_)):
            key = list(q)
            key[axis] = float(e)
            if cls == "area_edge_minx":                # the key stays at minX; the projection moves by one step instead
                c = _proj_case(cls, m, (100.0, 100.0), th=2.25, bounds=bounds, q0=(float(step(f32(109.0), -1 + m)), 100.0))
            else:
                c = _proj_case(cls, m, tuple(key), th=2.25, bounds=bounds, q0=q)
            out.append(c)
    return out


@functools.lru_cache(maxsize=None)
def cases():
    """Every case; world-point cases (no 'kind') are run through every world-point method."""
    return tuple(_pairs_frustum() + _pairs_other_world() + _pairs_last_levels() + _pairs_predict_scale() + _pairs_proj() + _pairs_tri()
                 + _pairs_sim3() + _pairs_rot() + _pairs_area_edges())


# which method decides each class's pair ("local_match": SearchLocalPoints' match rather than isInFrustum's in_view)
DECIDER = {"frustum_max_x": "local", "frustum_min_x": "local", "frustum_min_dist": "local", "frustum_max_dist": "local",
           "frustum_view_cos": "local", "camera_centre": "local", "last_max_x": "last", "kf_max_x": "kf", "image_max_x": "fuse",
           "fuse_normal_dot": "fuse", "fuse_chi2_stereo": "fuse_kf", "fuse_chi2_mono": "fuse_kf", "fuse_kr_zero": "fuse_kf",
           "frustum_max_y": "local", "frustum_min_y": "local", "pcz_sign": "local", "image_min_x": "fuse", "kf_behind_camera": "kf",
           "fwd_bwd_mb_fwd": "last", "fwd_bwd_mb_bwd": "last", **{cls: "last" for cls in LEVEL_PAIRS},
           **{cls: method for cls, (method, _) in PREDICT_SCALE.items()}, "predict_scale_ratio_inf": "local_match"}
WORLD_METHODS = ("local", "last", "kf", "sim3proj", "fuse", "sim3")


def kinds(c):
    return (c["kind"],) if "kind" in c else WORLD_METHODS


def last_view(c):
    """The world-point case as LastFrame: each point observed by a LastFrame keypoint, at octave 0 but for point 0 (last_oct)."""
    P = c["P"]
    n = len(P.world_pos)
    k = _keys([(0.0, 0.0)] * n)
    k["octave"][0] = c.get("last_oct", 0)
    if "last_angle" in c:
        k["angle"] = c["last_angle"]
    return LastFrameView(mvKeysUn=k, world_pos=P.world_pos, descriptors=P.descriptors, valid=np.ones(n, np.uint8), has_obs=np.ones(n, np.uint8))


# SearchBySim3 with the identity similarity: S12 = [1*I | 0], S21 = [(1/1)*I^T | -(sR21*t12)] = [I | -0] (ORBmatcher.cc:1118-1122)
S12_ID = np.concatenate([np.eye(3, dtype=np.float32), np.zeros((3, 1), np.float32)], 1)
S21_ID = np.concatenate([np.eye(3, dtype=np.float32), np.full((3, 1), -0.0, np.float32)], 1)


def sim3_args(c):
    """SearchBySim3(KF1 = KF2 = the case's keyframe, P1 = P2 = its points, T1w = T2w = its pose): both directions project every
    point into the same keyframe."""
    return c["F"], c["F"], c["P"], c["P"], c["Tcw"], c["Tcw"], S12_ID, S21_ID, c["K"], c["th"]


def scw(c):
    """Fuse(pKF, Scw, ...) on the same pose with scale 1: Scw = Tcw; its decomposition is exact."""
    return np.asarray(c["Tcw"], np.float32)


# ---------------------------------------------------------------------------------------------------------------------------
# the port and the verbatim reference, in comparable form
def _local_mps(fr, P, has_obs):
    return MapPointsView(fr["proj_x"], fr["proj_y"], fr["proj_xr"], fr["level"], fr["view_cos"], P.descriptors, valid=fr["in_view"],
                         has_obs=has_obs)


def run_port(O, c, method):
    """The port's result of one method on case c."""
    if method == "local":
        fr = O.port_is_in_frustum(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["vcl"])
        n, match = O.port_search_by_projection(c["F"], _local_mps(fr, c["P"], c["has_obs"]), c["th"], 0.8)
        return fr, n, match
    if method == "last":
        Cur = FrameView(c["F"].mvKeysUn, c["F"].mDescriptors, c["F"].mvScaleFactors, c["F"].bounds)
        return O.port_search_by_projection_last(Cur, last_view(c), c["Tcw"], c["K"], c["bf"], c["th"], c.get("fwd", False), c.get("bwd", False),
                                                c.get("ori", False))
    if method == "kf":
        return O.port_search_by_projection_kf(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["th"], 100, c.get("ori", False))
    if method == "sim3proj":
        return O.port_search_by_projection_sim3(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], int(c["th"]))
    if method == "fuse":
        return O.port_fuse(c["F"], c["P"], scw(c), c["Ow"], c["K"], c["bf"], c["th"], True)
    if method == "fuse_kf":
        return O.port_fuse(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], False)
    if method == "sim3" and "kind" in c:
        return O.port_search_by_sim3(c["KF1"], c["KF2"], c["P1"], c["P2"], c["T1w"], c["T2w"], c["S12"], c["S21"], c["K"], c["th"])
    if method == "sim3":
        return O.port_search_by_sim3(*sim3_args(c))
    if method == "proj":
        return O.port_search_by_projection(c["F"], c["mps"], c["th"], c["ratio"])
    if method == "tri":
        return O.port_search_for_triangulation(c["kf1"], c["kf2"], c["F12"], c["ep"], c["only_stereo"], c["ori"])
    raise ValueError(method)


def methods(c):
    k = kinds(c)
    return k + ("fuse_kf",) if "fuse" in k else k


def run_ref(O, c, method):
    """The verbatim reference's result, in the port's form where the two are compared directly."""
    if method == "local":
        fr = O.ref_is_in_frustum(c["F"], c["P"], c["Tcw"], c["K"], c["bf"], c["vcl"])
        mps = _local_mps(fr, c["P"], c["has_obs"])
        return fr, O.ref_search_by_projection(c["F"], mps, c["th"], 0.8), mps
    if method == "last":
        Cur = FrameView(c["F"].mvKeysUn, c["F"].mDescriptors, c["F"].mvScaleFactors, c["F"].bounds)
        # bMono unless the case has a last-frame pose of its own; the reference then decides forward / backward itself
        return O.ref_search_by_projection_last(Cur, last_view(c), c["Tcw"], c.get("Tlast", c["Tcw"]), c["K"], c["bf"], MB, c["th"],
                                               "Tlast" not in c, c.get("ori", False))
    if method == "kf":
        return O.ref_search_by_projection_kf(c["F"], c["P"], c["Tcw"], c["K"], c["th"], 100, c.get("ori", False))
    if method == "sim3proj":
        return O.ref_search_by_projection_sim3(c["F"], c["P"], scw(c), c["K"], int(c["th"]))
    if method == "fuse":
        return O.ref_fuse(c["F"], c["P"], scw(c), O.ref_decompose_scw(scw(c))[1], c["K"], c["bf"], c["th"], True)
    if method == "fuse_kf":
        return O.ref_fuse(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], False)
    if method == "sim3" and "kind" in c:
        return O.ref_search_by_sim3(c["KF1"], c["KF2"], c["P1"], c["P2"], c["T1w"], c["T2w"], *c["sim"], c["K"], c["th"])
    if method == "sim3":
        F, _, P, _, T, _, _, _, K, th = sim3_args(c)
        return O.ref_search_by_sim3(F, F, P, P, T, T, 1.0, np.eye(3, dtype=np.float32), np.zeros(3, np.float32), K, th)
    if method == "proj":
        return O.ref_search_by_projection(c["F"], c["mps"], c["th"], c["ratio"])
    if method == "tri":
        return O.ref_search_for_triangulation(c["kf1"], c["kf2"], c["F12"], c["Ow1"], c["T2w"], K_CAM, c["only_stereo"], c["ori"])
    raise ValueError(method)


def decided(O, c):
    """The reference's decision on the boundary input of case c (True: point / keypoint 0 gets through the gate)."""
    method = c.get("kind") or DECIDER[c["cls"]]
    r = run_ref(O, c, "local" if method == "local_match" else method)
    if method == "local":
        return bool(r[0]["in_view"][0])
    if method == "local_match":
        return bool(r[1][1][0] == 0)
    if method in ("last", "kf", "sim3proj", "proj"):
        return bool((r[1] == 0).any())
    if method in ("fuse", "fuse_kf", "sim3"):
        return bool(r[1][0] == 0)
    if method == "tri":
        return bool(len(r) and (r[:, 0] == 0).any() and (r[r[:, 0] == 0, 1] == 0).all())
    raise ValueError(method)


FLOAT_FIELDS = ("proj_x", "proj_y", "proj_xr", "view_cos")


def same_float(a, b):
    """Bit for bit, except that any NaN equals any NaN (payloads differ between x86 and the GPU)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def frustum_equal(got, want):
    """isInFrustum outputs: in_view and level exactly; the track fields only where in view (elsewhere the MapPoint keeps its
    old values, which both sides report as they please)."""
    iv = np.asarray(want["in_view"], bool)
    if not np.array_equal(np.asarray(got["in_view"], bool), iv) or not np.array_equal(got["level"][iv], want["level"][iv]):
        return False
    return all(same_float(got[f][iv], want[f][iv]) for f in FLOAT_FIELDS)


# ---------------------------------------------------------------------------------------------------------------------------
# dense variants: both members of every world-point class with a natural background of ~1000 keypoints and MapPoints
# (match_fixtures.world_points_case, moved into the case's pose), so that the boundary point rides the multi-wave candidate
# lists and the contested claims of a full-size call
def dense_classes():
    return sorted({c["cls"] for c in cases() if "kind" not in c})


@functools.lru_cache(maxsize=None)
def _background(O):
    from tests import match_fixtures as mf
    v = mf.two_views(O, 7)
    F, P, Tcw, _, _ = mf.world_points_case(v, 7, K=K_CAM)
    m = min(len(F.mvKeysUn), len(P.world_pos))
    R, t = Tcw[:, :3].astype(np.float64), Tcw[:, 3].astype(np.float64)
    Pc = P.world_pos[:m].astype(np.float64) @ R.T + t                  # the background in camera coordinates
    return dict(keys=F.mvKeysUn[:m], desc=F.mDescriptors[:m], occupied=F.occupied[:m], Pc=Pc, pdesc=P.descriptors[:m],
                mx=P.max_distance[:m], mn=P.min_distance[:m], normal=(P.normal[:m].astype(np.float64) @ R.T).astype(np.float32),
                angle=P.angle[:m], valid=P.valid[:m])


def dense_case(O, c):
    """World-point case c with the background appended after its own points and keypoints (index 0 stays the boundary)."""
    bg = _background(O)
    F, P, T = c["F"], c["P"], np.asarray(c["Tcw"], np.float32)
    n, m = len(F.mvKeysUn), len(bg["keys"])
    cat = lambda a, b: np.concatenate([np.asarray(a), np.asarray(b).astype(np.asarray(a).dtype)])
    Fd = FrameView(mvKeysUn=cat(F.mvKeysUn, bg["keys"]), mDescriptors=cat(F.mDescriptors, bg["desc"]), mvScaleFactors=F.mvScaleFactors,
                   bounds=F.bounds, mvuRight=cat(F.mvuRight, np.full(m, -1.0, np.float32)), mvInvLevelSigma2=F.mvInvLevelSigma2,
                   occupied=cat(np.zeros(n, np.uint8), bg["occupied"]))
    world = (bg["Pc"] - T[:, 3].astype(np.float64)).astype(np.float32)        # T = [I | t]: world = camera - t
    Pd = WorldPointsView(world_pos=cat(P.world_pos, world), descriptors=cat(P.descriptors, bg["pdesc"]),
                         max_distance=cat(P.max_distance, bg["mx"]), min_distance=cat(P.min_distance, bg["mn"]),
                         normal=cat(P.normal, bg["normal"]), angle=cat(P.angle, bg["angle"]), valid=cat(P.valid, bg["valid"]))
    return dict(c, F=Fd, P=Pd, has_obs=np.ones(n + m, np.uint8), dense=True)


def dense_cases(O):
    return [dense_case(O, c) for c in cases() if "kind" not in c]
