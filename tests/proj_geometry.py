"""Matcher inputs placed on the float decision boundaries of the projection searches: Frame::isInFrustum, the SearchByProjection
overloads, both Fuse overloads and the epipolar gates of SearchForTriangulation.  Test tooling: tests/test_oracle_proj_geometry.py
pins the port to the verbatim Frame.cc / ORBmatcher.cc on every case and checks that both members of every boundary pair are
decided differently by the verbatim build; tests/test_gpu_proj_geometry.py pins the CUDA library to the port.

Every case is a small call (one boundary point or keypoint, a few ordinary ones) whose outcome is readable.  A pair is two
cases that differ in one free input by one float32 step, found by bisecting over that input's bit patterns with the gate
restated here in numpy float32 / float64, in the reference's operation order.  Each gate is restated next to the kernel line
it exists for.  Nothing in this module calls the CUDA library.

No case separates the two flavours of 1/z the kernels use (1.0f/z and (float)(1.0/(double)z)): they are identical, because a
double quotient rounded to float is the correctly rounded float quotient (53 >= 2*24 + 2, double rounding is innocuous for
division)."""
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
    "frustum_max_x": "k_match.cu:176 u > maxX (inclusive bound) in Frame::isInFrustum",
    "frustum_min_x": "k_match.cu:176 u < minX (inclusive bound) in Frame::isInFrustum",
    "frustum_min_dist": "k_match.cu:210-211 dist < 0.8f*mfMinDistance, dist from cv::norm in double",
    "frustum_max_y": "k_match.cu:176 v > maxY (inclusive bound) in Frame::isInFrustum",
    "frustum_min_y": "k_match.cu:176 v < minY (inclusive bound) in Frame::isInFrustum",
    "frustum_max_dist": "k_match.cu:210-211 dist > 1.2f*mfMaxDistance",
    "frustum_view_cos": "k_match.cu:221-222 viewCos < viewingCosLimit",
    "camera_centre": "k_match.cu:171-178 PcZ == 0: NaN projection and NaN viewCos are in view, as the reference stores them",
    "pcz_sign": "k_match.cu:172 PcZ < 0: PcZ == -0 passes (NaN projection, in view), -(smallest subnormal) does not",
    "last_max_x": "k_match.cu:192 u > maxX in SearchByProjection(CurrentFrame, LastFrame)",
    "kf_max_x": "k_match.cu:192 u > maxX in SearchByProjection(CurrentFrame, KeyFrame)",
    "image_max_x": "k_match.cu:185 KeyFrame::IsInImage u < maxX (half-open) in both Fuse overloads",
    "image_min_x": "k_match.cu:185 KeyFrame::IsInImage u >= minX: the left bound is inside",
    "kf_behind_camera": "k_match.cu:189 the keyframe overload has no depth test: a point behind the camera is found",
    "fuse_normal_dot": "k_match.cu:214-215 PO.dot(Pn) < 0.5*dist in double, both Fuse overloads",
    "fuse_chi2_stereo": "k_proj.cu:225 e2*invSigma2 > 7.8 in double",
    "fuse_chi2_mono": "k_proj.cu:228 e2*invSigma2 > 5.99 in double",
    "fuse_kr_zero": "k_proj.cu:222 kpr >= 0 takes the stereo gate at kpr == +0",
    "proj_dx_eq_rs": "k_proj.cu:82 |dx| < rs (strict)",
    "proj_dy_eq_rs": "k_proj.cu:82 |dy| < rs (strict)",
    "proj_er_eq_rs": "k_proj.cu:86-87 |xr - ur| > rs rejects; equality is kept",
    "proj_ur_zero": "k_proj.cu:85 ur > 0: no stereo test at ur == 0",
    "proj_view_cos_0998": "k_proj.cu:117 mTrackViewCos > 0.998 in double: 0.998f takes radius 2.5",
    "proj_th_one": "k_proj.cu:118 th != 1 scales the radius; th == 1 does not",
    "tri_epipole": "k_match.cu:686-687 distance to the epipole < 100*scale (strict) rejects",
    "tri_dsqr": "k_match.cu:692 dsqr < 3.84*mvLevelSigma2 in double",
    "tri_den_zero": "k_match.cu:690 den == 0 rejects before the division",
}

# rows of the gate table these cases do not reach, each with the reason; test_every_class_is_reached keeps CLASSES and this
# table together, so a gate cannot silently fall out of both
NOT_COVERED = {
    "predict_scale": "MapPoint::PredictScale at ratio = sf^k, dist = 0 and subnormal ratios (k_match.cu:139-150): the restated "
                     "glibc logf is checked on every positive normal float by tests/test_libm_ports.py, and the port's "
                     "predict_scale against the verbatim MapPoint.cc by tests/test_oracle_map_ref.py; no search-level pair yet",
    "area_window_edges": "(x - minX +- r)*invW exactly an integer, and a key at x == minX > 0 (k_proj.cu:66-71): not built",
    "level_gates": "octave 0 / 7 level windows for forward / backward / neither in SearchByProjection(LastFrame) "
                   "(k_match.cu:197-201): not built",
    "sim3_chain": "SearchBySim3's own gates (p3Dc2 < 0, dist3D of the camera-frame point, k_match.cu:166-170,205) at a boundary: "
                  "SearchBySim3 runs on every world-point case with the identity Sim3, but no pair is placed on these gates",
    "rot_bin": "rotation bin at rot = -0.0, rot + 360 -> 360.0f, rot/30 at x.5: a single match is never culled, so these need a "
               "contested histogram; not built",
    "dense_variants": "each class mixed into a natural world_points_case: not built",
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
    """cv::Mat 3x3 * 3x1 + 3x1 in float32: ((r0*p0 + r1*p1) + r2*p2) + t (k_match.cu:162-164)."""
    T, P = np.asarray(T, np.float32), np.asarray(P, np.float32)
    return np.array([f32(f32(f32(T[r, 0] * P[0]) + f32(T[r, 1] * P[1])) + f32(T[r, 2] * P[2])) + T[r, 3] for r in range(3)], np.float32)


def camera_centre(T):
    """mOw = -mRcw.t()*mtcw as cv::Mat evaluates it: the negated transpose times t, ((a0*t0 + a1*t1) + a2*t2) in float, which
    decides the sign of a zero component."""
    A = (-np.asarray(T, np.float32)[:, :3].T).astype(np.float32)
    t = np.asarray(T, np.float32)[:, 3]
    return np.array([f32(f32(f32(A[r, 0] * t[0]) + f32(A[r, 1] * t[1])) + f32(A[r, 2] * t[2])) for r in range(3)], np.float32)


def project_frustum(Pc, K=K_CAM):
    """u, v of Frame::isInFrustum: fx*PcX*invz + cx, invz = 1.0f/PcZ (k_match.cu:173-175)."""
    fx, fy, cx, cy = [f32(k) for k in K]
    invz = f32(f32(1.0) / Pc[2])
    return f32(f32(f32(fx * Pc[0]) * invz) + cx), f32(f32(f32(fy * Pc[1]) * invz) + cy)


def norm_po(P, Ow=OW):
    """(PO, dist): PO = P - Ow in float, dist = cv::norm(PO), squares accumulated in double (k_match.cu:206-208)."""
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


def _world_case(cls, member, cam, key_xy, bounds=BOUNDS, mx=None, mn=None, normal=None, ur=-1.0, inv=None, T=T_CW, world0=None, **kw):
    """One boundary point (index 0, camera coordinates `cam` under the pose T = [I | t], or world position world0) and the
    ordinary points; keypoint f sits at key_xy for point 0 and at its projection + (0.5, 0) for the others.  Descriptors: point
    i equals keypoint i."""
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


def _proj_case(cls, member, key_xy, ur=-1.0, vc=0.9, th=1.0, xr=46.0):
    """SearchByProjection(F, vpMapPoints, th) with query 0 at (100, 100), level 0, and its keypoint at key_xy; two ordinary
    queries with keypoints right on their projections."""
    xy = [key_xy, (300.0, 200.0), (500.0, 400.0)]
    keys = _keys(xy)
    desc = _desc(zlib.crc32(cls.encode()) % 1000 + 11, 3)
    urs = np.array([ur, -1.0, 250.0], np.float32)
    F = FrameView(mvKeysUn=keys, mDescriptors=desc, mvScaleFactors=SCALE, bounds=BOUNDS, mvuRight=urs)
    mps = MapPointsView(mTrackProjX=np.array([100.0, 300.0, 500.0], np.float32), mTrackProjY=np.array([100.0, 200.0, 400.0], np.float32),
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


@functools.lru_cache(maxsize=None)
def cases():
    """Every case; world-point cases (no 'kind') are run through every world-point method."""
    return tuple(_pairs_frustum() + _pairs_other_world() + _pairs_proj() + _pairs_tri())


# which method decides each class's pair
DECIDER = {"frustum_max_x": "local", "frustum_min_x": "local", "frustum_min_dist": "local", "frustum_max_dist": "local",
           "frustum_view_cos": "local", "camera_centre": "local", "last_max_x": "last", "kf_max_x": "kf", "image_max_x": "fuse",
           "fuse_normal_dot": "fuse", "fuse_chi2_stereo": "fuse_kf", "fuse_chi2_mono": "fuse_kf", "fuse_kr_zero": "fuse_kf",
           "frustum_max_y": "local", "frustum_min_y": "local", "pcz_sign": "local", "image_min_x": "fuse", "kf_behind_camera": "kf"}
WORLD_METHODS = ("local", "last", "kf", "sim3proj", "fuse", "sim3")


def kinds(c):
    return (c["kind"],) if "kind" in c else WORLD_METHODS


def last_view(c):
    """The world-point case as LastFrame: each point observed by a LastFrame keypoint at octave 0."""
    P = c["P"]
    n = len(P.world_pos)
    return LastFrameView(mvKeysUn=_keys([(0.0, 0.0)] * n), world_pos=P.world_pos, descriptors=P.descriptors, valid=np.ones(n, np.uint8),
                         has_obs=np.ones(n, np.uint8))


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
        return O.port_search_by_projection_last(Cur, last_view(c), c["Tcw"], c["K"], c["bf"], c["th"], False, False, False)
    if method == "kf":
        return O.port_search_by_projection_kf(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["th"], 100, False)
    if method == "sim3proj":
        return O.port_search_by_projection_sim3(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], int(c["th"]))
    if method == "fuse":
        return O.port_fuse(c["F"], c["P"], scw(c), c["Ow"], c["K"], c["bf"], c["th"], True)
    if method == "fuse_kf":
        return O.port_fuse(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], False)
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
        return O.ref_search_by_projection_last(Cur, last_view(c), c["Tcw"], c["Tcw"], c["K"], c["bf"], c["bf"], c["th"], True, False)
    if method == "kf":
        return O.ref_search_by_projection_kf(c["F"], c["P"], c["Tcw"], c["K"], c["th"], 100, False)
    if method == "sim3proj":
        return O.ref_search_by_projection_sim3(c["F"], c["P"], scw(c), c["K"], int(c["th"]))
    if method == "fuse":
        return O.ref_fuse(c["F"], c["P"], scw(c), O.ref_decompose_scw(scw(c))[1], c["K"], c["bf"], c["th"], True)
    if method == "fuse_kf":
        return O.ref_fuse(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], False)
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
    r = run_ref(O, c, method)
    if method == "local":
        return bool(r[0]["in_view"][0])
    if method in ("last", "kf", "sim3proj", "proj"):
        return bool((r[1] == 0).any())
    if method in ("fuse", "fuse_kf"):
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
