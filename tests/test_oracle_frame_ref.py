"""CPU: pins the restatements of Frame::ComputeStereoMatches (oracle/orb_port_stereo.cpp), of the feature grid and of
Frame::isInFrustum (oracle/orb_port_match.cpp) — and through them the CUDA kernels — to the REFERENCE SOURCE:
/root/reference/src/Frame.cc compiled verbatim against the reference's real include/Frame.h (oracle/_ref/libframeref.so,
oracle/Makefile target `ref`, oracle/frameref_wrap.cpp, oracle/frameshim/pre.hpp)."""
import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import frame_input_cases as fic
from tests import match_fixtures as mf


@pytest.fixture(scope="module")
def O(oracle):
    if not oracle.have_frameref():
        pytest.skip("oracle/_ref/libframeref.so not built (reference tree absent)")
    return oracle


@pytest.mark.parametrize("shape,nf,bf,fx,seed", [((640, 360), 1000, 386.1448, 718.856, 1), ((752, 480), 1200, 47.9, 435.2, 2),
                                                 (synth.KITTI, 2000, 386.1448, 718.856, 3)])
def test_compute_stereo_matches_equals_reference_source(O, shape, nf, bf, fx, seed):
    w, h = shape
    L, R, _ = synth.stereo_pair(seed, 0, 0, w, h)
    E1, E2 = O.PortExtractor(nf), O.PortExtractor(nf)
    kl, dl = E1(L)
    kr, dr = E2(R)
    pl, pr = [E1.level(i) for i in range(8)], [E2.level(i) for i in range(8)]
    ur_p, dp_p, _ = O.port_stereo(kl, dl, kr, dr, pl, pr, E1.scale, E1.inv_scale, bf, fx)
    ur_r, dp_r = O.ref_stereo(kl, dl, kr, dr, pl, pr, E1.scale, E1.inv_scale, bf, fx)
    assert (ur_r >= 0).sum() > 0.3 * len(kl)
    assert np.array_equal(ur_r, ur_p) and np.array_equal(dp_r, dp_p), int((ur_r != ur_p).sum())


def test_stereo_degenerate_inputs(O):
    """Unrelated left / right images (few, poor matches: the median cull and the rejection branches dominate)."""
    L = synth.mono_frame(5, 0, 0, 640, 360)
    R = synth.mono_frame(6, 0, 0, 640, 360)
    E1, E2 = O.PortExtractor(800), O.PortExtractor(800)
    kl, dl = E1(L)
    kr, dr = E2(R)
    pl, pr = [E1.level(i) for i in range(8)], [E2.level(i) for i in range(8)]
    ur_p, dp_p, _ = O.port_stereo(kl, dl, kr, dr, pl, pr, E1.scale, E1.inv_scale, 386.1448, 718.856)
    ur_r, dp_r = O.ref_stereo(kl, dl, kr, dr, pl, pr, E1.scale, E1.inv_scale, 386.1448, 718.856)
    assert np.array_equal(ur_r, ur_p) and np.array_equal(dp_r, dp_p)


def test_feature_grid_equals_reference_source(O):
    v = mf.two_views(O, 7)
    k = v["kl"]
    rng = np.random.default_rng(1)
    for bounds in [(0.0, 0.0, 640.0, 480.0), (-12.5, -7.25, 652.0, 491.5)]:
        for _ in range(150):
            x, y, r = rng.uniform(-30, 670), rng.uniform(-30, 510), rng.uniform(2, 80)
            lo = int(rng.integers(-1, 7)); hi = int(rng.integers(-1, 8))
            got = O.port_features_in_area(k, bounds, x, y, r, lo, hi)
            want = O.ref_features_in_area(k, bounds, x, y, r, lo, hi)
            assert np.array_equal(got, want), (bounds, x, y, r, lo, hi)          # same features in the same order


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("limit", [0.5, 0.8])
def test_is_in_frustum_equals_reference_source(O, seed, limit):
    v = mf.two_views(O, seed)
    F, P, Tcw, _, K = mf.world_points_case(v, seed + 70)
    ref = O.ref_is_in_frustum(F, P, Tcw, K, 40.0, limit)
    port = O.port_is_in_frustum(F, P, Tcw, ref["Ow"], K, 40.0, limit)              # mOw as Frame::UpdatePoseMatrices computes it
    assert ref["count"] == port["count"] > 100
    for f in ("in_view", "proj_x", "proj_y", "proj_xr", "level", "view_cos"):
        assert np.array_equal(ref[f], port[f]), f


TUM1_K = (517.306408, 516.469215, 318.643040, 255.313989)
TUM1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)


def _synthetic_depth(seed, w=640, h=480):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    raw = (5000.0 * (1.5 + 0.8 * np.sin(xx / 90.0) * np.cos(yy / 70.0))).astype(np.uint16)
    raw[rng.random((h, w)) < 0.15] = 0                       # holes of the depth sensor
    return raw


@pytest.mark.parametrize("dist", [TUM1_DIST, TUM1_DIST[:4], (0.0, 0.0, 0.0, 0.0), (-0.28, 0.07, 0.0002, 0.00002)])
def test_rgbd_leg_port_equals_reference_and_cv2(oracle, dist):
    """UndistortKeyPoints + ComputeStereoFromRGBD + ComputeImageBounds (src/Frame.cc:404-464, :643-664): the restatement equals the
    verbatim Frame.cc (whose cv::undistortPoints stand-in is itself pinned here against cv2 4.13) bit for bit."""
    import cv2
    if not oracle.have_frameref():
        pytest.skip("libframeref.so not built")
    from orb_slam2_b200 import synth
    E = oracle.PortExtractor(1000)
    keys, _ = E(synth.mono_frame(5, 0, 0, 640, 480))
    depth = oracle.port_depth_to_float(_synthetic_depth(3), 1.0 / 5000.0)
    assert np.array_equal(depth, _synthetic_depth(3).astype(np.float32) * np.float32(1.0 / 5000.0))
    K4 = np.array(TUM1_K, np.float32); D = np.array(dist, np.float32)
    p = oracle.port_rgbd_frame(keys, K4, D, 40.0, depth)
    r = oracle.ref_rgbd_frame(keys, K4, D, 40.0, depth)
    for f in ("keys_un", "u_right", "depth", "bounds"):
        assert np.array_equal(p[f], r[f]), f
    assert p["count"] == r["count"] > 500
    # cv2 pin of the un-vendored primitive
    Km = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1]], np.float32)
    pts = np.stack([keys["x"], keys["y"]], 1).astype(np.float32).reshape(-1, 1, 2)
    if D[0] != 0:
        und = cv2.undistortPoints(pts, Km, D.reshape(-1, 1), None, Km).reshape(-1, 2)
        assert np.array_equal(und[:, 0], p["keys_un"]["x"]) and np.array_equal(und[:, 1], p["keys_un"]["y"])
        assert np.abs(und - pts.reshape(-1, 2)).max() > 0.5
        corners = cv2.undistortPoints(np.array([[[0, 0]], [[640, 0]], [[0, 480]], [[640, 480]]], np.float32), Km, D.reshape(-1, 1), None, Km).reshape(4, 2)
        want = [min(corners[0, 0], corners[2, 0]), min(corners[0, 1], corners[1, 1]), max(corners[1, 0], corners[3, 0]), max(corners[2, 1], corners[3, 1])]
        assert np.array_equal(p["bounds"], np.array(want, np.float32))
    else:
        assert np.array_equal(p["keys_un"], keys) and np.array_equal(p["bounds"], np.array([0, 0, 640, 480], np.float32))
    # depth association semantics: truncating (v, u) lookup on the DISTORTED keypoint, uRight from the undistorted x
    i = int(np.nonzero(p["depth"] > 0)[0][0])
    assert p["depth"][i] == depth[int(keys["y"][i]), int(keys["x"][i])]
    assert p["u_right"][i] == np.float32(p["keys_un"]["x"][i] - np.float32(40.0) / p["depth"][i])
    assert np.all(p["u_right"][p["depth"] < 0] == -1)


def _bits(a):
    """Bitwise identity (NaN payloads, signed zeros), also for structured arrays."""
    return np.ascontiguousarray(a).tobytes()


def _grid_keys(O, seed):
    """Extractor keypoints, plus keys placed on and around the grid's edges (rounding to -0, to column 64 / row 48, far outside)."""
    E = O.PortExtractor(1500)
    keys, _ = E(synth.mono_frame(seed, 0, 0, 640, 480))
    rng = np.random.default_rng(seed)
    extra = np.zeros(400, keys.dtype)
    extra["x"] = np.concatenate([rng.uniform(-60, 700, 200), rng.choice([-5.01, -4.99, -0.01, 0.0, 4.99, 5.0, 634.99, 640.0, 645.0, 1e9, -1e9, np.nan], 200)])
    extra["y"] = np.concatenate([rng.uniform(-60, 540, 200), rng.choice([-5.01, -4.99, -0.01, 0.0, 4.99, 5.0, 474.99, 480.0, 485.0, 1e9, -1e9, np.nan], 200)])
    extra["octave"] = rng.integers(0, 8, 400)
    k = np.concatenate([keys, extra])
    return k[rng.permutation(len(k))]


@pytest.mark.parametrize("bounds", [(0.0, 0.0, 640.0, 480.0), (-12.5, -7.25, 652.0, 491.5), (3.75, 2.5, 636.0, 478.25),
                                    (37.1, 21.9, 611.3, 455.2), (0.0, 0.0, 1241.0, 376.0), (-180.4, -140.2, 812.6, 611.7)])
def test_feature_grid_cells_equal_reference_source(O, bounds):
    """The whole grid, cell by cell in insertion order, as the device keeps it (cell = x*48 + y).  A positive min_x puts keys left
    of the bound at (x - min_x) * invW in (-0.5, 0): round() gives -0 and the key lands in column 0; further left it is dropped."""
    k = _grid_keys(O, 11)
    cs_p, ci_p = O.port_assign_grid(k, bounds)
    cs_r, ci_r = O.ref_assign_grid(k, bounds)
    assert np.array_equal(cs_p, cs_r) and np.array_equal(ci_p, ci_r)
    assert 0 < cs_r[-1] < len(k)                                          # some keys fall outside the grid
    assert np.all(np.diff(cs_r) >= 0)
    if bounds[0] > 0:
        invw = np.float32(64) / np.float32(np.float32(bounds[2]) - np.float32(bounds[0]))
        t = (k["x"] - np.float32(bounds[0])) * invw
        invh = np.float32(48) / np.float32(np.float32(bounds[3]) - np.float32(bounds[1]))
        ty = (k["y"] - np.float32(bounds[1])) * invh
        neg0 = np.nonzero((t < 0) & (t > -0.49) & (ty > -0.49) & (ty < 47.49))[0]
        assert len(neg0) > 0 and set(neg0.tolist()) <= set(ci_r[:cs_r[48]].tolist())      # column 0 = cells 0..47


@pytest.mark.parametrize("case", sorted(fic.DIST_CASES))
def test_undistort_and_bounds_sweep_port_equals_reference_and_cv2(O, case):
    """UndistortKeyPoints + ComputeImageBounds over the camera models of the frame-input sweep: k1 == 0 with nonzero k2 / p1 / p2 /
    k3 (the reference copies the keys unchanged), k1 == -0.0, 4- and 5-coefficient models, strong pincushion, and a model whose
    1/(1 + k1 r^2) turns negative inside the image (cv::undistortPoints then gives up on the point and keeps its normalised
    coordinates), which also moves the image bounds."""
    import cv2
    K, dist = fic.DIST_CASES[case]
    E = O.PortExtractor(1500)
    keys, _ = E(synth.mono_frame(12, 0, 0, 640, 480))
    depth = fic.edge_depth_float(5)
    K4 = np.array(K, np.float32); D = np.array(dist, np.float32)
    p = O.port_rgbd_frame(keys, K4, D, 40.0, depth)
    r = O.ref_rgbd_frame(keys, K4, D, 40.0, depth)
    for f in ("keys_un", "u_right", "depth", "bounds"):
        assert _bits(p[f]) == _bits(r[f]), f
    if D[0] == 0:                                                         # == also holds for -0.0
        assert np.array_equal(p["keys_un"], keys) and np.array_equal(p["bounds"], np.array([0, 0, 640, 480], np.float32))
        return
    Km = np.array([[K4[0], 0, K4[2]], [0, K4[1], K4[3]], [0, 0, 1]], np.float32)
    pts = np.stack([keys["x"], keys["y"]], 1).astype(np.float32).reshape(-1, 1, 2)
    und = cv2.undistortPoints(pts, Km, D.reshape(-1, 1), None, Km).reshape(-1, 2)
    assert np.array_equal(und[:, 0], p["keys_un"]["x"]) and np.array_equal(und[:, 1], p["keys_un"]["y"])
    corners = cv2.undistortPoints(np.array([[[0, 0]], [[640, 0]], [[0, 480]], [[640, 480]]], np.float32), Km, D.reshape(-1, 1), None, Km).reshape(4, 2)
    want = [min(corners[0, 0], corners[2, 0]), min(corners[0, 1], corners[1, 1]), max(corners[1, 0], corners[3, 0]), max(corners[2, 1], corners[3, 1])]
    assert np.array_equal(p["bounds"], np.array(want, np.float32))
    if case == "icdist_negative":
        x = (keys["x"].astype(np.float64) - K[2]) / K[0]; y = (keys["y"].astype(np.float64) - K[3]) / K[1]
        assert (1 + dist[0] * (x * x + y * y) < 0).sum() > 10                 # the early exit is taken for real keys
        cs_p, ci_p = O.port_assign_grid(p["keys_un"], p["bounds"])
        cs_r, ci_r = O.ref_assign_grid(r["keys_un"], r["bounds"])
        assert np.array_equal(cs_p, cs_r) and np.array_equal(ci_p, ci_r) and cs_r[-1] < len(keys)


@pytest.mark.parametrize("factor", fic.DEPTH_FACTORS)
def test_rgbd_edge_depths_port_equals_reference(O, factor):
    """ComputeStereoFromRGBD on depths that are 0, negative, NaN, +-inf or subnormal (only d > 0 is a measurement: NaN fails the
    test, a positive subnormal passes and gives a huge or infinite disparity), and on the raw 16-bit path with 65535 and the
    TUM / ICL / metre factors."""
    E = O.PortExtractor(1500)
    keys, _ = E(synth.mono_frame(13, 0, 0, 640, 480))
    K4 = np.array(fic.TUM1_K, np.float32); D = np.array(fic.DIST_CASES["tum1_5"][1], np.float32)
    for depth in (fic.edge_depth_float(int(factor * 1e4)), O.port_depth_to_float(fic.edge_depth_raw(7), factor)):
        assert fic.keys_on_depth_specials(keys, depth) > 50
        p = O.port_rgbd_frame(keys, K4, D, 40.0, depth)
        r = O.ref_rgbd_frame(keys, K4, D, 40.0, depth)
        for f in ("keys_un", "u_right", "depth", "bounds"):
            assert _bits(p[f]) == _bits(r[f]), f
        assert p["count"] == r["count"]
        d = depth[keys["y"].astype(int), keys["x"].astype(int)]
        assert np.array_equal(p["depth"] > 0, d > 0)                      # NaN, 0, -0, negatives and -inf are holes
    raw = fic.edge_depth_raw(7)
    assert np.array_equal(O.port_depth_to_float(raw, factor), raw.astype(np.float32) * np.float32(factor))
