"""GPU: the CUDA matcher equals the port on the float decision-boundary cases of tests/proj_geometry.py — match arrays, counts and
states exactly; isInFrustum's track fields bit for bit, except that any NaN equals any NaN — on host views and on resident
frames, and with every case of a method in one batched call next to an empty job."""
import dataclasses

import numpy as np
import pytest

from tests import proj_geometry as G

pytestmark = pytest.mark.gpu

CASES = G.cases()


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def mt(M):
    m = M.ORBmatcher(0.8, False)
    yield m
    m.close()


def _set(mt, ratio=0.8, ori=False):
    mt.mfNNratio = float(np.float32(ratio))
    mt.mbCheckOrientation = bool(ori)


def _cur(c):
    F = c["F"]
    return G.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds)


def run_gpu(mt, c, method, resident):
    """One method of case c on the CUDA library, in the form of proj_geometry.run_port's result."""
    _set(mt, ori=c.get("ori", False))
    F = c["F"].make_resident(mt) if resident and "F" in c else c.get("F")
    if method == "local":
        r = mt.SearchLocalPoints(F, c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], has_obs=c["has_obs"], viewingCosLimit=c["vcl"])
        return r, r["nmatches"], r["match"]
    if method == "last":
        Cur = _cur(c).make_resident(mt) if resident else _cur(c)
        return mt.SearchByProjectionLast(Cur, G.last_view(c), c["Tcw"], c["K"], c["bf"], c["th"], c.get("fwd", False), c.get("bwd", False))
    if method == "kf":
        return mt.SearchByProjectionKF(F, c["P"], c["Tcw"], c["Ow"], c["K"], c["th"], 100)
    if method == "sim3proj":
        return mt.SearchByProjectionSim3(F, c["P"], c["Tcw"], c["Ow"], c["K"], int(c["th"]))
    if method in ("fuse", "fuse_kf"):
        T = G.scw(c) if method == "fuse" else c["Tcw"]
        return mt.Fuse(F, c["P"], T, c["Ow"], c["K"], c["bf"], c["th"], Scw=method == "fuse")
    if method == "sim3" and "kind" in c:
        KF1, KF2 = (c["KF1"].make_resident(mt), c["KF2"].make_resident(mt)) if resident else (c["KF1"], c["KF2"])
        return mt.SearchBySim3(KF1, KF2, c["P1"], c["P2"], c["T1w"], c["T2w"], c["S12"], c["S21"], c["K"], c["th"])
    if method == "sim3":
        _, _, P1, P2, T1, T2, S12, S21, K, th = G.sim3_args(c)
        return mt.SearchBySim3(F, F, P1, P2, T1, T2, S12, S21, K, th)
    if method == "proj":
        _set(mt, c["ratio"], c.get("ori", False))
        return mt.SearchByProjection(F, c["mps"], c["th"])
    if method == "tri":
        return mt.SearchForTriangulation(c["kf1"], c["kf2"], c["F12"], c["ep"], c["only_stereo"])
    raise ValueError(method)


def _equal(method, got, want):
    if method == "local":
        return G.frustum_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])
    if method == "tri":
        return np.array_equal(got, want)
    return got[0] == want[0] and np.array_equal(got[1], want[1])


SINGLE = [(i, m, r) for i, c in enumerate(CASES) for m in G.methods(c) for r in ((False, True) if m != "tri" else (False,))]


@pytest.mark.parametrize("i,method,resident", SINGLE,
                         ids=[f"{CASES[i]['cls']}-{CASES[i]['member']}-{m}-{'res' if r else 'host'}" for i, m, r in SINGLE])
def test_single_call_equals_port(mt, oracle, i, method, resident):
    c = CASES[i]
    want = G.run_port(oracle, c, method)
    got = run_gpu(mt, c, method, resident)
    assert _equal(method, got, want), (c["cls"], c["member"], method, got, want)


def test_camera_centre_point_is_in_view_with_nan_track_fields(mt, oracle):
    """A point at the camera centre with mfMinDistance == 0 is in view (IncreaseVisible runs on it), its track fields are NaN,
    its level 0, and it gets no match; the smallest positive mfMinDistance takes it out of view."""
    for c in CASES:
        if c["cls"] != "camera_centre":
            continue
        r = run_gpu(mt, c, "local", False)[0]
        assert r["in_view"][0] == (1 if c["member"] == 0 else 0)
        if c["member"] == 0:
            assert r["level"][0] == 0 and all(np.isnan(r[f][0]) for f in G.FLOAT_FIELDS)
        assert r["match"][0] == -1 and (r["match"][1:] >= 0).all()


def _by(method, key=lambda c: None):
    groups = {}
    for c in CASES:
        if method in G.methods(c):
            groups.setdefault(key(c), []).append(c)
    return groups


def _empty_points(P):
    return dataclasses.replace(P, **{f: getattr(P, f)[:0] for f in ("world_pos", "descriptors", "max_distance", "min_distance", "normal",
                                                                      "angle", "valid")})


def test_local_points_batch(mt, oracle):
    """borb_search_local_points_batch: every SearchLocalPoints case of one viewing-cosine limit in one call, next to an empty job."""
    _set(mt)
    for vcl, cs in _by("local", lambda c: c["vcl"]).items():
        frames = [c["F"].make_resident(mt) for c in cs] + [cs[0]["F"].make_resident(mt)]
        points = [c["P"] for c in cs] + [_empty_points(cs[0]["P"])]
        poses = [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]]
        got = mt.SearchLocalPointsBatch(frames, points, poses, G.K_CAM, G.BF, [c["th"] for c in cs + cs[:1]],
                                        has_obs=[c["has_obs"] for c in cs] + [np.zeros(0, np.uint8)], viewingCosLimit=vcl)
        for j, c in enumerate(cs):
            assert _equal("local", (got[j], got[j]["nmatches"], got[j]["match"]), G.run_port(oracle, c, "local")), (c["cls"], c["member"])
        assert got[-1]["nmatches"] == 0 and len(got[-1]["match"]) == 0


def test_projection_batch(M, mt, oracle):
    """borb_search_by_projection_batch: every SearchByProjection case of one th in one call, next to a job without map points."""
    _set(mt)
    for th, cs in _by("proj", lambda c: c["th"]).items():
        frames = [c["F"].make_resident(mt) for c in cs] + [cs[0]["F"].make_resident(mt)]
        m0 = cs[0]["mps"]
        empty = M.MapPointsView(*[getattr(m0, f.name)[:0] for f in dataclasses.fields(m0)])
        got = mt.SearchByProjectionBatch(frames, [c["mps"] for c in cs] + [empty], th)
        for j, c in enumerate(cs):
            assert _equal("proj", got[j], G.run_port(oracle, c, "proj")), (c["cls"], c["member"])
        assert got[-1][0] == 0 and len(got[-1][1]) == 0


def test_last_frame_batch(M, mt, oracle):
    """borb_search_by_projection_last_batch: every LastFrame case in one call, each with its own forward / backward flags (the
    three modes mixed), next to a LastFrame without points."""
    groups = _by("last", lambda c: c.get("ori", False))
    assert sorted(groups) == [False, True]
    assert {(c.get("fwd", False), c.get("bwd", False)) for c in groups[False]} == {(True, False), (False, True), (False, False)}
    for ori, cs in groups.items():
        _last_frame_batch(M, mt, oracle, cs, ori)


def _last_frame_batch(M, mt, oracle, cs, ori):
    _set(mt, ori=ori)
    L0 = G.last_view(cs[0])
    empty = M.LastFrameView(L0.mvKeysUn[:0], L0.world_pos[:0], L0.descriptors[:0], L0.valid[:0], L0.has_obs[:0])
    curs = [_cur(c).make_resident(mt) for c in cs + cs[:1]]
    got = mt.SearchByProjectionLastBatch(curs, [G.last_view(c) for c in cs] + [empty], [c["Tcw"] for c in cs + cs[:1]], G.K_CAM, G.BF,
                                         [c["th"] for c in cs + cs[:1]], forward=[c.get("fwd", False) for c in cs + cs[:1]],
                                         backward=[c.get("bwd", False) for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("last", got[j], G.run_port(oracle, c, "last")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_keyframe_projection_batch(mt, oracle):
    """borb_search_by_projection_kf_batch: every SearchByProjection(CurrentFrame, KeyFrame) case in one call, next to a keyframe
    without points."""
    for ori, cs in _by("kf", lambda c: c.get("ori", False)).items():
        _set(mt, ori=ori)
        curs = [c["F"].make_resident(mt) for c in cs + cs[:1]]
        points = [c["P"] for c in cs] + [_empty_points(cs[0]["P"])]
        got = mt.SearchByProjectionKFBatch(curs, points, [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]], G.K_CAM, [c["th"] for c in cs + cs[:1]],
                                           100)
        for j, c in enumerate(cs):
            assert _equal("kf", got[j], G.run_port(oracle, c, "kf")), (c["cls"], c["member"])
        assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_sim3_projection_batch(mt, oracle):
    """borb_search_by_projection_sim3_batch: every SearchByProjection(pKF, Scw) case in one call, next to a job without points."""
    _set(mt)
    cs = _by("sim3proj")[None]
    kfs = [c["F"].make_resident(mt) for c in cs + cs[:1]]
    points = [c["P"] for c in cs] + [_empty_points(cs[0]["P"])]
    got = mt.SearchByProjectionSim3Batch(kfs, points, [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]], G.K_CAM, [int(c["th"]) for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("sim3proj", got[j], G.run_port(oracle, c, "sim3proj")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_sim3_batch(mt, oracle):
    """borb_search_by_sim3_batch: every SearchBySim3 case — the identity Sim3 of the world-point cases and the scaled, rotated
    similarities of the sim3_* cases — in one call, next to a keyframe pair without MapPoints."""
    _set(mt)
    cs = _by("sim3")[None]
    assert any("kind" in c for c in cs) and any("kind" not in c for c in cs)

    def job(c):
        if "kind" in c:
            return c["KF1"], c["KF2"], c["P1"], c["P2"], (c["T1w"], c["T2w"]), (c["S12"], c["S21"]), c["th"]
        F, _, P1, P2, T1, T2, S12, S21, _, th = G.sim3_args(c)
        return F, F, P1, P2, (T1, T2), (S12, S21), th
    jobs = [job(c) for c in cs]
    none = lambda P: dataclasses.replace(P, valid=np.zeros(len(P.world_pos), np.uint8))
    e = jobs[0]
    jobs.append((e[0], e[1], none(e[2]), none(e[3]), e[4], e[5], e[6]))
    got = mt.SearchBySim3Batch([j[0].make_resident(mt) for j in jobs], [j[1].make_resident(mt) for j in jobs], [j[2] for j in jobs],
                               [j[3] for j in jobs], [j[4] for j in jobs], [j[5] for j in jobs], G.K_CAM, [j[6] for j in jobs])
    for j, c in enumerate(cs):
        assert _equal("sim3", got[j], G.run_port(oracle, c, "sim3")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


@pytest.mark.parametrize("scw", [False, True])
def test_fuse_batch(mt, oracle, scw):
    """borb_fuse_batch: every Fuse case of one overload in one call, next to a job without points."""
    method = "fuse" if scw else "fuse_kf"
    cs = _by(method)[None]
    kfs = [c["F"].make_resident(mt) for c in cs + cs[:1]]
    points = [c["P"] for c in cs] + [_empty_points(cs[0]["P"])]
    poses = [(G.scw(c) if scw else c["Tcw"], c["Ow"]) for c in cs + cs[:1]]
    got = mt.FuseBatch(kfs, points, poses, G.K_CAM, G.BF, [c["th"] for c in cs + cs[:1]], Scw=scw)
    for j, c in enumerate(cs):
        assert _equal(method, got[j], G.run_port(oracle, c, method)), (c["cls"], c["member"])
    assert got[-1][0] == 0 and len(got[-1][1]) == 0


def test_triangulation_batch(mt, oracle):
    """borb_search_for_triangulation_batch: every SearchForTriangulation case in one call, next to a job whose keyframe features
    all have MapPoints (nothing to triangulate)."""
    for ori, cs in _by("tri", lambda c: c["ori"]).items():
        _set(mt, ori=ori)
        full = dataclasses.replace(cs[0]["kf1"], has_mp=np.ones(len(cs[0]["kf1"].mvKeysUn), np.uint8), _keep=[])
        kf1s = [c["kf1"] for c in cs] + [full]
        kf2s = [c["kf2"] for c in cs + cs[:1]]
        got = mt.SearchForTriangulationBatch(kf1s, kf2s, [c["F12"] for c in cs + cs[:1]], [c["ep"] for c in cs + cs[:1]])
        for j, c in enumerate(cs):
            assert _equal("tri", got[j], G.run_port(oracle, c, "tri")), (c["cls"], c["member"])
        assert len(got[-1]) == 0


@pytest.mark.parametrize("cls", G.dense_classes())
def test_dense_variants_equal_port(mt, oracle, cls):
    """Both members of every world-point class inside a natural ~1000-point call (proj_geometry.dense_case), every method, on
    host views and on resident frames."""
    for c in G.cases():
        if c["cls"] != cls or "kind" in c:
            continue
        d = G.dense_case(oracle, c)
        for method in G.methods(d):
            want = G.run_port(oracle, d, method)
            for resident in (False, True):
                assert _equal(method, run_gpu(mt, d, method, resident), want), (cls, c["member"], method, resident)
