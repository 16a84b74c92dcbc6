"""GPU: the CUDA matcher equals the port on the descriptor-distance gate cases of tests/match_gates.py — match arrays, counts and
states exactly — through the single entry points on host views and on resident frames, and with every case of a method in one
batched call next to an empty job."""
import dataclasses

import numpy as np
import pytest

from tests import match_gates as MG
from tests import proj_geometry as G

pytestmark = pytest.mark.gpu

CASES = MG.cases()


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def mt(M):
    m = M.ORBmatcher(0.8, False)
    yield m
    m.close()


def _set(mt, ratio=0.8):
    mt.mfNNratio = float(np.float32(ratio))
    mt.mbCheckOrientation = False


def _cur(c):
    F = c["F"]
    return G.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds)


RESIDENT = ("local", "last", "kf", "sim3proj", "fuse", "fuse_kf", "sim3", "proj")


def run_gpu(mt, c, method, resident):
    """One method of case c on the CUDA library, in the form of match_gates.run_port's result."""
    _set(mt, c.get("ratio", 0.8))
    F = c["F"].make_resident(mt) if resident else c.get("F")
    if method == "local":
        r = mt.SearchLocalPoints(F, c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], has_obs=c["has_obs"], viewingCosLimit=c["vcl"])
        return r, r["nmatches"], r["match"]
    if method == "last":
        Cur = _cur(c).make_resident(mt) if resident else _cur(c)
        return mt.SearchByProjectionLast(Cur, G.last_view(c), c["Tcw"], c["K"], c["bf"], c["th"], False, False)
    if method == "kf":
        return mt.SearchByProjectionKF(F, c["P"], c["Tcw"], c["Ow"], c["K"], c["th"], c["orb_dist"])
    if method == "sim3proj":
        return mt.SearchByProjectionSim3(F, c["P"], c["Tcw"], c["Ow"], c["K"], int(c["th"]))
    if method in ("fuse", "fuse_kf"):
        T = G.scw(c) if method == "fuse" else c["Tcw"]
        return mt.Fuse(F, c["P"], T, c["Ow"], c["K"], c["bf"], c["th"], Scw=method == "fuse")
    if method == "sim3":
        return mt.SearchBySim3(F, F, c["P"], c["P2"], c["Tcw"], c["Tcw"], MG.S12_ID, MG.S21_ID, c["K"], c["th"])
    if method == "proj":
        return mt.SearchByProjection(F, c["mps"], c["th"])
    if method == "bow0":
        return mt.SearchByBoW(c["kf"], c["F"])
    if method == "bow1":
        return mt.SearchByBoW_KF(c["kf"], c["F"])
    if method == "init":
        return mt.SearchForInitialization(c["F1"], c["F2"], c["prev"], c["window"])
    if method == "tri":
        return mt.SearchForTriangulation(c["kf1"], c["kf2"], c["F12"], c["ep"], False)
    raise ValueError(method)


def _equal(method, got, want):
    if method == "local":
        return G.frustum_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])
    if method == "tri":
        return np.array_equal(got, want)
    if method == "init":
        return got[0] == want[0] and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    return got[0] == want[0] and np.array_equal(got[1], want[1])


SINGLE = [(i, m, r) for i, c in enumerate(CASES) for m in MG.methods(c) for r in ((False, True) if m in RESIDENT else (False,))]


@pytest.mark.parametrize("i,method,resident", SINGLE,
                         ids=[f"{CASES[i]['cls']}-{CASES[i]['member']}-{m}-{'res' if r else 'host'}" for i, m, r in SINGLE])
def test_single_call_equals_port(mt, oracle, i, method, resident):
    c = CASES[i]
    want = MG.run_port(oracle, c, method)
    got = run_gpu(mt, c, method, resident)
    assert _equal(method, got, want), (c["cls"], c["member"], method, got, want)


def _by(method, key=lambda c: None):
    groups = {}
    for c in CASES:
        if method in MG.methods(c):
            groups.setdefault(key(c), []).append(c)
    return groups


def _empty_points(P):
    return dataclasses.replace(P, **{f: getattr(P, f)[:0] for f in ("world_pos", "descriptors", "max_distance", "min_distance", "normal",
                                                                      "angle", "valid")})


def _world():
    cs = _by("local")[None]
    return cs, [c["F"] for c in cs]


def test_local_points_batch(mt, oracle):
    """borb_search_local_points_batch: every world-point case in one call, next to a job without points."""
    _set(mt)
    cs, Fs = _world()
    got = mt.SearchLocalPointsBatch([F.make_resident(mt) for F in Fs + Fs[:1]], [c["P"] for c in cs] + [_empty_points(cs[0]["P"])],
                                    [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]], G.K_CAM, G.BF, [c["th"] for c in cs + cs[:1]],
                                    has_obs=[c["has_obs"] for c in cs] + [np.zeros(0, np.uint8)], viewingCosLimit=cs[0]["vcl"])
    for j, c in enumerate(cs):
        assert _equal("local", (got[j], got[j]["nmatches"], got[j]["match"]), MG.run_port(oracle, c, "local")), (c["cls"], c["member"])
    assert got[-1]["nmatches"] == 0 and len(got[-1]["match"]) == 0


def test_projection_batch(M, mt, oracle):
    """borb_search_by_projection_batch: every SearchByProjection(F, vpMapPoints) case of one nnratio in one call, next to a job
    without map points."""
    for ratio, cs in _by("proj", lambda c: c["ratio"]).items():
        _set(mt, ratio)
        m0 = cs[0]["mps"]
        empty = M.MapPointsView(*[getattr(m0, f.name)[:0] for f in dataclasses.fields(m0)])
        got = mt.SearchByProjectionBatch([c["F"].make_resident(mt) for c in cs + cs[:1]], [c["mps"] for c in cs] + [empty], cs[0]["th"])
        for j, c in enumerate(cs):
            assert _equal("proj", got[j], MG.run_port(oracle, c, "proj")), (c["cls"], c["member"])
        assert got[-1][0] == 0 and len(got[-1][1]) == 0


def test_last_frame_batch(M, mt, oracle):
    """borb_search_by_projection_last_batch: every world-point case in one call, next to a LastFrame without points."""
    _set(mt)
    cs, _ = _world()
    L0 = G.last_view(cs[0])
    empty = M.LastFrameView(L0.mvKeysUn[:0], L0.world_pos[:0], L0.descriptors[:0], L0.valid[:0], L0.has_obs[:0])
    got = mt.SearchByProjectionLastBatch([_cur(c).make_resident(mt) for c in cs + cs[:1]], [G.last_view(c) for c in cs] + [empty],
                                         [c["Tcw"] for c in cs + cs[:1]], G.K_CAM, G.BF, [c["th"] for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("last", got[j], MG.run_port(oracle, c, "last")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_keyframe_projection_batch(mt, oracle):
    """borb_search_by_projection_kf_batch: every world-point case in one call, each with its own ORBdist (64 or 100), next to a
    keyframe without points."""
    _set(mt)
    cs, Fs = _world()
    assert {c["orb_dist"] for c in cs} == {64, 100}
    got = mt.SearchByProjectionKFBatch([F.make_resident(mt) for F in Fs + Fs[:1]], [c["P"] for c in cs] + [_empty_points(cs[0]["P"])],
                                       [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]], G.K_CAM, [c["th"] for c in cs + cs[:1]],
                                       [c["orb_dist"] for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("kf", got[j], MG.run_port(oracle, c, "kf")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_sim3_projection_batch(mt, oracle):
    """borb_search_by_projection_sim3_batch: every world-point case in one call, next to a job without points."""
    _set(mt)
    cs, Fs = _world()
    got = mt.SearchByProjectionSim3Batch([F.make_resident(mt) for F in Fs + Fs[:1]], [c["P"] for c in cs] + [_empty_points(cs[0]["P"])],
                                         [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]], G.K_CAM, [int(c["th"]) for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("sim3proj", got[j], MG.run_port(oracle, c, "sim3proj")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_sim3_batch(mt, oracle):
    """borb_search_by_sim3_batch: every world-point case, with its own MapPoints for each keyframe, in one call, next to a
    keyframe pair without MapPoints."""
    _set(mt)
    cs, Fs = _world()
    none = lambda P: dataclasses.replace(P, valid=np.zeros(len(P.world_pos), np.uint8))
    kfs = [F.make_resident(mt) for F in Fs + Fs[:1]]
    got = mt.SearchBySim3Batch(kfs, kfs, [c["P"] for c in cs] + [none(cs[0]["P"])], [c["P2"] for c in cs] + [none(cs[0]["P2"])],
                               [(c["Tcw"], c["Tcw"]) for c in cs + cs[:1]], [(MG.S12_ID, MG.S21_ID)] * (len(cs) + 1), G.K_CAM,
                               [c["th"] for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("sim3", got[j], MG.run_port(oracle, c, "sim3")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


@pytest.mark.parametrize("scw", [False, True])
def test_fuse_batch(mt, oracle, scw):
    """borb_fuse_batch: every world-point case of one overload in one call, next to a job without points."""
    method = "fuse" if scw else "fuse_kf"
    cs, Fs = _world()
    poses = [(G.scw(c) if scw else c["Tcw"], c["Ow"]) for c in cs + cs[:1]]
    got = mt.FuseBatch([F.make_resident(mt) for F in Fs + Fs[:1]], [c["P"] for c in cs] + [_empty_points(cs[0]["P"])], poses, G.K_CAM,
                       G.BF, [c["th"] for c in cs + cs[:1]], Scw=scw)
    for j, c in enumerate(cs):
        assert _equal(method, got[j], MG.run_port(oracle, c, method)), (c["cls"], c["member"])
    assert got[-1][0] == 0 and len(got[-1][1]) == 0


def test_bow_batch(M, mt, oracle):
    """borb_search_by_bow_batch: every SearchByBoW(KF, F) case of one nnratio in one call, next to a keyframe with an empty
    FeatureVector.  The frames are resident with their BoW from ComputeBoWBatch at levelsup = L, which puts every feature in
    node 0, as the cases' host FeatureVectors do."""
    pv = oracle.PortVocabulary.random(10, 2, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    for ratio, cs in _by("bow0", lambda c: c["ratio"]).items():
        _set(mt, ratio)
        Fs = [M.FrameView(c["F"].mvKeysUn, c["F"].mDescriptors, G.SCALE, G.BOUNDS).make_resident(mt) for c in cs + cs[:1]]
        bows = mt.ComputeBoWBatch(voc, Fs, int(e["L"]))
        for (_, fv), c in zip(bows, cs):
            assert np.array_equal(fv.node_id, c["F"].mFeatVec.node_id) and np.array_equal(fv.start, c["F"].mFeatVec.start)
            assert np.array_equal(fv.feat_idx, c["F"].mFeatVec.feat_idx)
        kf0 = cs[0]["kf"]
        empty = M.KeyFrameView(kf0.mvKeysUn, kf0.mDescriptors, M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32),
                                                                                np.zeros(0, np.uint32)), has_mp=kf0.has_mp)
        got = mt.SearchByBoWBatch([c["kf"] for c in cs] + [empty], Fs)
        for j, c in enumerate(cs):
            assert _equal("bow0", got[j], MG.run_port(oracle, c, "bow0")), (c["cls"], c["member"])
        assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_initialization_batch(mt, oracle):
    """borb_search_for_initialization_batch: every SearchForInitialization case of one nnratio in one call on resident frames,
    next to a job whose windows hold no F2 feature."""
    for ratio, cs in _by("init", lambda c: c["ratio"]).items():
        _set(mt, ratio)
        F1s = [c["F1"].make_resident(mt) for c in cs + cs[:1]]
        F2s = [c["F2"].make_resident(mt) for c in cs + cs[:1]]
        away = np.full_like(cs[0]["prev"], 500.0)
        got = mt.SearchForInitializationBatch(F1s, F2s, [c["prev"] for c in cs] + [away], MG.INIT_WINDOW)
        for j, c in enumerate(cs):
            assert _equal("init", got[j], MG.run_port(oracle, c, "init")), (c["cls"], c["member"])
        assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_triangulation_batch(mt, oracle):
    """borb_search_for_triangulation_batch: every SearchForTriangulation case in one call, next to a job whose keyframe features
    all have MapPoints (nothing to triangulate)."""
    _set(mt)
    cs = _by("tri")[None]
    full = dataclasses.replace(cs[0]["kf1"], has_mp=np.ones(len(cs[0]["kf1"].mvKeysUn), np.uint8), _keep=[])
    got = mt.SearchForTriangulationBatch([c["kf1"] for c in cs] + [full], [c["kf2"] for c in cs + cs[:1]],
                                         [c["F12"] for c in cs + cs[:1]], [c["ep"] for c in cs + cs[:1]])
    for j, c in enumerate(cs):
        assert _equal("tri", got[j], MG.run_port(oracle, c, "tri")), (c["cls"], c["member"])
    assert len(got[-1]) == 0
