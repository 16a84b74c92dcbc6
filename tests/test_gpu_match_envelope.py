"""GPU: the CUDA matcher equals the port bit for bit (counts, match arrays, states, pairs) on the size-envelope cases of
tests/match_envelope.py, on host views and on device-resident frames, alone and in batches next to small and empty jobs, and
refuses one feature or one query beyond MATCH_MAX_FEATURES without losing the handle.

One matcher handle serves the whole module: at 8192 x 8192 its arena holds a 256 MB candidate buffer, and it is released
when the module ends."""
import dataclasses

import numpy as np
import pytest

from tests import match_envelope as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def mt(M):
    m = M.ORBmatcher(0.8, True)
    yield m
    m.close()


def _set(mt, ratio, ori):
    mt.mfNNratio = float(np.float32(ratio))
    mt.mbCheckOrientation = bool(ori)


def run_gpu(mt, c, resident):
    """The case on the CUDA library, in the form of match_envelope.run_port's result."""
    m = c["method"]
    if m == "proj":
        _set(mt, c["ratio"], True)
        F = c["F"].make_resident(mt) if resident else c["F"]
        return mt.SearchByProjection(F, c["mps"], c["th"])
    if m == "last":
        _set(mt, 0.8, c["ori"])
        F = c["F"].make_resident(mt) if resident else c["F"]
        return mt.SearchByProjectionLast(F, c["Last"], c["Tcw"], c["K"], 40.0, c["th"])
    if m == "local":
        _set(mt, c["ratio"], True)
        F = c["F"].make_resident(mt) if resident else c["F"]
        r = mt.SearchLocalPoints(F, c["P"], c["Tcw"], c["Ow"], c["K"], 40.0, c["th"], has_obs=c["has_obs"])
        return r["nmatches"], r["match"]
    if m == "bow":
        _set(mt, c["ratio"], c["ori"])
        return mt.SearchByBoW(c["kf1"], c["kf2"]), mt.SearchByBoW_KF(c["kf1"], c["kf2"])
    if m == "tri":
        _set(mt, 0.6, c["ori"])
        return mt.SearchForTriangulation(c["kf1"], c["kf2"], c["F12"], c["ep"], c["only_stereo"])
    if m == "init":
        _set(mt, c["ratio"], c["ori"])
        return mt.SearchForInitialization(c["F1"], c["F2"], c["prev"], c["window"])          # (n, vnMatches12, vbPrevMatched)
    if m == "fuse":
        _set(mt, 0.6, True)
        return (mt.Fuse(c["KF"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], Scw=False),
                mt.Fuse(c["KF"], c["P"], c["Ts"], c["Ows"], c["K"], c["bf"], c["th"], Scw=True))
    if m == "sim3":
        _set(mt, 0.75, True)
        return mt.SearchBySim3(c["KF1"], c["KF2"], c["P1"], c["P2"], c["T1w"], c["T2w"], c["S12"], c["S21"], c["K"], c["th"])
    raise ValueError(m)


def _same(a, b):
    """Results equal element by element: counts, index arrays, nested (first search, second search) tuples."""
    if isinstance(a, tuple):
        return isinstance(b, tuple) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return np.array_equal(a, b)
    return a == b


RESIDENT = ("self", "proj", "contested", "hist", "local", "tied_proj", "tied_last", "tied_local", "extract")
SINGLE = [(n, False) for n in E.NAMES] + [(n, True) for n in E.NAMES if n.startswith(RESIDENT)]


@pytest.mark.parametrize("name,resident", SINGLE)
def test_single_call_equals_port(mt, oracle, name, resident):
    """Host views, and resident frames for the projection searches.  The resident hist_* calls stage fewer than 96 KB of inputs
    (read in place from pinned memory), the resident 8192-feature calls far more (copied to the device first)."""
    c = E.case(oracle, name)
    want = E.run_port(oracle, c)
    got = run_gpu(mt, c, resident)
    assert _same(got, want), name


def _empty_mps(M, mps):
    z = slice(0, 0)
    return M.MapPointsView(mps.mTrackProjX[z], mps.mTrackProjY[z], mps.mTrackProjXR[z], mps.mnTrackScaleLevel[z], mps.mTrackViewCos[z],
                           mps.descriptors[z], mps.valid[z], mps.has_obs[z])


def test_projection_batch_with_an_envelope_job(M, mt, oracle):
    """borb_search_by_projection_batch: the 8192 x 8192 job sets the block size and shared memory of the launch; the small,
    contested and empty jobs next to it must give their single-call results."""
    names = ["self_kitti_8192", "tied_proj", "contested_sorted_mixed", None]
    frames, lists, want = [], [], []
    for nm in names:
        c = E.case(oracle, nm or "tied_proj")
        mps = c["mps"] if nm else _empty_mps(M, c["mps"])
        frames.append(c["F"].make_resident(mt)); lists.append(mps)
        want.append(oracle.port_search_by_projection(c["F"], mps, 3.0, 0.8) if nm else (0, np.zeros(0, np.int32)))
    _set(mt, 0.8, True)
    got = mt.SearchByProjectionBatch(frames, lists, 3.0)
    for j, (g, w) in enumerate(zip(got, want)):
        assert _same(g, w), names[j]
    assert got[0][0] > 8000


def test_last_frame_batch_with_an_envelope_job(M, mt, oracle):
    """borb_search_by_projection_last_batch: a contested 2500-query job over three waves next to a histogram-boundary job and
    a job without LastFrame points."""
    cases = [E.case(oracle, "contested_unsorted_last"), E.case(oracle, "hist_max2_tenth"), E.case(oracle, "contested_sorted_last")]
    empty = dataclasses.replace(cases[1]["Last"], mvKeysUn=cases[1]["Last"].mvKeysUn[:0], world_pos=cases[1]["Last"].world_pos[:0],
                                descriptors=cases[1]["Last"].descriptors[:0], valid=cases[1]["Last"].valid[:0],
                                has_obs=cases[1]["Last"].has_obs[:0])
    curs = [c["F"].make_resident(mt) for c in cases] + [cases[1]["F"].make_resident(mt)]
    lasts = [c["Last"] for c in cases] + [empty]
    ths = [c["th"] for c in cases] + [3.0]
    _set(mt, 0.8, True)
    got = mt.SearchByProjectionLastBatch(curs, lasts, [c["Tcw"] for c in cases] + [cases[0]["Tcw"]], E.K_CAM, 40.0, ths)
    for j, c in enumerate(cases):
        want = oracle.port_search_by_projection_last(c["F"], c["Last"], c["Tcw"], c["K"], 40.0, c["th"], False, False, True)
        assert _same(got[j], want), j
    assert got[3][0] == 0 and np.all(got[3][1] == -1)


def _refused(call):
    from orb_slam2_b200._lib import BorbError
    with pytest.raises(BorbError) as e:
        call()
    assert e.value.status == 1, str(e.value)                        # BORB_ERR_INVALID_ARG


def test_refusals_leave_the_handle_working(M, mt, oracle):
    """One feature, query, LastFrame point, keyframe feature or local map point beyond MATCH_MAX_FEATURES is refused with
    BORB_ERR_INVALID_ARG, each with everything else inside the limit; the same handle then still matches 8192 x 8192."""
    v = E.envelope_views(oracle, E.KITTI, n=E.MATCH_MAX_FEATURES + 1)
    F, mps = E.self_query(v)
    c = E.case(oracle, "self_kitti_8192")
    F8, mps8 = c["F"], c["mps"]
    few = dataclasses.replace(mps8, **{f: getattr(mps8, f)[:100] for f in ("mTrackProjX", "mTrackProjY", "mTrackProjXR", "mnTrackScaleLevel",
                                                                           "mTrackViewCos", "descriptors", "valid", "has_obs")})
    _set(mt, 0.8, True)
    _refused(lambda: mt.SearchByProjection(F, few, 3.0))                           # 8193 features, 100 queries
    _refused(lambda: mt.SearchByProjection(F8, mps, 3.0))                          # 8192 features, 8193 queries
    _refused(lambda: F.make_resident(mt))                                          # a resident frame of 8193 features
    n1 = E.MATCH_MAX_FEATURES + 1
    Last = M.LastFrameView(v["kr"], np.tile(np.float32([0.1, 0.1, 5.0]), (n1, 1)), v["dr"], np.ones(n1, np.uint8), np.ones(n1, np.uint8))
    _refused(lambda: mt.SearchByProjectionLast(F8, Last, np.eye(4, dtype=np.float32)[:3], E.K_CAM, 40.0, 15.0))   # 8193 LastFrame points
    ci = E.case(oracle, "init_kitti_8192")
    F1 = M.FrameView(v["kl"], v["dl"], v["scale"], ci["F1"].bounds)
    _refused(lambda: mt.SearchForInitialization(F1, ci["F2"], np.zeros((n1, 2), np.float32), 100))          # 8193 features in F1
    ct = E.case(oracle, "tri_one_node_8192")
    kf = M.KeyFrameView(v["kl"], v["dl"], M.FeatureVector.from_nodes(np.zeros(n1, np.int64)), has_mp=np.zeros(n1, np.uint8),
                        mvScaleFactors=v["scale"], mvLevelSigma2=v["sigma2"])
    _refused(lambda: mt.SearchForTriangulation(kf, ct["kf2"], ct["F12"], ct["ep"]))                         # 8193 keyframe features
    cl = E.case(oracle, "local_kitti_8192")
    P = cl["P"]
    P9 = dataclasses.replace(P, **{f: np.concatenate([getattr(P, f), getattr(P, f)[:1]]) for f in ("world_pos", "descriptors", "max_distance",
                                                                                                     "min_distance", "normal", "angle")},
                             valid=np.ones(n1, np.uint8))
    _refused(lambda: mt.SearchLocalPoints(cl["F"], P9, cl["Tcw"], cl["Ow"], cl["K"], 40.0, 3.0))            # 8193 valid local map points
    assert _same(run_gpu(mt, c, False), E.run_port(oracle, c))
    assert _same(run_gpu(mt, c, True), E.run_port(oracle, c))
    assert _same(run_gpu(mt, cl, False), E.run_port(oracle, cl))


def test_resident_frame_capacities(mt, oracle):
    """borb_frame_create rounds a frame's capacity (2048, then multiples of 1024) and reuses released frames of at least the
    size asked for: frames just below, at and above each rounding step, in an order that reuses the larger blocks."""
    v = E.envelope_views(oracle, E.EUROC)
    _set(mt, 0.8, True)
    for n in (8192, 2047, 2049, 3073, 2048, 8191, 3072, 1):
        vn = dict(v, kl=v["kl"][:n], dl=v["dl"][:n], ur=v["ur"][:n])
        F, mps = E.self_query(vn)
        FR = F.make_resident(mt)
        assert _same(mt.SearchByProjection(FR, mps, 3.0), oracle.port_search_by_projection(F, mps, 3.0, 0.8)), n
        FR.resident.close()


def test_frames_from_extractor_at_the_envelope(M, mt, oracle):
    """borb_frames_from_extractor builds resident frames (and their grids, with grid_sort_jobs_kernel) from a GPU extraction:
    the first 8192 keypoints of a KITTI frame without distortion (every key in the grid, the sort's last slot a real key — the
    extract_kitti_8192 case) and all keypoints of a TUM-sized frame with TUM distortion.  A count beyond MATCH_MAX_FEATURES is
    refused."""
    from orb_slam2_b200 import synth
    from orb_slam2_b200.extractor import ORBextractor
    c = E.case(oracle, "extract_kitti_8192")
    TUM_K, TUM_DIST = (517.306408, 516.469215, 318.643040, 255.313989), (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)
    _set(mt, 0.8, True)
    for img, image, K, dist in ((0, synth.stereo_pair(9, 0, 0, *E.KITTI)[0], E.K_CAM, (0, 0, 0, 0, 0)),
                                (1, synth.mono_frame(5, 0, 0, 640, 480), TUM_K, TUM_DIST)):
        X = ORBextractor(E.MATCH_MAX_FEATURES)
        outs = {img: X.extract_batch([image])[0]}
        if img == 0:
            assert len(outs[0][0]) > E.MATCH_MAX_FEATURES
            _refused(lambda: M.frames_from_extractor(mt, X, [0], [E.MATCH_MAX_FEATURES + 1], K))
        n = min(len(outs[img][0]), E.MATCH_MAX_FEATURES)
        frames, host = M.frames_from_extractor(mt, X, [0], [n], K, dist)
        keys_un, b = host["keys_un"][0], tuple(float(x) for x in host["bounds"])
        desc = outs[img][1][:n]
        F, mps = E.self_query(dict(kl=keys_un, dl=desc, ur=np.full(n, -1, np.float32), scale=X.GetScaleFactors()), bounds=b)
        F = dataclasses.replace(F, mvuRight=None)
        FR = dataclasses.replace(frames[0], occupied=None)
        assert _same(mt.SearchByProjection(FR, mps, 3.0), oracle.port_search_by_projection(F, mps, 3.0, 0.8)), img
        if img == 0:
            assert np.array_equal(keys_un, c["F"].mvKeysUn) and np.array_equal(desc, c["F"].mDescriptors)
            assert E.in_grid(keys_un, b).all() and n == E.MATCH_MAX_FEATURES
        frames[0].resident.close()


def _empty_points(P):
    return dataclasses.replace(P, **{f: getattr(P, f)[:0] for f in ("world_pos", "descriptors", "max_distance", "min_distance", "normal",
                                                                      "angle", "valid")})


def test_local_points_batch_with_an_envelope_job(M, mt, oracle):
    """borb_search_local_points_batch: an 8192-point job next to a tied 1000-point job and an empty one."""
    cases = [E.case(oracle, "local_kitti_8192"), E.case(oracle, "tied_local")]
    frames = [c["F"].make_resident(mt) for c in cases] + [cases[1]["F"].make_resident(mt)]
    points = [c["P"] for c in cases] + [_empty_points(cases[1]["P"])]
    _set(mt, 0.8, True)
    got = mt.SearchLocalPointsBatch(frames, points, [(c["Tcw"], c["Ow"]) for c in cases] + [(cases[1]["Tcw"], cases[1]["Ow"])],
                                    [c["K"] for c in cases] + [cases[1]["K"]], 40.0, 3.0,
                                    has_obs=[c["has_obs"] for c in cases] + [np.zeros(0, np.uint8)])
    for j, c in enumerate(cases):
        assert _same((got[j]["nmatches"], got[j]["match"]), E.run_port(oracle, c)), j
        fr = oracle.port_is_in_frustum(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], 40.0, 0.5)
        assert np.array_equal(got[j]["in_view"], fr["in_view"]), j
    assert got[2]["nmatches"] == 0 and len(got[2]["match"]) == 0


def test_bow_batch_with_wide_nodes(M, mt, oracle):
    """borb_search_by_bow_batch (bow_match_kernel with per-pair frames): a one-node 8192-feature job (direct evaluation), an
    8192-feature job of row chunks and a 1000-feature job, each equal to the port; the frames' BoW comes from ComputeBoWBatch."""
    pv = E._wide_voc(oracle)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    import tests.match_fixtures as mf
    small = mf.keyframe_views(mf.two_views(oracle, 7), pv, 3, levelsup=2)
    jobs = [(E.case(oracle, "bow_one_node_8192"), 3), (E.case(oracle, "bow_row_chunks_8192"), 2), (dict(kf1=small[0], kf2=small[1], ratio=0.8), 2)]
    kfs, frames = [], []
    for c, levelsup in jobs:
        kf2 = c["kf2"]
        FR = M.FrameView(kf2.mvKeysUn, kf2.mDescriptors, kf2.mvScaleFactors, (0.0, 0.0, 2000.0, 2000.0)).make_resident(mt)
        (_, fv), = mt.ComputeBoWBatch(voc, [FR], levelsup)
        assert np.array_equal(fv.node_id, kf2.mFeatVec.node_id) and np.array_equal(fv.feat_idx, kf2.mFeatVec.feat_idx)
        kfs.append(c["kf1"]); frames.append(FR)
    _set(mt, 0.8, True)
    got = mt.SearchByBoWBatch(kfs, frames)
    for j, (c, _) in enumerate(jobs):
        assert _same(got[j], oracle.port_search_by_bow(c["kf1"], c["kf2"], 0.8, True)), j
    assert got[0][0] > 1000
