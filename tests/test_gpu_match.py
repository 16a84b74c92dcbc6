"""GPU parity for the ORBmatcher paths and the BoW feeder through the C ABI, against the restatements in
oracle/orb_port_match.cpp: bit-exact indices and counts (all integer / order-dependent work)."""
import os

import numpy as np
import pytest

from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def views(oracle):
    return {s: mf.two_views(oracle, s) for s in (7, 8)}


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("th,ratio", [(1.0, 0.8), (3.0, 0.8), (5.0, 0.9)])
def test_search_by_projection(M, oracle, views, seed, th, ratio):
    F, mps = mf.projection_case(views[seed], seed + 10, n_mp=400)
    n_o, m_o = oracle.port_search_by_projection(F, mps, th, ratio)
    n_g, m_g = M.ORBmatcher(ratio, True).SearchByProjection(F, mps, th)
    assert n_o > 30
    assert n_g == n_o and np.array_equal(m_g, m_o), int((m_g != m_o).sum())


def test_search_by_projection_edge_cases(M, oracle, views):
    v = views[7]
    F, mps = mf.projection_case(v, 99, n_mp=50)
    mt = M.ORBmatcher(0.8, True)
    # monocular frame (no stereo check), no occupancy, all map points valid and observed
    F2 = M.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds)
    mp2 = M.MapPointsView(mps.mTrackProjX, mps.mTrackProjY, mps.mTrackProjXR, mps.mnTrackScaleLevel, mps.mTrackViewCos, mps.descriptors)
    assert_same = lambda a, b: (a[0] == b[0] and np.array_equal(a[1], b[1]))
    assert assert_same(mt.SearchByProjection(F2, mp2, 3.0), oracle.port_search_by_projection(F2, mp2, 3.0, 0.8))
    # every map point projects to the same place: the order-dependent claiming decides
    mp3 = M.MapPointsView(np.full(50, 320.0, np.float32), np.full(50, 240.0, np.float32), np.full(50, 300.0, np.float32),
                          np.zeros(50, np.int32), np.full(50, 0.9, np.float32), mps.descriptors)
    assert assert_same(mt.SearchByProjection(F2, mp3, 15.0), oracle.port_search_by_projection(F2, mp3, 15.0, 0.8))
    # projections outside the image / nothing in range
    mp4 = M.MapPointsView(np.full(50, -500.0, np.float32), np.full(50, 9000.0, np.float32), np.zeros(50, np.float32),
                          np.full(50, 7, np.int32), np.ones(50, np.float32), mps.descriptors)
    n, m = mt.SearchByProjection(F2, mp4, 3.0)
    assert n == 0 and np.all(m == -1)
    # zero map points
    mp5 = M.MapPointsView(*[np.zeros(0, np.float32)] * 3, np.zeros(0, np.int32), np.zeros(0, np.float32), np.zeros((0, 32), np.uint8))
    n, m = mt.SearchByProjection(F2, mp5, 3.0)
    assert n == 0 and len(m) == 0


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("ratio,ori", [(0.7, True), (0.9, True), (0.75, False)])
def test_search_by_bow_both_variants(M, oracle, views, seed, ratio, ori):
    voc = oracle.PortVocabulary.random(10, 4, 5)
    kf1, kf2 = mf.keyframe_views(views[seed], voc, seed)
    mt = M.ORBmatcher(ratio, ori)
    n_o, m_o = oracle.port_search_by_bow(kf1, kf2, ratio, ori)
    n_g, m_g = mt.SearchByBoW(kf1, kf2)
    assert n_o > 20 and n_g == n_o and np.array_equal(m_g, m_o)
    n_o, m_o = oracle.port_search_by_bow_kf(kf1, kf2, ratio, ori)
    n_g, m_g = mt.SearchByBoW_KF(kf1, kf2)
    assert n_g == n_o and np.array_equal(m_g, m_o)


def test_search_by_bow_batched_keyframes(M, oracle, views):
    """Config-5 shape in miniature: one query frame against several keyframes in one launch."""
    voc = oracle.PortVocabulary.random(10, 4, 5)
    a1, a2 = mf.keyframe_views(views[7], voc, 1)
    b1, b2 = mf.keyframe_views(views[8], voc, 2)
    kfs = [a1, b1, b2, a1]
    nm, match = M.ORBmatcher(0.75, True).SearchByBoW(kfs, a2)
    for i, kf in enumerate(kfs):
        n_o, m_o = oracle.port_search_by_bow(kf, a2, 0.75, True)
        assert nm[i] == n_o and np.array_equal(match[i], m_o), i
    assert np.array_equal(match[0], match[3])


@pytest.mark.parametrize("only_stereo", [False, True])
@pytest.mark.parametrize("ori", [True, False])
def test_search_for_triangulation(M, oracle, views, only_stereo, ori):
    voc = oracle.PortVocabulary.random(10, 4, 5)
    for seed in (7, 8):
        kf1, kf2 = mf.keyframe_views(views[seed], voc, seed + 3, mp_frac=0.3)
        F12 = mf.rectified_F12(seed)
        ep = (-1000.0, 200.0) if seed == 7 else (300.0, 240.0)      # the second epipole sits inside the image: exercises :743-749
        want = oracle.port_search_for_triangulation(kf1, kf2, F12, ep, only_stereo, ori)
        got = M.ORBmatcher(0.6, ori).SearchForTriangulation(kf1, kf2, F12, ep, only_stereo)
        assert len(want) > 5 and np.array_equal(got, want)


def test_vocabulary_transform_and_blob_round_trip(M, oracle, views, tmp_path):
    pv = oracle.PortVocabulary.random(10, 5, 21)             # 111,111 nodes
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    d = np.concatenate([views[7]["dl"], views[8]["dr"]])
    for levelsup in (4, 3, 0, 7):
        wg, tg, ng = voc.transform_raw(d, levelsup)
        wo, to, no = pv.transform_raw(d, levelsup)
        assert np.array_equal(wg, wo) and np.array_equal(tg, to) and np.array_equal(ng, no), levelsup
    # text loader (ORBvoc.txt format) gives the same tree
    path = os.path.join(tmp_path, "voc.txt")
    small = oracle.PortVocabulary.random(10, 3, 4)
    small.save_text(path)
    v2 = M.ORBVocabulary.loadFromTextFile(path)
    assert all(np.array_equal(a, b) for a, b in zip(v2.transform_raw(d[:500], 2), small.transform_raw(d[:500], 2)))
    # packed blob adoption (what the NCCL broadcast receiver does)
    ptr, nbytes = voc.blob()
    v3 = M.ORBVocabulary.from_blob(ptr, nbytes)
    assert all(np.array_equal(a, b) for a, b in zip(v3.transform_raw(d[:300], 4), pv.transform_raw(d[:300], 4)))
    bow, fv = voc.transform(views[7]["dl"], 4)
    assert abs(sum(bow.values()) - 1.0) < 1e-9 and list(bow) == sorted(bow)
    assert np.all(np.diff(fv.node_id.astype(np.int64)) > 0) and fv.start[-1] == len(views[7]["dl"])


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("mode", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("th,ori", [(7.0, True), (15.0, True), (15.0, False)])
def test_search_by_projection_from_last_frame(M, oracle, views, seed, mode, th, ori):
    """SearchByProjection(CurrentFrame, LastFrame, th, bMono), src/ORBmatcher.cc:1328-1470 (TrackWithMotionModel)."""
    Cur, Last, Tcw, K = mf.last_frame_case(views[seed], seed + 20)
    fw, bw = mode
    n_o, s_o = oracle.port_search_by_projection_last(Cur, Last, Tcw, K, 40.0, th, fw, bw, ori)
    n_g, s_g = M.ORBmatcher(0.9, ori).SearchByProjectionLast(Cur, Last, Tcw, K, 40.0, th, fw, bw)
    assert n_o > 20
    assert n_g == n_o and np.array_equal(s_g, s_o), int((s_g != s_o).sum())
    m = s_g[s_g >= 0]
    assert np.all(Last.valid[m] == 1) and np.all(Cur.occupied[np.nonzero(s_g >= 0)[0]] == 0)


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("th,orb_dist,ori", [(10.0, 100, True), (3.0, 64, True), (10.0, 100, False), (25.0, 50, True)])
def test_search_by_projection_from_keyframe(M, oracle, views, seed, th, orb_dist, ori):
    """SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist), src/ORBmatcher.cc:1472-1599 (Relocalization)."""
    Cur, P, Tcw, Ow, K = mf.world_points_case(views[seed], seed + 30)
    n_o, s_o = oracle.port_search_by_projection_kf(Cur, P, Tcw, Ow, K, th, orb_dist, ori)
    n_g, s_g = M.ORBmatcher(0.9, ori).SearchByProjectionKF(Cur, P, Tcw, Ow, K, th, orb_dist)
    assert n_o > 20
    assert n_g == n_o and np.array_equal(s_g, s_o), int((s_g != s_o).sum())
    hit = np.nonzero(s_g >= 0)[0]
    assert np.all(P.valid[s_g[hit]] == 1) and np.all(Cur.occupied[hit] == 0)


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("th", [3, 10, 25])
def test_search_by_projection_sim3(M, oracle, views, seed, th):
    """SearchByProjection(pKF, Scw, vpPoints, vpMatched, th), src/ORBmatcher.cc:290-403 (LoopClosing::ComputeSim3)."""
    KF, P, Tcw, Ow, K = mf.world_points_case(views[seed], seed + 40)
    n_o, s_o = oracle.port_search_by_projection_sim3(KF, P, Tcw, Ow, K, th)
    n_g, s_g = M.ORBmatcher(0.75, True).SearchByProjectionSim3(KF, P, Tcw, Ow, K, th)
    assert n_o > 20
    assert n_g == n_o and np.array_equal(s_g, s_o), int((s_g != s_o).sum())
    hit = np.nonzero(s_g >= 0)[0]
    assert np.all(P.valid[s_g[hit]] == 1) and np.all(KF.occupied[hit] == 0)


def test_pose_projection_overloads_edge_cases(M, oracle, views):
    v = views[7]
    F, P, Tcw, Ow, K = mf.world_points_case(v, 77)
    mt = M.ORBmatcher(0.9, True)
    same = lambda a, b: (a[0] == b[0] and np.array_equal(a[1], b[1]))
    # no occupancy, no validity mask; identity pose puts most points outside the image
    F2 = M.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds)
    P2 = M.WorldPointsView(P.world_pos, P.descriptors, P.max_distance, P.min_distance, P.normal, P.angle)
    assert same(mt.SearchByProjectionKF(F2, P2, Tcw, Ow, K, 10.0, 100), oracle.port_search_by_projection_kf(F2, P2, Tcw, Ow, K, 10.0, 100, True))
    assert same(mt.SearchByProjectionSim3(F2, P2, Tcw, Ow, K, 10), oracle.port_search_by_projection_sim3(F2, P2, Tcw, Ow, K, 10))
    I = np.eye(4, dtype=np.float32)[:3]
    z3 = np.zeros(3, np.float32)
    assert same(mt.SearchByProjectionKF(F2, P2, I, z3, K, 10.0, 100), oracle.port_search_by_projection_kf(F2, P2, I, z3, K, 10.0, 100, True))
    assert same(mt.SearchByProjectionSim3(F2, P2, I, z3, K, 10), oracle.port_search_by_projection_sim3(F2, P2, I, z3, K, 10))
    # points exactly at the camera centre (zero distance, division by zero depth) and at infinity must not crash or match
    bad = P.world_pos.copy(); bad[:40] = Ow; bad[40:80] = 1e30
    P3 = M.WorldPointsView(bad, P.descriptors, P.max_distance, P.min_distance, P.normal, P.angle)
    assert same(mt.SearchByProjectionKF(F2, P3, Tcw, Ow, K, 10.0, 100), oracle.port_search_by_projection_kf(F2, P3, Tcw, Ow, K, 10.0, 100, True))
    assert same(mt.SearchByProjectionSim3(F2, P3, Tcw, Ow, K, 10), oracle.port_search_by_projection_sim3(F2, P3, Tcw, Ow, K, 10))
    # zero query points
    P0 = M.WorldPointsView(np.zeros((0, 3), np.float32), np.zeros((0, 32), np.uint8), np.zeros(0, np.float32), np.zeros(0, np.float32),
                           np.zeros((0, 3), np.float32), np.zeros(0, np.float32))
    n, s = mt.SearchByProjectionSim3(F2, P0, Tcw, Ow, K, 10)
    assert n == 0 and np.all(s == -1)


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("th,scw", [(3.0, False), (6.0, False), (3.0, True), (4.0, True)])
def test_fuse_search_part(M, oracle, views, seed, th, scw):
    """Fuse(pKF, vpMapPoints, th) :825-970 and Fuse(pKF, Scw, vpPoints, th, vpReplacePoint) :972-1100 — the search part."""
    KF, P, Tcw, Ow, K, bf = mf.fuse_case(views[seed], seed + 50)
    n_o, b_o = oracle.port_fuse(KF, P, Tcw, Ow, K, bf, th, scw)
    n_g, b_g = M.ORBmatcher(0.6, True).Fuse(KF, P, Tcw, Ow, K, bf, th, Scw=scw)
    assert n_o > 20 and n_o == int((b_o >= 0).sum())
    assert n_g == n_o and np.array_equal(b_g, b_o), int((b_g != b_o).sum())
    assert np.all(b_g[P.valid == 0] == -1)


def test_fuse_gates_matter(M, oracle, views):
    """The stereo / mono reprojection gates (7.8 / 5.99) must bite: with them off (Scw variant) more points are fused."""
    KF, P, Tcw, Ow, K, bf = mf.fuse_case(views[7], 61, jitter=2.0)
    n0, b0 = M.ORBmatcher().Fuse(KF, P, Tcw, Ow, K, bf, 6.0, Scw=False)
    n1, b1 = M.ORBmatcher().Fuse(KF, P, Tcw, Ow, K, bf, 6.0, Scw=True)
    assert (n0, n1) == (oracle.port_fuse(KF, P, Tcw, Ow, K, bf, 6.0, False)[0], oracle.port_fuse(KF, P, Tcw, Ow, K, bf, 6.0, True)[0])
    assert n1 > n0 > 10
    mono = M.FrameView(KF.mvKeysUn, KF.mDescriptors, KF.mvScaleFactors, KF.bounds, mvInvLevelSigma2=KF.mvInvLevelSigma2)
    n2, b2 = M.ORBmatcher().Fuse(mono, P, Tcw, Ow, K, bf, 6.0)
    n2o, b2o = oracle.port_fuse(mono, P, Tcw, Ow, K, bf, 6.0, False)
    assert n2 == n2o and np.array_equal(b2, b2o)


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("th", [7.5, 3.0, 15.0])
def test_search_by_sim3(M, oracle, views, seed, th):
    """SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th), src/ORBmatcher.cc:1102-1326."""
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = mf.sim3_case(views[seed], seed + 60)
    n_o, m_o = oracle.port_search_by_sim3(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K, th)
    n_g, m_g = M.ORBmatcher(0.75, True).SearchBySim3(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K, th)
    assert n_o > 20 and n_o == int((m_o >= 0).sum())
    assert n_g == n_o and np.array_equal(m_g, m_o), int((m_g != m_o).sum())
    hit = np.nonzero(m_g >= 0)[0]
    assert np.all(P1.valid[hit] == 1) and np.all(P2.valid[m_g[hit]] == 1)
    assert len(set(m_g[hit].tolist())) == len(hit)                       # mutual agreement makes the matching one-to-one


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("window,ratio,ori", [(100, 0.9, True), (30, 0.9, True), (100, 0.7, False), (10, 0.9, True)])
def test_search_for_initialization(M, oracle, views, seed, window, ratio, ori):
    """SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize), src/ORBmatcher.cc:405-520."""
    v = views[seed]
    b = (0.0, 0.0, float(v["w"]), float(v["h"]))
    F1 = M.FrameView(v["kl"], v["dl"], v["scale"], b)
    F2 = M.FrameView(v["kr"], v["dr"], v["scale"], b)
    prev = np.stack([v["kl"]["x"], v["kl"]["y"]], 1).astype(np.float32)      # mvbPrevMatched = initial keypoint positions
    n_o, m_o, p_o = oracle.port_search_for_initialization(F1, F2, prev, window, ratio, ori)
    n_g, m_g, p_g = M.ORBmatcher(ratio, ori).SearchForInitialization(F1, F2, prev, window)
    assert n_o == int((m_o >= 0).sum()) and (n_o > 20 or window < 30)
    assert n_g == n_o and np.array_equal(m_g, m_o), int((m_g != m_o).sum())
    assert np.array_equal(p_g, p_o)
    hit = np.nonzero(m_g >= 0)[0]
    assert np.all(v["kl"]["octave"][hit] == 0) and np.all(v["kr"]["octave"][m_g[hit]] == 0)
    assert len(set(m_g[hit].tolist())) == len(hit)                           # displacement keeps the matching one-to-one
    # second round with the updated window centres (what the tracker does on the next frame)
    n_o2, m_o2, p_o2 = oracle.port_search_for_initialization(F1, F2, p_o, max(window // 2, 5), ratio, ori)
    n_g2, m_g2, p_g2 = M.ORBmatcher(ratio, ori).SearchForInitialization(F1, F2, p_g, max(window // 2, 5))
    assert n_g2 == n_o2 and np.array_equal(m_g2, m_o2) and np.array_equal(p_g2, p_o2)


def test_distinctive_descriptors(M, oracle, views):
    """MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307), batched over MapPoints."""
    rng = np.random.default_rng(5)
    d = views[7]["dl"]
    groups = []
    for n in [1, 2, 3, 4, 5, 8, 13, 33, 64, 100, 300, 0, 7]:
        base = d[rng.integers(0, len(d))]
        g = np.repeat(base[None], n, 0).copy()
        flips = rng.integers(0, 256, (n, 12))
        for i in range(n):                                    # noisy copies of one descriptor: a realistic observation set
            for b in flips[i][: rng.integers(0, 12)]:
                g[i, b >> 3] ^= np.uint8(1 << (b & 7))
        groups.append(g)
    groups.append(np.repeat(d[:1], 6, 0))                     # all identical: every median 0, first index wins
    groups.append(d[rng.integers(0, len(d), 40)])             # unrelated descriptors
    got = M.ORBmatcher().ComputeDistinctiveDescriptors(groups)
    want = np.array([oracle.port_distinctive_descriptor(g) for g in groups], np.int32)
    assert np.array_equal(got, want), (got, want)
    assert want[11] == -1 and want[13] == 0


@pytest.mark.parametrize("seed", [7, 8])
@pytest.mark.parametrize("th,ratio", [(1.0, 0.8), (3.0, 0.8), (5.0, 0.9)])
def test_search_local_points_frustum_plus_projection(M, oracle, views, seed, th, ratio):
    """Frame::isInFrustum (src/Frame.cc:269-325) + SearchByProjection(F, vpMapPoints, th) (src/ORBmatcher.cc:45-129) fused."""
    v = views[seed]
    F, P, Tcw, Ow, K = mf.world_points_case(v, seed + 70)
    F = M.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds, mvuRight=v["ur"], occupied=F.occupied)
    rng = np.random.default_rng(seed)
    has_obs = (rng.random(len(P.world_pos)) < 0.9).astype(np.uint8)
    fr = oracle.port_is_in_frustum(F, P, Tcw, Ow, K, 40.0, 0.5)
    mps = M.MapPointsView(fr["proj_x"], fr["proj_y"], fr["proj_xr"], fr["level"], fr["view_cos"], P.descriptors, valid=fr["in_view"],
                          has_obs=has_obs)
    n_o, m_o = oracle.port_search_by_projection(F, mps, th, ratio)
    got = M.ORBmatcher(ratio, True).SearchLocalPoints(F, P, Tcw, Ow, K, 40.0, th, has_obs=has_obs)
    assert fr["count"] > 200 and n_o > 30
    assert np.array_equal(got["in_view"], fr["in_view"])
    for f in ("proj_x", "proj_y", "proj_xr", "level", "view_cos"):
        assert np.array_equal(got[f], fr[f]), f                           # bit-identical floats, not just close
    assert got["nmatches"] == n_o and np.array_equal(got["match"], m_o), int((got["match"] != m_o).sum())


from tests.golden_match_cases import CASES as GOLDEN_CASES, flatten as golden_flatten     # noqa: E402


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_matches_reference_golden_vectors(M, oracle, name):
    """tests/golden/match_ref.npz holds what the reference's own src/ORBmatcher.cc (compiled verbatim, oracle/_ref/libmatchref.so)
    produced for these seeded cases (tests/golden/make_golden_match.py); the CUDA library must reproduce it bit for bit."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "match_ref.npz"))
    build, _port, gpu = GOLDEN_CASES[name]
    assert np.array_equal(golden_flatten(gpu(M, build(oracle))), g[name])


@pytest.mark.parametrize("seed", [7, 8])
def test_resident_frame_gives_the_same_results(M, oracle, views, seed):
    """borb_frame (device-resident Frame, §8 f4): the three Tracking-thread searches through a resident frame equal the
    host-view calls and the oracle; the resident frame is reused across calls and across matcher handles."""
    v = views[seed]
    mt, mt2 = M.ORBmatcher(0.8, True), M.ORBmatcher(0.9, True)
    F, mps = mf.projection_case(v, seed + 10, n_mp=400)
    FR = F.make_resident(mt)
    n_o, m_o = oracle.port_search_by_projection(F, mps, 3.0, 0.8)
    for _ in range(2):
        n_g, m_g = mt.SearchByProjection(FR, mps, 3.0)
        assert n_g == n_o and np.array_equal(m_g, m_o)
    # the occupancy mask still travels per call
    import dataclasses
    occ2 = np.zeros(len(F.mvKeysUn), np.uint8); occ2[::3] = 1
    F2, FR2 = dataclasses.replace(F, occupied=occ2), dataclasses.replace(FR, occupied=occ2)
    n_o2, m_o2 = oracle.port_search_by_projection(F2, mps, 3.0, 0.8)
    n_g2, m_g2 = mt.SearchByProjection(FR2, mps, 3.0)
    assert n_g2 == n_o2 and np.array_equal(m_g2, m_o2) and not np.array_equal(m_o2, m_o)
    # motion-model search on another matcher handle (another thread's stream) against the same resident frame
    Cur, Last, Tcw, K = mf.last_frame_case(v, seed + 20)
    CurR = Cur.make_resident(mt)
    n_o3, s_o3 = oracle.port_search_by_projection_last(Cur, Last, Tcw, K, 40.0, 7.0, False, False, True)
    n_g3, s_g3 = mt2.SearchByProjectionLast(CurR, Last, Tcw, K, 40.0, 7.0)
    assert n_g3 == n_o3 and np.array_equal(s_g3, s_o3)
    # SearchLocalPoints
    Fw, P, Tcw2, Ow, K2 = mf.world_points_case(v, seed + 70)
    Fw = M.FrameView(Fw.mvKeysUn, Fw.mDescriptors, Fw.mvScaleFactors, Fw.bounds, mvuRight=v["ur"], occupied=Fw.occupied)
    a = mt.SearchLocalPoints(Fw, P, Tcw2, Ow, K2, 40.0, 3.0)
    b = mt.SearchLocalPoints(Fw.make_resident(mt), P, Tcw2, Ow, K2, 40.0, 3.0)
    assert a["nmatches"] == b["nmatches"] > 30
    for f in a:
        assert np.array_equal(a[f], b[f]), f


def test_search_local_points_skips_invalid_points(M, oracle, views):
    """Points that never reach isInFrustum (already matched / bad, src/Tracking.cc:1171-1175) are not staged: results of the
    valid ones are unchanged and the invalid ones read 'not in view'."""
    v = views[7]
    F, P, Tcw, Ow, K = mf.world_points_case(v, 77)
    F = M.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds, mvuRight=v["ur"], occupied=F.occupied)
    import dataclasses
    rng = np.random.default_rng(5)
    valid = (rng.random(len(P.world_pos)) < 0.6).astype(np.uint8)
    Pv = dataclasses.replace(P, valid=valid)
    mt = M.ORBmatcher(0.8, True)
    got = mt.SearchLocalPoints(F, Pv, Tcw, Ow, K, 40.0, 3.0)
    fr = oracle.port_is_in_frustum(F, Pv, Tcw, Ow, K, 40.0, 0.5)
    mps = M.MapPointsView(fr["proj_x"], fr["proj_y"], fr["proj_xr"], fr["level"], fr["view_cos"], P.descriptors, valid=fr["in_view"])
    n_o, m_o = oracle.port_search_by_projection(F, mps, 3.0, 0.8)
    assert np.array_equal(got["in_view"], fr["in_view"]) and not np.any(got["in_view"][valid == 0])
    for f in ("proj_x", "proj_y", "proj_xr", "level", "view_cos"):
        assert np.array_equal(got[f], fr[f]), f
    assert got["nmatches"] == n_o > 20 and np.array_equal(got["match"], m_o)


@pytest.mark.parametrize("th", [40.0, 150.0])
def test_long_candidate_lists(M, oracle, views, th):
    """Candidate lists beyond one warp (sorted in place up to 128 entries) and beyond the sort capacity (kept in position order,
    resolved by full scans): huge search windows on the motion-model search and on SearchByProjection(F, MapPoints)."""
    v = views[8]
    Cur, Last, Tcw, K = mf.last_frame_case(v, 31)
    for fw, bw in ((False, False), (True, False)):
        n_o, s_o = oracle.port_search_by_projection_last(Cur, Last, Tcw, K, 40.0, th, fw, bw, True)
        n_g, s_g = M.ORBmatcher(0.9, True).SearchByProjectionLast(Cur, Last, Tcw, K, 40.0, th, fw, bw)
        assert n_g == n_o > 20 and np.array_equal(s_g, s_o), int((s_g != s_o).sum())
    F, mps = mf.projection_case(v, 19, n_mp=300)
    n_o, m_o = oracle.port_search_by_projection(F, mps, th, 0.9)
    n_g, m_g = M.ORBmatcher(0.9, True).SearchByProjection(F, mps, th)
    assert n_g == n_o and np.array_equal(m_g, m_o), int((m_g != m_o).sum())


def test_compute_bow_equals_the_reference_bookkeeping(M, oracle, views):
    """borb_compute_bow (Frame::ComputeBoW, src/Frame.cc:395-402): BowVector / FeatureVector built on the device equal the Python mirror of
    TemplatedVocabulary::transform's map bookkeeping, which tests/test_oracle_dbow_ref.py pins to the verbatim DBoW2 (bit-exact doubles)."""
    pv = oracle.PortVocabulary.random(10, 5, 21)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    for d, levelsup in ((views[7]["dl"], 4), (views[8]["dr"], 3), (views[7]["dl"][:1], 4), (views[7]["dl"][:0], 4)):
        bow_c, fv_c = voc.ComputeBoW(d, levelsup)
        bow_p, fv_p = voc.transform(d, levelsup)
        assert list(bow_c.items()) == list(bow_p.items())                  # same words, same order, bit-identical doubles
        assert np.array_equal(fv_c.node_id, fv_p.node_id) and np.array_equal(fv_c.start, fv_p.start) and np.array_equal(fv_c.feat_idx, fv_p.feat_idx)


def test_search_by_projection_batch_equals_single_calls(M, oracle, views):
    """borb_search_by_projection_batch: many independent (resident frame, MapPoint list) jobs in one launch pair — every job's
    result equals the single call and the oracle; jobs of different sizes, with and without occupancy masks / validity flags,
    an empty MapPoint list, and a list long enough for the 512- and 1024-thread resolve configurations."""
    import dataclasses
    mt = M.ORBmatcher(0.8, True)
    frames, lists, want = [], [], []
    for j, (seed, n_mp) in enumerate([(7, 300), (8, 40), (7, 700), (8, 0), (7, 1), (8, 300)]):
        v = views[seed]
        F, mps = mf.projection_case(v, 100 + j, n_mp=max(n_mp, 1))
        if n_mp == 0:
            mps = dataclasses.replace(mps, mTrackProjX=mps.mTrackProjX[:0], mTrackProjY=mps.mTrackProjY[:0], mTrackProjXR=mps.mTrackProjXR[:0],
                                      mnTrackScaleLevel=mps.mnTrackScaleLevel[:0], mTrackViewCos=mps.mTrackViewCos[:0], descriptors=mps.descriptors[:0],
                                      valid=None if mps.valid is None else mps.valid[:0], has_obs=None if mps.has_obs is None else mps.has_obs[:0])
        if j % 2 == 1:
            occ = np.zeros(len(F.mvKeysUn), np.uint8); occ[j::4] = 1
            F = dataclasses.replace(F, occupied=occ)
        FR = dataclasses.replace(F.make_resident(mt), occupied=F.occupied)
        frames.append(FR); lists.append(mps)
        want.append(oracle.port_search_by_projection(F, mps, 3.0, 0.8) if n_mp else (0, np.zeros(0, np.int32)))
    got = mt.SearchByProjectionBatch(frames, lists, 3.0)
    assert len(got) == len(want)
    for j, ((n_g, m_g), (n_o, m_o)) in enumerate(zip(got, want)):
        assert n_g == n_o and np.array_equal(m_g, m_o), j
        if len(m_o):
            n_s, m_s = mt.SearchByProjection(frames[j], lists[j], 3.0)
            assert n_s == n_o and np.array_equal(m_s, m_o), j
    assert got[0][0] > 50 and got[2][0] > 100
    # a host view (not resident) is refused loudly
    F0, mps0 = mf.projection_case(views[7], 100, n_mp=10)
    with pytest.raises(Exception):
        mt.SearchByProjectionBatch([F0], [mps0], 3.0)
