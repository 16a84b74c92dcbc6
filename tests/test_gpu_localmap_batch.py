"""GPU parity of the batched LocalMapping searches: borb_search_for_triangulation_batch (CreateNewMapPoints' SearchForTriangulation
against every neighbour) and borb_fuse_batch (the Fuse calls of SearchInNeighbors / SearchAndFuse).  Every job must equal the oracle
restatement and the single call bit for bit; a call is one launch (triangulation) or two (Fuse) whatever its size, and argument
errors are refused before anything is launched."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from tests import localmap_fixtures as lf
from tests import match_fixtures as mf
from tests.test_gpu_track_batch import reanchor

pytestmark = pytest.mark.gpu

LEVELSUP = 2


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def views(oracle):
    return {s: mf.two_views(oracle, s) for s in (7, 8)}


@pytest.fixture(scope="module")
def vocs(M, oracle):
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    return pv, M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def make_resident(M, mt, voc, kf):
    """kf as a device-resident frame with the BoW of borb_frames_compute_bow (which must be kf's FeatureVector)."""
    k = kf.mvKeysUn
    bounds = (0.0, 0.0, float(max(640.0, k["x"].max() + 1 if len(k) else 0)), float(max(480.0, k["y"].max() + 1 if len(k) else 0)))
    F = M.FrameView(k, kf.mDescriptors, kf.mvScaleFactors, bounds, mvuRight=kf.mvuRight).make_resident(mt)
    _, fv = mt.ComputeBoWBatch(voc, [F], LEVELSUP)[0]
    assert np.array_equal(fv.node_id, kf.mFeatVec.node_id) and np.array_equal(fv.feat_idx, kf.mFeatVec.feat_idx)
    return dataclasses.replace(F, has_mp=kf.has_mp)


def big_keyframe(views, pv, rng):
    """An 8192-feature keyframe (the four views tiled, descriptors perturbed)."""
    k = np.concatenate([views[7]["kl"], views[7]["kr"], views[8]["kl"], views[8]["kr"]] * 3)[:8192]
    d = lf.flip_bits(rng, np.concatenate([views[7]["dl"], views[7]["dr"], views[8]["dl"], views[8]["dr"]] * 3)[:8192], 0.03)
    _, w, node = pv.transform_raw(d, LEVELSUP)
    ur = np.where(rng.random(len(k)) < 0.5, k["x"] - 20.0, -1.0).astype(np.float32)
    return dict(mvKeysUn=k, mDescriptors=d, mFeatVec=mf.FeatureVector.from_nodes(node, w > 0), mvuRight=ur,
                has_mp=(rng.random(len(k)) < 0.3).astype(np.uint8), mvScaleFactors=views[7]["scale"], mvLevelSigma2=views[7]["sigma2"])


def triangulation_world(M, views, vocs, mt):
    """(jobs as (kf1, kf2, F12, epipole, only_stereo) with sides as host views or resident frames, the host views of every job)."""
    pv, voc = vocs
    rng = np.random.default_rng(4)
    host = {}
    for s in (7, 8):
        host[s] = mf.keyframe_views(views[s], pv, s + 3, mp_frac=0.3)
    kf1, kf2s = lf.neighbourhood(views[7], pv)
    big = M.KeyFrameView(**big_keyframe(views, pv, rng))
    h7a, h7b = host[7]
    empty = M.KeyFrameView(mvKeysUn=h7a.mvKeysUn[:0], mDescriptors=h7a.mDescriptors[:0], mFeatVec=M.FeatureVector(np.zeros(0, np.uint32),
                           np.zeros(1, np.int32), np.zeros(0, np.uint32)), has_mp=np.zeros(0, np.uint8), mvuRight=np.zeros(0, np.float32),
                           mvScaleFactors=h7a.mvScaleFactors, mvLevelSigma2=h7a.mvLevelSigma2)
    no_fv = dataclasses.replace(h7b, mFeatVec=M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32)))
    res = {id(x): make_resident(M, mt, voc, x) for x in [kf1, h7a, h7b, host[8][0], host[8][1], big, empty]}
    R = lambda x: res[id(x)]
    ep_out, ep_in = (-1000.0, 200.0), (300.0, 240.0)              # outside / inside the image: the inside one exercises :743-749
    F7, F8 = mf.rectified_F12(7), mf.rectified_F12(8)
    jobs = []
    # one kf1 against its six neighbours, kf1 alternately a host view and a resident frame
    for i, kf2 in enumerate(kf2s):
        jobs.append(((kf1, R(kf1) if i % 2 else kf1), (kf2, kf2), F7, ep_in if i % 3 else ep_out, i == 4))
    jobs += [((h7a, R(h7a)), (h7b, R(h7b)), F7, ep_out, False),
             ((host[8][0], host[8][0]), (host[8][1], R(host[8][1])), F8, ep_in, False),
             ((host[8][0], R(host[8][0])), (host[8][1], host[8][1]), F8, ep_in, True),
             ((big, R(big)), (h7b, R(h7b)), F7, ep_out, False),
             ((h7a, h7a), (big, big), F7, ep_in, False),
             ((empty, R(empty)), (h7b, h7b), F7, ep_in, False),
             ((h7a, h7a), (empty, empty), F7, ep_in, False),
             ((h7a, R(h7a)), (no_fv, no_fv), F7, ep_in, False)]
    return jobs


@pytest.mark.parametrize("ori", [False, True])
def test_triangulation_batch_equals_oracle_and_single_calls(M, oracle, views, vocs, ori):
    mt = M.ORBmatcher(0.6, ori)
    jobs = triangulation_world(M, views, vocs, mt)
    c0 = launches(mt)
    got = mt.SearchForTriangulationBatch([j[0][1] for j in jobs], [j[1][1] for j in jobs], [j[2] for j in jobs], [j[3] for j in jobs], [j[4] for j in jobs])
    assert launches(mt) - c0 == 1
    for i, ((h1, _), (h2, _), F12, ep, st) in enumerate(jobs):
        single = mt.SearchForTriangulation(h1, h2, F12, ep, st)
        assert np.array_equal(got[i], single), i
        if len(h1.mvKeysUn) and len(h2.mvKeysUn):
            want = oracle.port_search_for_triangulation(h1, h2, F12, ep, st, ori)
            assert np.array_equal(got[i], want), i
    assert all(len(got[i]) > 5 for i in (0, 1, 2, 3, 5, 6, 7, 9)) and len(got[10]) > 5
    assert len(got[11]) == len(got[12]) == len(got[13]) == 0
    assert len(got[4]) < len(got[3])                                # only_stereo


def test_one_launch_per_triangulation_call_and_none_without_work(M, views, vocs):
    pv, _ = vocs
    mt = M.ORBmatcher(0.6, False)
    kf1, kf2s = lf.neighbourhood(views[7], pv)
    F12 = mf.rectified_F12(7)
    for n in (1, 6):
        c0 = launches(mt)
        mt.SearchForTriangulationBatch([kf1] * n, kf2s[:n], [F12] * n, [(300.0, 240.0)] * n)
        assert launches(mt) - c0 == 1
    empty = dataclasses.replace(kf1, mvKeysUn=kf1.mvKeysUn[:0], mDescriptors=kf1.mDescriptors[:0], has_mp=kf1.has_mp[:0],
                                mvuRight=kf1.mvuRight[:0], mFeatVec=mf.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32)))
    c0 = launches(mt)
    assert [len(p) for p in mt.SearchForTriangulationBatch([empty, kf1], [kf2s[0], empty], [F12] * 2, [(300.0, 240.0)] * 2)] == [0, 0]
    assert launches(mt) == c0


def test_replay_of_create_new_map_points_equals_sequential_single_calls(M, views, vocs):
    pv, _ = vocs
    mt = M.ORBmatcher(0.6, False)
    kf1, kf2s = lf.neighbourhood(views[7], pv)
    F12, ep = mf.rectified_F12(7), (300.0, 240.0)
    entry = mt.SearchForTriangulationBatch([kf1] * len(kf2s), kf2s, [F12] * len(kf2s), [ep] * len(kf2s))
    rep = lf.replay(entry, kf1.has_mp)
    seq = lf.sequential(lambda a, b: mt.SearchForTriangulation(a, b, F12, ep), kf1, kf2s)
    for i, (a, b) in enumerate(zip(seq, rep)):
        assert np.array_equal(a, b), i
    assert all(len(p) > 10 for p in seq) and sum(len(e) - len(r) for e, r in zip(entry, rep)) > 20


def test_triangulation_capacity_names_the_first_overflowing_job(M, views, vocs):
    pv, _ = vocs
    mt = M.ORBmatcher(0.6, False)
    kf1, kf2s = lf.neighbourhood(views[7], pv)
    F12, ep = mf.rectified_F12(7), (300.0, 240.0)
    full = mt.SearchForTriangulationBatch([kf1] * 3, kf2s[:3], [F12] * 3, [ep] * 3)
    caps = [None, 5, 3]
    n = 3
    jobs = (M._TriangulationJobC * n)()
    keep, outs = [], []
    for j in range(n):
        J = jobs[j]
        J.kf1, J.kf1_frame, n1 = mt._tri_side(kf1, keep)
        J.kf2, J.kf2_frame, _ = mt._tri_side(kf2s[j], keep)
        J.F12 = (C.c_float * 9)(*F12.reshape(9).tolist())
        J.ex, J.ey = ep
        cap = n1 if caps[j] is None else caps[j]
        pairs, npairs = np.zeros((max(cap, 1), 2), np.int32), np.zeros(1, np.int32)
        J.pairs, J.cap, J.n_pairs = pairs.ctypes.data, cap, npairs.ctypes.data
        outs.append((pairs, npairs))
    c0 = launches(mt)
    assert mt._lib.borb_search_for_triangulation_batch(mt._h, jobs, n, 0) == 5          # BORB_ERR_CAPACITY
    err = mt._lib.borb_last_error().decode()
    assert err.startswith("job 1:"), err
    assert launches(mt) - c0 == 1
    for j, (pairs, npairs) in enumerate(outs):
        assert int(npairs[0]) == len(full[j]) > 5
        k = min(len(full[j]), len(pairs))
        assert np.array_equal(pairs[:k], full[j][:k])


def fuse_job(M, mt, v, seed, a, mono=False, valid="fixture", n_points=None):
    KF, P, Tcw, _, K, bf = mf.fuse_case(v, seed)
    if mono:
        KF = dataclasses.replace(KF, mvuRight=None)
    Pw, T2, Ow, nr = reanchor(a, P.world_pos, Tcw, P.normal)
    P = dataclasses.replace(P, world_pos=Pw, normal=nr)
    if n_points is not None:
        idx = np.arange(n_points) % len(P.world_pos)
        P = dataclasses.replace(P, world_pos=P.world_pos[idx], descriptors=P.descriptors[idx], max_distance=P.max_distance[idx],
                                min_distance=P.min_distance[idx], normal=P.normal[idx], valid=P.valid[idx])
    if valid is None:
        P = dataclasses.replace(P, valid=None)
    elif isinstance(valid, str) and valid == "none":
        P = dataclasses.replace(P, valid=np.zeros(len(P.world_pos), np.uint8))
    return KF, KF.make_resident(mt), P, (T2, Ow), K, bf


def test_fuse_batch_equals_oracle_and_single_calls(M, oracle, views):
    mt = M.ORBmatcher(0.6, True)
    specs = [  # (view, seed, angle, mono, valid, points, th, scw)
        (7, 57, 0.0, False, "fixture", None, 3.0, False), (8, 58, 0.3, False, "fixture", None, 6.0, False),
        (7, 59, -0.2, True, "fixture", None, 3.0, False), (8, 60, 0.5, False, "fixture", None, 3.0, True),
        (7, 61, 0.1, True, "fixture", None, 4.0, True), (7, 62, 0.2, False, None, None, 5.0, False),
        (8, 63, 0.4, False, "fixture", 0, 3.0, False), (7, 64, -0.4, False, "none", None, 3.0, True),
        (7, 57, 0.0, False, "fixture", None, 3.0, False),          # a repeated keyframe and point set
    ]
    jobs = [fuse_job(M, mt, views[vs], sd, a, mono, valid, npts) + (th, scw) for vs, sd, a, mono, valid, npts, th, scw in specs]
    c0 = launches(mt)
    got = mt.FuseBatch([j[1] for j in jobs], [j[2] for j in jobs], [j[3] for j in jobs], [j[4] for j in jobs], [j[5] for j in jobs],
                       [j[6] for j in jobs], [j[7] for j in jobs])
    assert launches(mt) - c0 == 2
    for i, ((KF, KFr, P, (T, Ow), K, bf, th, scw), (n_g, b_g)) in enumerate(zip(jobs, got)):
        n_o, b_o = oracle.port_fuse(KF, P, T, Ow, K, bf, th, scw)
        n_s, b_s = mt.Fuse(KF, P, T, Ow, K, bf, th, Scw=scw)
        n_r, b_r = mt.Fuse(KFr, P, T, Ow, K, bf, th, Scw=scw)
        assert n_g == n_o == n_s == n_r and np.array_equal(b_g, b_o) and np.array_equal(b_g, b_s) and np.array_equal(b_g, b_r), (i, n_g, n_o)
    assert all(got[i][0] > 20 for i in (0, 1, 2, 3, 4, 5, 8))
    assert got[6][0] == 0 and len(got[6][1]) == 0 and got[7][0] == 0 and np.all(got[7][1] == -1)
    assert np.array_equal(got[0][1], got[8][1])


def test_fuse_batch_envelope_8192_points_against_8192_features(M, oracle, views, vocs):
    """16 jobs of 8192 valid points against 8192-feature keyframes in one call: a candidate list per point would need 16 x 256 MB."""
    pv, _ = vocs
    rng = np.random.default_rng(6)
    mt = M.ORBmatcher(0.6, True)
    KF, P, Tcw, Ow, K, bf = mf.fuse_case(views[7], 57)
    big = big_keyframe(views, pv, rng)
    k = big["mvKeysUn"].copy()
    k[:len(KF.mvKeysUn)] = KF.mvKeysUn                             # the fixture's keyframe first: its points find their features
    d = big["mDescriptors"].copy()
    d[:len(KF.mvKeysUn)] = KF.mDescriptors
    ur = big["mvuRight"].copy()
    ur[:len(KF.mvKeysUn)] = KF.mvuRight
    BK = M.FrameView(k, d, KF.mvScaleFactors, KF.bounds, mvuRight=ur, mvInvLevelSigma2=KF.mvInvLevelSigma2)
    BKr = BK.make_resident(mt)
    idx = np.arange(8192) % len(P.world_pos)
    jit = rng.normal(0, 0.01, (8192, 3)).astype(np.float32)
    P8 = dataclasses.replace(P, world_pos=(P.world_pos[idx] + jit).astype(np.float32), descriptors=lf.flip_bits(rng, P.descriptors[idx], 0.01),
                             max_distance=P.max_distance[idx], min_distance=P.min_distance[idx], normal=P.normal[idx], valid=None)
    n = 16
    scw = [bool(j % 2) for j in range(n)]
    got = mt.FuseBatch([BKr] * n, [P8] * n, [(Tcw, Ow)] * n, K, bf, [3.0 + (j % 4) for j in range(n)], scw)
    for j in range(n):
        n_s, b_s = mt.Fuse(BKr, P8, Tcw, Ow, K, bf, 3.0 + (j % 4), Scw=scw[j])
        assert got[j][0] == n_s > 1000 and np.array_equal(got[j][1], b_s), j
    n_o, b_o = oracle.port_fuse(BK, P8, Tcw, Ow, K, bf, 3.0, False)
    assert got[0][0] == n_o and np.array_equal(got[0][1], b_o)


def test_fuse_batch_launches_and_refusals(M, oracle, views):
    from orb_slam2_b200._lib import BorbError
    mt = M.ORBmatcher(0.6, True)
    KF, KFr, P, pose, K, bf = fuse_job(M, mt, views[7], 57, 0.0)
    P0 = dataclasses.replace(P, world_pos=P.world_pos[:0], descriptors=P.descriptors[:0], max_distance=P.max_distance[:0],
                             min_distance=P.min_distance[:0], normal=P.normal[:0], valid=P.valid[:0])
    for n in (1, 5):
        c0 = launches(mt)
        mt.FuseBatch([KFr] * n, [P] * n, [pose] * n, K, bf)
        assert launches(mt) - c0 == 2
    c0 = launches(mt)
    assert mt.FuseBatch([KFr, KFr], [P0, dataclasses.replace(P, valid=np.zeros(len(P.world_pos), np.uint8))], [pose] * 2, K, bf)[0][0] == 0
    assert launches(mt) - c0 == 2                                  # the invalid points are still projected
    c0 = launches(mt)
    (n0, b0), = mt.FuseBatch([KFr], [P0], [pose], K, bf)
    assert n0 == 0 and len(b0) == 0 and launches(mt) == c0         # nothing live: no launch

    def refused(call, job):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        assert ei.value.status == 1 and str(ei.value).find(f"job {job}:") >= 0, str(ei.value)
        assert launches(mt) == c0

    refused(lambda: mt.FuseBatch([KFr, KF], [P, P], [pose] * 2, K, bf), 1)                       # host view
    no_sigma = dataclasses.replace(KFr, mvInvLevelSigma2=None)
    refused(lambda: mt.FuseBatch([KFr, KFr, no_sigma], [P] * 3, [pose] * 3, K, bf), 2)
    refused(lambda: mt.FuseBatch([KFr, dataclasses.replace(KFr, mfLogScaleFactor=0.0)], [P] * 2, [pose] * 2, K, bf), 1)
    big = dataclasses.replace(P, world_pos=np.zeros((8193, 3), np.float32), descriptors=np.zeros((8193, 32), np.uint8),
                              max_distance=np.ones(8193, np.float32), min_distance=np.ones(8193, np.float32), normal=np.zeros((8193, 3), np.float32),
                              valid=None)
    refused(lambda: mt.FuseBatch([KFr, KFr], [P, big], [pose] * 2, K, bf), 1)
    n, b = mt.FuseBatch([KFr], [P], [pose], K, bf)[0]
    assert (n, list(b)) == (lambda r: (r[0], list(r[1])))(oracle.port_fuse(KF, P, pose[0], pose[1], K, bf, 3.0, False))


def test_triangulation_refusals_name_the_job_and_launch_nothing(M, views, vocs):
    from orb_slam2_b200._lib import BorbError
    pv, voc = vocs
    mt = M.ORBmatcher(0.6, False)
    kf1, kf2s = lf.neighbourhood(views[7], pv)
    F12, ep = mf.rectified_F12(7), (300.0, 240.0)
    good = make_resident(M, mt, voc, kf1)
    no_bow = dataclasses.replace(M.FrameView(kf1.mvKeysUn, kf1.mDescriptors, kf1.mvScaleFactors, (0.0, 0.0, 640.0, 480.0)).make_resident(mt),
                                 has_mp=kf1.has_mp)
    idx = np.arange(8193) % len(kf1.mvKeysUn)
    too_big = dataclasses.replace(kf1, mvKeysUn=kf1.mvKeysUn[idx], mDescriptors=kf1.mDescriptors[idx], has_mp=kf1.has_mp[idx], mvuRight=kf1.mvuRight[idx])

    def refused(kf1s, kf2s_, job):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            mt.SearchForTriangulationBatch(kf1s, kf2s_, [F12] * len(kf1s), [ep] * len(kf1s))
        assert ei.value.status == 1 and f"job {job}:" in str(ei.value), str(ei.value)
        assert launches(mt) == c0

    refused([good, no_bow], kf2s[:2], 1)
    refused([kf1, kf1, kf1], [kf2s[0], kf2s[1], dataclasses.replace(kf2s[2], mvLevelSigma2=None)], 2)
    refused([kf1, too_big], kf2s[:2], 1)
    assert len(mt.SearchForTriangulationBatch([good], kf2s[:1], [F12], [ep])[0]) > 5
