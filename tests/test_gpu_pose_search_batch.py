"""GPU parity of the batched pose searches on resident frames: borb_search_by_projection_kf_batch (relocalisation after PnP),
borb_search_by_projection_sim3_batch and borb_search_by_sim3_batch (LoopClosing::ComputeSim3).  Every job must equal the single call
on host views of the same frames and the oracle restatement bit for bit; each batch is three launches whatever its size, and argument
errors are refused before anything is launched."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from tests import match_envelope as E
from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu

RELOC = [(10.0, 100, True), (3.0, 64, True), (10.0, 100, False), (3.0, 64, False)]      # src/Tracking.cc:1452, 1466
S12_ARGS = (np.float32(1.03), 0.004, np.array([0.4, 0.01, -0.02], np.float32))            # the transform behind mf.sim3_case


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def views(oracle):
    return {s: mf.two_views(oracle, s) for s in (7, 8)}


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1])


def resident(mt, F):
    return F.make_resident(mt)


def sim3_mats(O):
    s12, a, t12 = S12_ARGS
    R12 = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], np.float32)
    return (s12, R12, t12), O.ref_sim3_mats(s12, R12, t12)


# ---- job builders: host-view cases cycling through the views, each job with its own seed
def kf_cases(views, n_jobs, seed):
    keys = sorted(views)
    return [mf.world_points_case(views[keys[j % len(keys)]], seed + j % 5) for j in range(n_jobs)]


def sim3_cases(O, views, n_jobs, seed):
    _, (S12, S21) = sim3_mats(O)
    keys = sorted(views)
    out = []
    for j in range(n_jobs):
        KF1, KF2, P1, P2, T1w, T2w, _, _, K = mf.sim3_case(views[keys[j % len(keys)]], seed + j % 5)
        out.append((KF1, KF2, P1, P2, T1w, T2w, S12, S21, K))
    return out


def run_kf(mt, O, cases, th, od):
    """cases = [(Cur, P, Tcw, Ow, K)] host views: the batch on resident copies equals the single call and the port."""
    got = mt.SearchByProjectionKFBatch([resident(mt, c[0]) for c in cases], [c[1] for c in cases], [(c[2], c[3]) for c in cases],
                                       [c[4] for c in cases], th, od)
    ths, ods = np.broadcast_to(th, len(cases)), np.broadcast_to(od, len(cases))
    for (Cur, P, Tcw, Ow, K), g, t, o in zip(cases, got, ths, ods):
        assert same(g, mt.SearchByProjectionKF(Cur, P, Tcw, Ow, K, t, o))
        assert same(g, O.port_search_by_projection_kf(Cur, P, Tcw, Ow, K, float(t), int(o), mt.mbCheckOrientation))
    return got


def run_sim3proj(mt, O, cases, th):
    got = mt.SearchByProjectionSim3Batch([resident(mt, c[0]) for c in cases], [c[1] for c in cases], [(c[2], c[3]) for c in cases],
                                         [c[4] for c in cases], th)
    for (KF, P, Tcw, Ow, K), g, t in zip(cases, got, np.broadcast_to(th, len(cases))):
        assert same(g, mt.SearchByProjectionSim3(KF, P, Tcw, Ow, K, int(t)))
        assert same(g, O.port_search_by_projection_sim3(KF, P, Tcw, Ow, K, int(t)))
    return got


def run_sim3(mt, O, cases, th=7.5, res=None):
    """cases = [(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K)] host views; res: resident copy per id(host view), shared across jobs."""
    res = {} if res is None else res
    for c in cases:
        for F in c[:2]:
            if id(F) not in res:
                res[id(F)] = resident(mt, F)
    got = mt.SearchBySim3Batch([res[id(c[0])] for c in cases], [res[id(c[1])] for c in cases], [c[2] for c in cases],
                               [c[3] for c in cases], [(c[4], c[5]) for c in cases], [(c[6], c[7]) for c in cases],
                               [c[8] for c in cases], th)
    for c, g, t in zip(cases, got, np.broadcast_to(th, len(cases))):
        assert same(g, mt.SearchBySim3(*c, float(t)))
        assert same(g, O.port_search_by_sim3(*c, float(t)))
    return got


# ---- equality
@pytest.mark.parametrize("n_jobs", [1, 3, 32])
@pytest.mark.parametrize("th,od,ori", RELOC)
def test_kf_batch_equals_the_single_call(M, oracle, views, n_jobs, th, od, ori):
    mt = M.ORBmatcher(0.9, ori)
    got = run_kf(mt, oracle, kf_cases(views, n_jobs, 30 + n_jobs), th, od)
    assert sum(g[0] for g in got) > 20 * n_jobs


def test_kf_batch_mixes_the_two_call_sites(M, oracle, views):
    mt = M.ORBmatcher(0.9, True)
    run_kf(mt, oracle, kf_cases(views, 6, 90), [10.0, 3.0] * 3, [100, 64] * 3)


@pytest.mark.parametrize("n_jobs", [1, 3, 32])
@pytest.mark.parametrize("th", [10, 3, 25])
def test_sim3_projection_batch_equals_the_single_call(M, oracle, views, n_jobs, th):
    mt = M.ORBmatcher(0.75, True)
    got = run_sim3proj(mt, oracle, kf_cases(views, n_jobs, 40 + n_jobs), th)
    assert sum(g[0] for g in got) > 10 * n_jobs


@pytest.mark.parametrize("n_jobs", [1, 3, 32])
@pytest.mark.parametrize("th", [7.5, 3.0, 15.0])
def test_sim3_batch_equals_the_single_call(M, oracle, views, n_jobs, th):
    mt = M.ORBmatcher(0.75, True)
    got = run_sim3(mt, oracle, sim3_cases(oracle, views, n_jobs, 60 + n_jobs), th)
    assert sum(g[0] for g in got) > 10 * n_jobs
    for (_, _, P1, P2, *_), (n, m12) in zip(sim3_cases(oracle, views, n_jobs, 60 + n_jobs), got):
        hit = np.nonzero(m12 >= 0)[0]
        assert n == len(hit) and np.all(P1.valid[hit] == 1) and np.all(P2.valid[m12[hit]] == 1)
        assert len(set(m12[hit].tolist())) == len(hit)


def test_batches_equal_the_verbatim_reference(M, oracle_ref, views):
    O = oracle_ref
    mt = M.ORBmatcher(0.9, True)
    for (Cur, P, Tcw, _, K), th, od in zip(kf_cases(views, 3, 130), (10.0, 3.0, 10.0), (100, 64, 100)):
        Ow = O.ref_camera_center(Tcw)                                   # -Rcw.t()*tcw as the reference evaluates it (:1478)
        n, s = mt.SearchByProjectionKFBatch([resident(mt, Cur)], [P], [(Tcw, Ow)], K, th, od)[0]
        n_r, owner = O.ref_search_by_projection_kf(Cur, P, Tcw, K, th, od, True)
        assert n == n_r and np.array_equal(owner, O.owner_from_state(Cur.occupied, s))
    for (KF, P, Tcw, _, K), scale in zip(kf_cases(views, 3, 140), (1.0, 1.7, 0.6)):
        Scw = (np.float32(scale) * np.asarray(Tcw, np.float32)).astype(np.float32)
        T, Ow = O.ref_decompose_scw(Scw)                                # :298-303 evaluated by the reference-side arithmetic
        n, s = mt.SearchByProjectionSim3Batch([resident(mt, KF)], [P], [(T, Ow)], K, 10)[0]
        n_r, owner = O.ref_search_by_projection_sim3(KF, P, Scw, K, 10)
        assert n == n_r and np.array_equal(owner, O.owner_from_state(KF.occupied, s))
    (s12, R12, t12), _ = sim3_mats(O)
    cases = sim3_cases(O, views, 3, 150)
    got = mt.SearchBySim3Batch([resident(mt, c[0]) for c in cases], [resident(mt, c[1]) for c in cases], [c[2] for c in cases],
                               [c[3] for c in cases], [(c[4], c[5]) for c in cases], [(c[6], c[7]) for c in cases], cases[0][8], 7.5)
    for c, g in zip(cases, got):
        KF1, KF2, P1, P2, T1w, T2w, _, _, K = c
        assert same(g, O.ref_search_by_sim3(KF1, KF2, P1, P2, T1w, T2w, s12, R12, t12, K, 7.5))


def test_extractor_frames_at_2000_features(M, oracle):
    """The real path: frames made by borb_frames_from_extractor (TUM-shaped 640x480, 2000 features) against the single calls on the
    extractor's host copies."""
    from orb_slam2_b200 import synth
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(2000)
    pairs = [synth.stereo_pair(300 + s, 0, 0, 640, 480) for s in range(3)]
    outs = X.extract_batch([p[0] for p in pairs] + [p[1] for p in pairs])
    mt = M.ORBmatcher(0.9, True)
    frames, host = M.frames_from_extractor(mt, X, list(range(6)), [len(o[0]) for o in outs], (517.3, 516.5, 318.6, 255.3), mode=0)
    b = tuple(float(x) for x in host["bounds"])
    sf = X.GetScaleFactors()
    kf_jobs, sp_jobs, s3_jobs = [], [], []
    _, (S12, S21) = sim3_mats(oracle)
    for s in range(3):
        assert len(outs[s][0]) > 1500
        v = dict(w=640, h=480, kl=host["keys_un"][s], dl=outs[s][1], kr=host["keys_un"][3 + s], dr=outs[3 + s][1], disp=pairs[s][2],
                 scale=sf)
        Cur, P, Tcw, Ow, K = mf.world_points_case(v, 200 + s)
        Cur = dataclasses.replace(Cur, bounds=b)
        kf_jobs.append((Cur, dataclasses.replace(Cur, resident=frames[s].resident), P, Tcw, Ow, K))
        KF1, KF2, P1, P2, T1w, T2w, _, _, K = mf.sim3_case(v, 210 + s)
        KF1, KF2 = dataclasses.replace(KF1, bounds=b), dataclasses.replace(KF2, bounds=b)
        s3_jobs.append(((KF1, KF2, P1, P2, T1w, T2w, S12, S21, K), frames[s], frames[3 + s]))
    got = mt.SearchByProjectionKFBatch([j[1] for j in kf_jobs], [j[2] for j in kf_jobs], [(j[3], j[4]) for j in kf_jobs], kf_jobs[0][5],
                                       10.0, 100)
    for j, g in zip(kf_jobs, got):
        assert same(g, mt.SearchByProjectionKF(j[0], j[2], j[3], j[4], j[5], 10.0, 100)) and g[0] > 20
    got = mt.SearchByProjectionSim3Batch([j[1] for j in kf_jobs], [j[2] for j in kf_jobs], [(j[3], j[4]) for j in kf_jobs], kf_jobs[0][5])
    for j, g in zip(kf_jobs, got):
        assert same(g, mt.SearchByProjectionSim3(j[0], j[2], j[3], j[4], j[5], 10)) and g[0] > 20
    got = mt.SearchBySim3Batch([j[1] for j in s3_jobs], [j[2] for j in s3_jobs], [j[0][2] for j in s3_jobs], [j[0][3] for j in s3_jobs],
                               [(j[0][4], j[0][5]) for j in s3_jobs], [(S12, S21)] * 3, s3_jobs[0][0][8], 7.5)
    for j, g in zip(s3_jobs, got):
        assert same(g, mt.SearchBySim3(*j[0], 7.5)) and g[0] > 20


# ---- SearchBySim3 specifics
def test_sim3_shared_and_identical_keyframes(M, oracle, views):
    """kf1 == kf2 (each keyframe against itself with the identity similarity) and one keyframe in several jobs."""
    mt = M.ORBmatcher(0.75, True)
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = sim3_cases(oracle, views, 1, 70)[0]
    I12, I21 = oracle.ref_sim3_mats(1.0, np.eye(3, dtype=np.float32), np.zeros(3, np.float32))
    G1, G2, Q1, Q2, U1w, U2w, _, _, _ = sim3_cases(oracle, views, 2, 70)[1]
    cases = [(KF1, KF1, P1, P1, T1w, T1w, I12, I21, K), (KF1, KF2, P1, P2, T1w, T2w, S12, S21, K), (KF2, KF2, P2, P2, T2w, T2w, I12, I21, K),
             (KF1, G2, P1, Q2, T1w, U2w, S12, S21, K), (G1, KF2, Q1, P2, U1w, T2w, S12, S21, K), (KF1, KF2, P1, P2, T1w, T2w, S12, S21, K)]
    got = run_sim3(mt, oracle, cases)
    assert got[0][0] > 0.5 * int(P1.valid.sum()) and same(got[1], got[5])


def test_sim3_valid_masks(M, oracle, views):
    """Points already matched by the RANSAC inliers (vbAlreadyMatched) and bad points enter through pts*.valid."""
    mt = M.ORBmatcher(0.75, True)
    base = sim3_cases(oracle, views, 2, 80)
    rng = np.random.default_rng(5)
    cases = []
    for KF1, KF2, P1, P2, *rest in base:
        for frac in (0.0, 0.5, 1.0):
            V1 = dataclasses.replace(P1, valid=(P1.valid * (rng.random(len(P1.valid)) >= frac)).astype(np.uint8))
            V2 = dataclasses.replace(P2, valid=(P2.valid * (rng.random(len(P2.valid)) >= frac / 2)).astype(np.uint8))
            cases.append((KF1, KF2, V1, V2, *rest))
    got = run_sim3(mt, oracle, cases)
    assert got[0][0] > got[1][0] > 0 and got[2][0] == 0


def test_sim3_agreement_drops_matches(M, oracle, views):
    """KF1 doubled (every feature and its MapPoint listed twice): each copy's forward search finds the same KF2 feature as the
    original, but the reverse search sends that feature back to the first copy only (the first minimum, lower index, wins the tie),
    so the agreement test drops every second copy that matched on its own."""
    mt = M.ORBmatcher(0.75, True)
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = sim3_cases(oracle, views, 1, 90)[0]
    n1 = len(KF1.mvKeysUn)
    D1 = dataclasses.replace(KF1, mvKeysUn=np.concatenate([KF1.mvKeysUn] * 2), mDescriptors=np.concatenate([KF1.mDescriptors] * 2))
    Q1 = dataclasses.replace(P1, **{f: np.concatenate([getattr(P1, f)] * 2) for f in ("world_pos", "descriptors", "max_distance",
                                                                                      "min_distance", "valid")})
    got = run_sim3(mt, oracle, [(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K), (D1, KF2, Q1, P2, T1w, T2w, S12, S21, K)])
    (n_a, m_a), (n_b, m_b) = got
    assert n_a > 20
    assert np.array_equal(m_b[:n1], m_a) and np.all(m_b[n1:] == -1) and n_b == n_a


def test_sim3_tied_distances_take_the_first_minimum(M, oracle):
    """The tied_sim3 envelope case (duplicated descriptors at several positions) through the batch."""
    mt = M.ORBmatcher(0.75, True)
    c = E.case(oracle, "tied_sim3")
    case = (c["KF1"], c["KF2"], c["P1"], c["P2"], c["T1w"], c["T2w"], c["S12"], c["S21"], c["K"])
    got = run_sim3(mt, oracle, [case, case], c["th"])
    assert got[0][0] > 0 and same(got[0], got[1])


# ---- envelope
def random_keyframes(M, oracle, seed, n):
    """Two n-feature keyframes seeing one scene from cameras 0.2 apart, every feature with a MapPoint, and the world points of the
    second keyframe as a relocalisation / Sim3-projection query of the first."""
    from orb_slam2_b200._lib import KP_DTYPE
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = K = (525.0, 525.0, 319.5, 239.5)
    sc = (1.2 ** np.arange(8)).astype(np.float32)
    k1 = np.zeros(n, KP_DTYPE)
    k1["x"] = rng.uniform(0, 640, n); k1["y"] = rng.uniform(0, 480, n)
    k1["angle"] = rng.uniform(0, 360, n); k1["size"] = 31.0; k1["class_id"] = -1
    k1["octave"] = rng.integers(0, 8, n)
    z = rng.uniform(2.0, 20.0, n)
    Pw = np.stack([(k1["x"] - cx) * z / fx, (k1["y"] - cy) * z / fy, z], 1)
    t2 = np.array([-0.2, 0.0, 0.0])
    p2 = Pw + t2
    k2 = k1.copy()
    k2["x"] = p2[:, 0] / p2[:, 2] * fx + cx + rng.normal(0, 0.5, n); k2["y"] = p2[:, 1] / p2[:, 2] * fy + cy + rng.normal(0, 0.5, n)
    keep = (k2["x"] >= 0) & (k2["x"] < 640) & (k2["y"] >= 0) & (k2["y"] < 480)
    k2["x"][~keep] = rng.uniform(0, 640, (~keep).sum())
    d1 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    d2 = d1 ^ np.packbits(rng.random((n, 32, 8)) < 0.05, axis=2, bitorder="little").reshape(n, 32)
    perm = rng.permutation(n)
    k2, d2, p2w = k2[perm], d2[perm], Pw[perm]

    def points(Pw_, k, d, cam_t):
        dist = np.linalg.norm(Pw_ + cam_t, axis=1)
        maxd = (dist * sc[k["octave"]] * rng.uniform(0.95, 1.05, len(k))).astype(np.float32)
        view = Pw_ + cam_t
        return M.WorldPointsView(world_pos=Pw_.astype(np.float32), descriptors=d, max_distance=maxd, min_distance=(maxd / sc[-1] / 2).astype(np.float32),
                                 normal=(view / dist[:, None]).astype(np.float32), angle=k["angle"].astype(np.float32),
                                 valid=(rng.random(len(k)) < 0.95).astype(np.uint8))
    b = (0.0, 0.0, 640.0, 480.0)
    KF1 = M.FrameView(k1, d1, sc, b, occupied=(rng.random(n) < 0.05).astype(np.uint8))
    KF2 = M.FrameView(k2, d2, sc, b)
    P1, P2 = points(Pw, k1, d1, np.zeros(3)), points(p2w, k2, d2, t2)
    T1w = np.eye(4, dtype=np.float32)[:3]
    T2w = T1w.copy(); T2w[:, 3] = t2
    S12, S21 = oracle.ref_sim3_mats(1.0, np.eye(3, dtype=np.float32), (-t2).astype(np.float32))
    return KF1, KF2, P1, P2, T1w, T2w, S12, S21, K


def test_8192_feature_keyframes_and_8192_points(M, oracle):
    mt = M.ORBmatcher(0.9, True)
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = random_keyframes(M, oracle, 11, 8192)
    Ow = np.zeros(3, np.float32)
    kf = run_kf(mt, oracle, [(KF1, P2, T1w, Ow, K)] * 2, [10.0, 3.0], [100, 64])
    sp = run_sim3proj(mt, oracle, [(KF1, P2, T1w, Ow, K)], 10)
    s3 = run_sim3(mt, oracle, [(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K), (KF2, KF1, P2, P1, T2w, T1w, S21, S12, K)])
    assert kf[0][0] > 1000 and sp[0][0] > 1000 and s3[0][0] > 1000 and s3[1][0] > 1000


def test_empty_jobs(M, oracle, views):
    """0 features, 0 points and all points invalid next to live jobs: the single call's defaults (-1 everywhere, 0 matches)."""
    mt = M.ORBmatcher(0.9, True)
    Cur, P, Tcw, Ow, K = kf_cases(views, 1, 100)[0]
    E0 = dataclasses.replace(Cur, mvKeysUn=Cur.mvKeysUn[:0], mDescriptors=Cur.mDescriptors[:0], occupied=None)
    P0 = M.WorldPointsView(*[np.zeros((0, 3) if f in ("world_pos", "normal") else (0, 32) if f == "descriptors" else 0,
                                      np.uint8 if f in ("descriptors", "valid") else np.float32)
                             for f in ("world_pos", "descriptors", "max_distance", "min_distance", "normal", "angle", "valid")])
    Pn = dataclasses.replace(P, valid=np.zeros(len(P.valid), np.uint8))
    live = (Cur, P, Tcw, Ow, K)
    jobs = [live, (E0, P, Tcw, Ow, K), (Cur, P0, Tcw, Ow, K), (Cur, Pn, Tcw, Ow, K), live]
    for got in (run_kf(mt, oracle, jobs, 10.0, 100), run_sim3proj(mt, oracle, jobs, 10)):
        assert got[0][0] > 0 and same(got[0], got[4])
        assert all(g[0] == 0 and np.all(g[1] == -1) for g in got[1:4])
        assert len(got[1][1]) == 0 and len(got[2][1]) == len(Cur.mvKeysUn)
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = sim3_cases(oracle, views, 1, 100)[0]
    F0 = dataclasses.replace(KF2, mvKeysUn=KF2.mvKeysUn[:0], mDescriptors=KF2.mDescriptors[:0])
    Q2 = dataclasses.replace(P2, **{f: getattr(P2, f)[:0] for f in ("world_pos", "descriptors", "max_distance", "min_distance", "valid")})
    N1 = dataclasses.replace(P1, valid=np.zeros(len(P1.valid), np.uint8))
    live = (KF1, KF2, P1, P2, T1w, T2w, S12, S21, K)
    got = run_sim3(mt, oracle, [live, (KF1, F0, P1, Q2, T1w, T2w, S12, S21, K), (F0, KF2, Q2, P2, T1w, T2w, S12, S21, K),
                                (KF1, KF2, N1, P2, T1w, T2w, S12, S21, K), live])
    assert got[0][0] > 0 and same(got[0], got[4])
    assert all(g[0] == 0 and np.all(g[1] == -1) for g in got[1:4])
    assert len(got[1][1]) == len(KF1.mvKeysUn) and len(got[2][1]) == 0


def test_no_jobs(M):
    mt = M.ORBmatcher(0.9, True)
    c0 = launches(mt)
    assert mt.SearchByProjectionKFBatch([], [], [], (1.0, 1.0, 0.0, 0.0), 10.0, 100) == []
    assert mt.SearchByProjectionSim3Batch([], [], [], (1.0, 1.0, 0.0, 0.0), 10) == []
    assert mt.SearchBySim3Batch([], [], [], [], [], [], (1.0, 1.0, 0.0, 0.0), 7.5) == []
    assert launches(mt) == c0


def test_launch_count_does_not_depend_on_the_batch(M, oracle, views):
    mt = M.ORBmatcher(0.9, True)
    kc = kf_cases(views, 32, 110)
    kr = [resident(mt, c[0]) for c in kc]
    sc = sim3_cases(oracle, views, 32, 120)
    s1, s2 = [resident(mt, c[0]) for c in sc], [resident(mt, c[1]) for c in sc]
    counts = []
    for n in (1, 8, 32):
        row = []
        c0 = launches(mt)
        mt.SearchByProjectionKFBatch(kr[:n], [c[1] for c in kc[:n]], [(c[2], c[3]) for c in kc[:n]], kc[0][4], 10.0, 100)
        row.append(launches(mt) - c0)
        c0 = launches(mt)
        mt.SearchByProjectionSim3Batch(kr[:n], [c[1] for c in kc[:n]], [(c[2], c[3]) for c in kc[:n]], kc[0][4], 10)
        row.append(launches(mt) - c0)
        c0 = launches(mt)
        mt.SearchBySim3Batch(s1[:n], s2[:n], [c[2] for c in sc[:n]], [c[3] for c in sc[:n]], [(c[4], c[5]) for c in sc[:n]],
                             [(c[6], c[7]) for c in sc[:n]], sc[0][8], 7.5)
        row.append(launches(mt) - c0)
        counts.append(row)
    assert counts == [[3, 3, 3]] * 3


def test_argument_errors_name_the_job_and_launch_nothing(M, oracle, views):
    from orb_slam2_b200._lib import BorbError, check
    from orb_slam2_b200.matcher import _KfProjectionJobC, _Sim3JobC, _Sim3ProjectionJobC
    mt = M.ORBmatcher(0.9, True)
    Cur, P, Tcw, Ow, K = kf_cases(views, 1, 160)[0]
    R = resident(mt, Cur)
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, _ = sim3_cases(oracle, views, 1, 160)[0]
    R1, R2 = resident(mt, KF1), resident(mt, KF2)

    def refused(call, job):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        assert ei.value.status == 1 and str(ei.value).split(": ", 2)[2].startswith(f"job {job}:"), str(ei.value)
        assert launches(mt) == c0

    # host views
    refused(lambda: mt.SearchByProjectionKFBatch([R, Cur], [P, P], [(Tcw, Ow)] * 2, K, 10.0, 100), 1)
    refused(lambda: mt.SearchByProjectionSim3Batch([R, R, Cur], [P] * 3, [(Tcw, Ow)] * 3, K, 10), 2)
    refused(lambda: mt.SearchBySim3Batch([R1, R1], [R2, KF2], [P1] * 2, [P2] * 2, [(T1w, T2w)] * 2, [(S12, S21)] * 2, K, 7.5), 1)
    refused(lambda: mt.SearchBySim3Batch([KF1], [R2], [P1], [P2], [(T1w, T2w)], [(S12, S21)], K, 7.5), 0)
    # pts.n different from the keyframe's n (SearchBySim3: one slot per feature)
    short = dataclasses.replace(P2, **{f: getattr(P2, f)[:-1] for f in ("world_pos", "descriptors", "max_distance", "min_distance", "valid")})
    refused(lambda: mt.SearchBySim3Batch([R1, R1], [R2, R2], [P1] * 2, [P2, short], [(T1w, T2w)] * 2, [(S12, S21)] * 2, K, 7.5), 1)
    # more than BORB_MATCH_MAX_FEATURES query points
    big = M.WorldPointsView(*[np.zeros((8193, 3), np.float32), np.zeros((8193, 32), np.uint8)] + [np.ones(8193, np.float32)] * 2 +
                            [np.zeros((8193, 3), np.float32), np.zeros(8193, np.float32)])
    refused(lambda: mt.SearchByProjectionKFBatch([R, R], [P, big], [(Tcw, Ow)] * 2, K, 10.0, 100), 1)
    refused(lambda: mt.SearchByProjectionSim3Batch([R, R], [big, P], [(Tcw, Ow)] * 2, K, 10), 0)

    # the raw tables: log_scale_factor <= 0, incomplete points views, NULL outputs
    def raw(fn, cls, fill, n=2, mutate=lambda J: None):
        J = (cls * n)()
        keep = [fill(J[j]) for j in range(n)]
        mutate(J)
        out = np.zeros(n, np.int32)
        args = (mt._h, J, n, 1, out.ctypes.data) if fn == "borb_search_by_projection_kf_batch" else (mt._h, J, n, out.ctypes.data)
        check(getattr(mt._lib, fn)(*args), fn)
        return keep

    fv, pv, logs, n_cur, keep = mt._points_call(R, P)
    state = np.zeros(n_cur, np.int32)

    def fill_kf(J):
        J.cur, J.pts, J.Tcw, J.Ow = fv, pv, M._pose12(Tcw), M._vec3(Ow)
        J.fx, J.fy, J.cx, J.cy = K
        J.log_scale_factor, J.th, J.orb_dist, J.state_cur = logs, 10.0, 100, state.ctypes.data

    def fill_sp(J):
        J.kf, J.pts, J.Tcw, J.Ow = fv, pv, M._pose12(Tcw), M._vec3(Ow)
        J.fx, J.fy, J.cx, J.cy = K
        J.log_scale_factor, J.th, J.state_kf = logs, 10, state.ctypes.data

    f1, p1, l1, n1, k1 = mt._points_call(R1, P1)
    f2, p2, l2, _, k2 = mt._points_call(R2, P2)
    m12 = np.zeros(n1, np.int32)

    def fill_s3(J):
        J.kf1, J.kf2, J.pts1, J.pts2 = f1, f2, p1, p2
        J.T1w, J.T2w, J.S12, J.S21 = M._pose12(T1w), M._pose12(T2w), M._pose12(S12), M._pose12(S21)
        J.fx, J.fy, J.cx, J.cy = K
        J.log_scale_factor1, J.log_scale_factor2, J.th, J.match12 = l1, l2, 7.5, m12.ctypes.data

    for fn, cls, fill, out in (("borb_search_by_projection_kf_batch", _KfProjectionJobC, fill_kf, "state_cur"),
                               ("borb_search_by_projection_sim3_batch", _Sim3ProjectionJobC, fill_sp, "state_kf")):
        raw(fn, cls, fill)                                              # the well-formed table runs
        refused(lambda: raw(fn, cls, fill, mutate=lambda J: setattr(J[1], "log_scale_factor", 0.0)), 1)
        refused(lambda: raw(fn, cls, fill, mutate=lambda J: setattr(J[0].pts, "max_distance", None)), 0)
        refused(lambda: raw(fn, cls, fill, mutate=lambda J: setattr(J[1].pts, "desc", None)), 1)
        refused(lambda: raw(fn, cls, fill, mutate=lambda J: setattr(J[1], out, None)), 1)
    raw("borb_search_by_sim3_batch", _Sim3JobC, fill_s3)
    refused(lambda: raw("borb_search_by_sim3_batch", _Sim3JobC, fill_s3, mutate=lambda J: setattr(J[1], "log_scale_factor2", -1.0)), 1)
    refused(lambda: raw("borb_search_by_sim3_batch", _Sim3JobC, fill_s3, mutate=lambda J: setattr(J[0], "log_scale_factor1", 0.0)), 0)
    refused(lambda: raw("borb_search_by_sim3_batch", _Sim3JobC, fill_s3, mutate=lambda J: setattr(J[1].pts2, "min_distance", None)), 1)
    refused(lambda: raw("borb_search_by_sim3_batch", _Sim3JobC, fill_s3, mutate=lambda J: setattr(J[0].pts1, "world_pos", None)), 0)
    refused(lambda: raw("borb_search_by_sim3_batch", _Sim3JobC, fill_s3, mutate=lambda J: setattr(J[1], "match12", None)), 1)
