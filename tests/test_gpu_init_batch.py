"""GPU parity of borb_search_for_initialization_batch: SearchForInitialization (src/ORBmatcher.cc:405-520) of many camera streams on
resident frames.  Every job must equal the oracle restatement and the single call on host views of the same frames bit for bit;
the batch is two launches whatever its size, and argument errors are refused before anything is launched."""
import ctypes as C

import numpy as np
import pytest

from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu

SETTINGS = [(100, 0.9, True), (30, 0.9, True), (100, 0.7, False), (10, 0.9, True)]
BOUNDS = (0.0, 0.0, 640.0, 480.0)


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def views(oracle):
    return {s: mf.two_views(oracle, s) for s in (7, 8, 9)}


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def host_views(M, v):
    b = (0.0, 0.0, float(v["w"]), float(v["h"]))
    return M.FrameView(v["kl"], v["dl"], v["scale"], b), M.FrameView(v["kr"], v["dr"], v["scale"], b)


def jobs_from_views(M, mt, views, n_jobs, seed):
    """n_jobs (F1, F2, prev) host-view jobs cycling through the views, each with its own jitter of the window centres, and the
    resident frames of every view."""
    rng = np.random.default_rng(seed)
    res = {s: tuple(F.make_resident(mt) for F in host_views(M, v)) for s, v in views.items()}
    keys = sorted(views)
    out = []
    for j in range(n_jobs):
        s = keys[j % len(keys)]
        F1, F2 = host_views(M, views[s])
        kl = views[s]["kl"]
        prev = (np.stack([kl["x"], kl["y"]], 1) + rng.normal(0, 3.0 * (j % 4), (len(kl), 2))).astype(np.float32)
        out.append((F1, F2, res[s][0], res[s][1], prev))
    return out, res


def check_batch(M, mt, oracle, jobs, window, ratio, ori):
    got = mt.SearchForInitializationBatch([j[2] for j in jobs], [j[3] for j in jobs], [j[4] for j in jobs], window)
    for (F1, F2, _, _, prev), g in zip(jobs, got):
        one = mt.SearchForInitialization(F1, F2, prev, window)
        o = oracle.port_search_for_initialization(F1, F2, prev, window, ratio, ori)
        assert same(g, one) and same(g, o)
    return got


@pytest.mark.parametrize("n_jobs", [1, 3, 32])
@pytest.mark.parametrize("window,ratio,ori", SETTINGS)
def test_batch_equals_the_single_call(M, oracle, views, n_jobs, window, ratio, ori):
    mt = M.ORBmatcher(ratio, ori)
    jobs, _ = jobs_from_views(M, mt, views, n_jobs, n_jobs * 7 + window)
    got = check_batch(M, mt, oracle, jobs, window, ratio, ori)
    assert sum(g[0] for g in got) > 10 * n_jobs or window < 30


def test_batch_equals_the_verbatim_reference(M, oracle_ref, views):
    mt = M.ORBmatcher(0.9, True)
    jobs, _ = jobs_from_views(M, mt, views, 3, 5)
    got = mt.SearchForInitializationBatch([j[2] for j in jobs], [j[3] for j in jobs], [j[4] for j in jobs], 100)
    for (F1, F2, _, _, prev), g in zip(jobs, got):
        assert same(g, oracle_ref.ref_search_for_initialization(F1, F2, prev, 100, 0.9, True))


def test_two_rounds_follow_the_tracker(M, oracle, views):
    """Round 1's vbPrevMatched feeds round 2 with a smaller window, as on the tracker's next frame."""
    mt = M.ORBmatcher(0.9, True)
    jobs, _ = jobs_from_views(M, mt, views, 6, 11)
    r1 = mt.SearchForInitializationBatch([j[2] for j in jobs], [j[3] for j in jobs], [j[4] for j in jobs], 100)
    r2 = mt.SearchForInitializationBatch([j[2] for j in jobs], [j[3] for j in jobs], [g[2] for g in r1], [50, 50, 20, 20, 5, 5])
    for (F1, F2, _, _, prev), g1, g2, w in zip(jobs, r1, r2, [50, 50, 20, 20, 5, 5]):
        s1 = mt.SearchForInitialization(F1, F2, prev, 100)
        s2 = mt.SearchForInitialization(F1, F2, s1[2], w)
        o1 = oracle.port_search_for_initialization(F1, F2, prev, 100, 0.9, True)
        o2 = oracle.port_search_for_initialization(F1, F2, o1[2], w, 0.9, True)
        assert same(g1, s1) and same(g2, s2)
        assert same(g1, o1) and same(g2, o2)


def test_extractor_frames_at_2000_features(M, oracle):
    """The real path: frames made by borb_frames_from_extractor (mono) against the single call on the extractor's host copies
    and the oracle port."""
    from orb_slam2_b200 import synth
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(2000)
    pairs = [synth.stereo_pair(300, s, 0, 640, 480) for s in range(4)]
    outs = X.extract_batch([p[0] for p in pairs] + [p[1] for p in pairs])
    mt = M.ORBmatcher(0.9, True)
    frames, host = M.frames_from_extractor(mt, X, list(range(8)), [len(o[0]) for o in outs], (517.3, 516.5, 318.6, 255.3), mode=0)
    b = tuple(float(x) for x in host["bounds"])
    sf = X.GetScaleFactors()
    prevs = [np.stack([k["x"], k["y"]], 1).astype(np.float32) for k in host["keys_un"][:4]]
    got = mt.SearchForInitializationBatch(frames[:4], frames[4:], prevs, 100)
    for s in range(4):
        assert len(outs[s][0]) > 1500
        F1 = M.FrameView(host["keys_un"][s], outs[s][1], sf, b)
        F2 = M.FrameView(host["keys_un"][4 + s], outs[4 + s][1], sf, b)
        assert same(got[s], mt.SearchForInitialization(F1, F2, prevs[s], 100))
        assert same(got[s], oracle.port_search_for_initialization(F1, F2, prevs[s], 100, 0.9, True))
        assert got[s][0] > 50


# ---- the prefix fallback: queries whose INIT_K best window entries hold fewer than two that are not excluded
INIT_K = 8                                                               # csrc/borb_match.h
def _grid_order(keys, bounds):
    """Position of every feature in its GetFeaturesInArea walk order: (cell x, cell y, insertion)."""
    minx, miny, maxx, maxy = [np.float32(v) for v in bounds]
    iw, ih = np.float32(64) / (maxx - minx), np.float32(48) / (maxy - miny)
    cx = np.round((keys["x"] - minx) * iw).astype(np.int64)
    cy = np.round((keys["y"] - miny) * ih).astype(np.int64)
    return cx * 48 * 100000 + cy * 100000 + np.arange(len(keys))


def fallback_queries(F1, F2, prev, window, ratio, ori, K=INIT_K):
    """Replays the reference's exclusion state in NumPy; returns the queries whose K smallest (dist, walk order) window entries
    hold fewer than two that are not excluded while the window holds more than K."""
    d = np.unpackbits(F1.mDescriptors[:, None, :] ^ F2.mDescriptors[None, :, :], axis=2).sum(2)
    order = _grid_order(F2.mvKeysUn, F2.bounds)
    k2 = F2.mvKeysUn
    matched = np.full(len(k2), 1 << 30)
    hits = []
    for i1 in range(len(F1.mvKeysUn)):
        if F1.mvKeysUn["octave"][i1] > 0:
            continue
        x, y = prev[i1]
        win = np.nonzero((k2["octave"] == 0) & (np.abs(k2["x"] - x) < window) & (np.abs(k2["y"] - y) < window))[0]
        if len(win) == 0:
            continue
        win = win[np.lexsort((order[win], d[i1, win]))]
        open_ = [i2 for i2 in win if matched[i2] > d[i1, i2]]
        if len(win) > K and sum(matched[i2] > d[i1, i2] for i2 in win[:K]) < 2:
            hits.append(i1)
        if not open_:
            continue
        best = d[i1, open_[0]]
        second = d[i1, open_[1]] if len(open_) > 1 else 2 ** 31
        if best <= 50 and best < np.float32(second) * np.float32(ratio):
            matched[open_[0]] = best
    return hits


def fallback_case(M, seed):
    from orb_slam2_b200._lib import KP_DTYPE
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, 32, dtype=np.uint8)

    def flip(d, bits):
        d = d.copy()
        for b in bits:
            d[b // 8] ^= np.uint8(1 << (b % 8))
        return d
    # F2: D0..D7 = base with 8 own bits flipped (8 from base, 16 from each other), D8 = base with 10 others, then random features
    K = INIT_K
    near = [flip(base, range(8 * k, 8 * k + 8)) for k in range(K)] + [flip(base, range(8 * K, 8 * K + 10))]
    n_far = 300
    d2 = np.concatenate([np.stack(near), rng.integers(0, 256, (n_far, 32), dtype=np.uint8)])
    k2 = np.zeros(len(d2), KP_DTYPE)
    k2["x"][:K + 1] = 300 + 7 * np.arange(K + 1); k2["y"][:K + 1] = 240 - 5 * np.arange(K + 1)
    k2["x"][K + 1:] = rng.uniform(5, 635, n_far); k2["y"][K + 1:] = rng.uniform(5, 475, n_far)
    k2["angle"] = rng.uniform(0, 360, len(d2)); k2["size"] = 31.0; k2["class_id"] = -1
    k2["octave"][K + 1:] = rng.integers(0, 3, n_far)
    # F1: exact copies of D0..D6 take them at distance 0; the query `base` then sees D0..D6 excluded and D7 open (one open entry
    # of eight: the second comes from outside the prefix); a second `base` sees all eight excluded and takes D8
    n_rand = 200
    d1 = np.concatenate([np.stack(near[:K - 1] + [base, base]), rng.integers(0, 256, (n_rand, 32), dtype=np.uint8)])
    k1 = np.zeros(len(d1), KP_DTYPE)
    k1["x"] = rng.uniform(5, 635, len(d1)); k1["y"] = rng.uniform(5, 475, len(d1))
    k1["angle"] = rng.uniform(0, 360, len(d1)); k1["size"] = 31.0; k1["class_id"] = -1
    k1["octave"][K + 1:] = rng.integers(0, 2, n_rand)
    k1["angle"][:K + 1] = k2["angle"][:K + 1] + 1.0
    prev = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    prev[:K + 1] = (310.0, 235.0)
    sc = (1.2 ** np.arange(8)).astype(np.float32)
    return M.FrameView(k1, d1, sc, BOUNDS), M.FrameView(k2, d2, sc, BOUNDS), prev


@pytest.mark.parametrize("ori", [True, False])
def test_prefix_fallback(M, oracle, ori):
    mt = M.ORBmatcher(0.9, ori)
    cases = [fallback_case(M, s) for s in (1, 2, 3)]
    for F1, F2, prev in cases:
        hits = fallback_queries(F1, F2, prev, 100, 0.9, ori)
        assert INIT_K - 1 in hits and INIT_K in hits, hits
    R = [(F1.make_resident(mt), F2.make_resident(mt)) for F1, F2, _ in cases]
    got = mt.SearchForInitializationBatch([r[0] for r in R], [r[1] for r in R], [c[2] for c in cases], 100)
    for (F1, F2, prev), g in zip(cases, got):
        assert same(g, mt.SearchForInitialization(F1, F2, prev, 100))
        assert same(g, oracle.port_search_for_initialization(F1, F2, prev, 100, 0.9, ori))
        assert g[1][INIT_K - 1] == INIT_K - 1 and g[1][INIT_K] == INIT_K     # both took their feature through the fallback


# ---- envelope
def random_frames(M, seed, n, shift=(12.0, -3.0), level0=0.3):
    """An n-feature frame and its moved copy: descriptors with a few bits flipped, a quarter of the features elsewhere."""
    from orb_slam2_b200._lib import KP_DTYPE
    rng = np.random.default_rng(seed)
    k1 = np.zeros(n, KP_DTYPE)
    k1["x"] = rng.uniform(0, 640, n); k1["y"] = rng.uniform(0, 480, n)
    k1["angle"] = rng.uniform(0, 360, n); k1["size"] = 31.0; k1["class_id"] = -1
    k1["octave"] = np.where(rng.random(n) < level0, 0, rng.integers(1, 8, n))
    d1 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    k2 = k1.copy()
    k2["x"] = np.clip(k1["x"] + shift[0] + rng.normal(0, 1, n), 0, 639.9); k2["y"] = np.clip(k1["y"] + shift[1] + rng.normal(0, 1, n), 0, 479.9)
    k2["angle"] = (k1["angle"] + rng.normal(0, 4, n)) % 360
    move = rng.random(n) < 0.25
    k2["x"][move] = rng.uniform(0, 640, move.sum())
    d2 = d1 ^ np.packbits(rng.random((n, 32, 8)) < 0.05, axis=2, bitorder="little").reshape(n, 32)
    perm = rng.permutation(n)
    sc = (1.2 ** np.arange(8)).astype(np.float32)
    return M.FrameView(k1, d1, sc, BOUNDS), M.FrameView(k2[perm], d2[perm], sc, BOUNDS)


def run_jobs(M, mt, oracle, jobs, ratio, ori):
    """jobs = [(F1, F2, prev, window)] as host views: the batch on their resident copies equals the single call and the port."""
    res = {}
    for F1, F2, _, _ in jobs:
        for F in (F1, F2):
            if id(F) not in res:
                res[id(F)] = F.make_resident(mt)
    got = mt.SearchForInitializationBatch([res[id(j[0])] for j in jobs], [res[id(j[1])] for j in jobs], [j[2] for j in jobs],
                                          [j[3] for j in jobs])
    for (F1, F2, prev, w), g in zip(jobs, got):
        assert same(g, mt.SearchForInitialization(F1, F2, prev, w))
        assert same(g, oracle.port_search_for_initialization(F1, F2, prev, w, ratio, ori))
    return got


def test_8192_feature_frames(M, oracle):
    mt = M.ORBmatcher(0.9, True)
    jobs = []
    for s in range(3):
        F1, F2 = random_frames(M, 40 + s, 8192)
        prev = np.stack([F1.mvKeysUn["x"], F1.mvKeysUn["y"]], 1).astype(np.float32)
        jobs.append((F1, F2, prev, 100 if s else 30))
    got = run_jobs(M, mt, oracle, jobs, 0.9, True)
    assert all(g[0] > 200 for g in got)


def test_window_sizes_and_centres_outside_the_image(M, oracle, views):
    mt = M.ORBmatcher(0.9, True)
    F1, F2 = host_views(M, views[7])
    kl = views[7]["kl"]
    prev = np.stack([kl["x"], kl["y"]], 1).astype(np.float32)
    rng = np.random.default_rng(3)
    out = prev.copy()
    out[::3] = rng.choice([-80.0, -5.0, 660.0, 700.0, 2000.0], (len(out[::3]), 2))   # centres left of, right of and far off the image
    out[1::7, 1] = -40.0
    jobs = [(F1, F2, prev, 0), (F1, F2, prev, 1), (F1, F2, prev, 1000), (F1, F2, out, 100), (F1, F2, out, 40)]
    got = run_jobs(M, mt, oracle, jobs, 0.9, True)
    assert got[0][0] == 0 and np.all(got[0][1] == -1) and np.array_equal(got[0][2], prev)
    assert got[2][0] > 0 and got[3][0] > 0


def test_frames_without_level0_or_without_features(M, oracle, views):
    mt = M.ORBmatcher(0.9, True)
    F1, F2 = host_views(M, views[8])
    kl = views[8]["kl"].copy()
    prev = np.stack([kl["x"], kl["y"]], 1).astype(np.float32)
    kl["octave"] = np.maximum(kl["octave"], 1)
    F1up = M.FrameView(kl, F1.mDescriptors, F1.mvScaleFactors, F1.bounds)
    E = M.FrameView(kl[:0], F1.mDescriptors[:0], F1.mvScaleFactors, F1.bounds)
    live = (F1, F2, prev, 100)
    jobs = [live, (F1up, F2, prev, 100), (E, F2, prev[:0], 100), live, (F1, E, prev, 100), (E, E, prev[:0], 100), live]
    got = run_jobs(M, mt, oracle, jobs, 0.9, True)
    assert got[1][0] == 0 and np.all(got[1][1] == -1) and np.array_equal(got[1][2], prev)
    assert got[2][0] == 0 and len(got[2][1]) == 0
    assert got[4][0] == 0 and np.all(got[4][1] == -1) and np.array_equal(got[4][2], prev)
    assert got[0][0] > 20 and same(got[0], got[3]) and same(got[0], got[6])


def test_shared_and_identical_frames(M, oracle, views):
    """One initial frame against several current frames, and initial == current."""
    mt = M.ORBmatcher(0.9, True)
    F1, F2 = host_views(M, views[7])
    G1, G2 = host_views(M, views[9])
    kl = views[7]["kl"]
    prev = np.stack([kl["x"], kl["y"]], 1).astype(np.float32)
    prev2 = np.stack([F2.mvKeysUn["x"], F2.mvKeysUn["y"]], 1).astype(np.float32)
    jobs = [(F1, F2, prev, 100), (F1, F1, prev, 100), (F1, G2, prev, 100), (F1, G1, prev, 30), (F2, F2, prev2, 10)]
    got = run_jobs(M, mt, oracle, jobs, 0.9, True)
    lvl0 = np.nonzero(kl["octave"] == 0)[0]
    assert got[1][0] > 0.8 * len(lvl0)                                  # a frame against itself matches most of its level 0


def test_no_jobs(M):
    mt = M.ORBmatcher(0.9, True)
    c0 = launches(mt)
    assert mt.SearchForInitializationBatch([], [], [], 100) == []
    assert launches(mt) == c0


def test_launch_count_does_not_depend_on_the_batch(M, views):
    mt = M.ORBmatcher(0.9, True)
    jobs, _ = jobs_from_views(M, mt, views, 32, 2)
    counts = []
    for n in (1, 8, 32):
        c0 = launches(mt)
        mt.SearchForInitializationBatch([j[2] for j in jobs[:n]], [j[3] for j in jobs[:n]], [j[4] for j in jobs[:n]], 100)
        counts.append(launches(mt) - c0)
    assert counts == [2, 2, 2]


def test_argument_errors_name_the_job_and_launch_nothing(M, views):
    from orb_slam2_b200._lib import BorbError
    from orb_slam2_b200.matcher import _InitJobC
    mt = M.ORBmatcher(0.9, True)
    jobs, _ = jobs_from_views(M, mt, views, 3, 4)
    R1, R2, prev = jobs[0][2], jobs[0][3], jobs[0][4]
    lib = mt._lib

    def refused(call, job):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        assert ei.value.status == 1 and str(ei.value).split(": ", 2)[2].startswith(f"job {job}:"), str(ei.value)
        assert launches(mt) == c0

    # a NULL frame (a host view has no resident frame)
    refused(lambda: mt.SearchForInitializationBatch([R1, jobs[1][0]], [R2, R2], [prev, prev], 100), 1)
    refused(lambda: mt.SearchForInitializationBatch([R1, R1, R1], [R2, R2, jobs[2][1]], [prev] * 3, 100), 2)

    def raw(mutate, n=2, table=True, nm=True):
        p = prev.copy()
        m12 = np.zeros(len(prev), np.int32)
        J = (_InitJobC * n)()
        for j in range(n):
            J[j] = _InitJobC(R1.resident._h, R2.resident._h, p.ctypes.data, 100, m12.ctypes.data)
        mutate(J)
        out = np.zeros(n, np.int32)
        from orb_slam2_b200._lib import check
        check(lib.borb_search_for_initialization_batch(mt._h, J if table else None, n, 0.9, 1, out.ctypes.data if nm else None),
              "borb_search_for_initialization_batch")

    raw(lambda J: None)                                                   # the well-formed table runs
    refused(lambda: raw(lambda J: setattr(J[1], "prev_matched", None)), 1)
    refused(lambda: raw(lambda J: setattr(J[0], "matches12", None)), 0)
    refused(lambda: raw(lambda J: setattr(J[1], "current", None)), 1)
    refused(lambda: raw(lambda J: None, table=False), 0)
    refused(lambda: raw(lambda J: None, nm=False), 0)
