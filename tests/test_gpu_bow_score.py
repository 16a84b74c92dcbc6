"""GPU parity of borb_bow_score_batch: TemplatedVocabulary::score(v1, v2) cast to float between BowVectors already on the device,
resident frames and database slots in any mix, as LoopClosing::DetectLoop takes minScore (src/LoopClosing.cc:121-140).  Every score
must equal, bit for bit, the verbatim DBoW2 score (oracle/_ref/libdbowref.so) and the port's, including -0.0f for vectors that share
no word; for every live slot it must equal the score borb_kfdb_query_batch gives the same query; and a DetectLoop replay of many
streams whose covisible keyframes are not all in the database yet must give the verbatim DetectLoopCandidates lists."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from orb_slam2_b200 import _lib
from orb_slam2_b200 import sharding
from orb_slam2_b200._lib import BorbError
from tests import bow_envelope as BE

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL_ARR = os.path.join(ROOT, "oracle", "_ref", "orbvoc_arrays.npz")
GOLDEN = ["extract_euroc_1200", "extract_kitti_2000", "extract_tum_1000"]
SCALE = (1.2 ** np.arange(8)).astype(np.float32)
LEVELSUP = 4


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def mt(M):
    return M.ORBmatcher(0.75, True)


@pytest.fixture(scope="module")
def rv(oracle, tmp_path_factory):
    """The verbatim DBoW2 vocabulary (L1 scoring, 70,000 words: its database's inverted file spans every word id used here), or
    None where the reference build is absent."""
    if not oracle.have_dbowref():
        return None
    path = BE.write_voc(BE.vocabulary("flat70000"), str(tmp_path_factory.mktemp("bow_score") / "flat70000.txt"))
    return oracle.RefVocabulary(path)


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def random_keys(rng, n):
    from orb_slam2_b200._lib import KP_DTYPE
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(20, 730, n); k["y"] = rng.uniform(20, 460, n); k["angle"] = rng.uniform(0, 360, n)
    k["size"] = 31.0; k["octave"] = rng.integers(0, 8, n); k["class_id"] = -1
    return k


def flip_bits(rng, d, p):
    f = rng.random((len(d), 32, 8)) < p
    return d ^ np.packbits(f, axis=2, bitorder="little").reshape(len(d), 32)


def resident(M, mt, keys, desc):
    return M.FrameView(keys, np.ascontiguousarray(desc, np.uint8), SCALE, (0.0, 0.0, 752.0, 480.0)).make_resident(mt)


def want(oracle, rv, b1, b2):
    """float(score(b1, b2)) of the port, pinned to the verbatim DBoW2 score where it is built."""
    s = oracle.port_bow_score(b1, b2)[0]
    if rv is not None:
        r = rv.score(b1, b2)
        assert np.float64(r).view(np.uint64) == np.float64(s).view(np.uint64)
    return np.float32(s)


def frames_with_bow(M, mt, voc, descs, levelsup=LEVELSUP, seed=0):
    rng = np.random.default_rng(seed)
    frames = [resident(M, mt, random_keys(rng, len(d)), d) for d in descs]
    host = mt.ComputeBoWBatch(voc, frames, levelsup)
    return frames, [b for b, _ in host]


def items_of(M, mt, frames, bows, dbs):
    """Every frame as itself and as a slot of one of `dbs` (added from the frame, so with the same BowVector): [(ref, bow)]."""
    items = [(F, b) for F, b in zip(frames, bows)]
    owner = [dbs[i % len(dbs)] for i in range(len(frames))]
    slots = mt.KfdbAddFramesBatch(owner, frames, None)
    return items + [((db, s), b) for db, s, b in zip(owner, slots, bows)]


def check_all_pairs(oracle, rv, mt, items):
    """One call: every item against every item (itself included).  Both argument orders agree bitwise."""
    got = mt.BowScoreBatch([(r, [t for t, _ in items]) for r, _ in items])
    n = len(items)
    for a in range(n):
        for b in range(n):
            w = want(oracle, rv, items[a][1], items[b][1])
            assert bits(got[a][b]) == bits(w), (a, b, got[a][b], w)
        assert np.array_equal(bits(got[a]), bits([got[b][a] for b in range(n)])), a
    return got


def test_random_k10_L6_parity(M, mt, oracle, rv):
    """EuRoC-shaped keyframes of one scene (bit noise), random frames of 1, 1000 and 8192 features and a 0-feature frame, frames and
    slots of two databases, on a random k=10 L=6 tree."""
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    rng = np.random.default_rng(1)
    d0 = np.load(os.path.join(ROOT, "tests", "golden", "extract_euroc_1200.npz"))["descriptors"]
    descs = [flip_bits(rng, d0, p) for p in (0.0, 0.02, 0.05, 0.1)] + \
        [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (1, 1000, 8192)] + [np.zeros((0, 32), np.uint8)]
    frames, bows = frames_with_bow(M, mt, voc, descs)
    assert len(bows[-1]) == 0 and len(bows[-2]) > 4000
    dbs = [M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt)]
    items = items_of(M, mt, frames, bows, dbs)
    got = check_all_pairs(oracle, rv, mt, items)
    assert got[0][1] > 0.05 and got[0][0] > 0.99                      # the scene's keyframes do score against each other
    empty = len(frames) - 1
    assert (bits(got[empty]) == 0x80000000).all()                     # a 0-feature frame: -0.0f against everything


def test_real_vocabulary_parity(M, mt, oracle, rv):
    """The BowVectors the reference's own DBoW2 gives the golden descriptor sets on ORBvoc.txt (tests/golden/voc_real.npz) and
    re-weighted subsets of them as database slots; where the real tree is built, resident frames of the same sets with bit noise."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "voc_real.npz"))
    rng = np.random.default_rng(2)
    bows = []
    for name in GOLDEN:
        w, v = g[name + "_bow_word"], g[name + "_bow_value"]
        bows.append(dict(zip(w.tolist(), v.tolist())))
        for keep in (0.8, 0.4):
            sel = rng.random(len(w)) < keep
            vv = v[sel] * rng.uniform(0.3, 3.0, int(sel.sum()))
            bows.append(dict(zip(w[sel].tolist(), (vv / np.abs(vv).sum()).tolist())))
    dbs = [M.KeyFrameDatabase(mt) for _ in range(3)]
    empty = M.KeyFrameView(mvKeysUn=random_keys(rng, 0), mDescriptors=np.zeros((0, 32), np.uint8),
                           mFeatVec=M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32)))
    items = [((dbs[i % 3], dbs[i % 3].add(empty, b)), b) for i, b in enumerate(bows)]
    if os.path.exists(REAL_ARR):
        a = np.load(REAL_ARR)
        voc = M.ORBVocabulary.from_arrays(a["parent"], a["is_leaf"], a["desc"], a["weight"], int(a["k"][0]), int(a["L"][0]))
        descs = []
        for name in GOLDEN:
            d = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["descriptors"]
            descs += [d, flip_bits(rng, d, 0.03)]
        frames, fb = frames_with_bow(M, mt, voc, descs, seed=3)
        for name, b in zip(GOLDEN, fb[0::2]):                          # the device BoW is the golden one
            assert list(b) == g[name + "_bow_word"].tolist()
        items += [(F, b) for F, b in zip(frames, fb)]
    got = check_all_pairs(oracle, rv, mt, items)
    assert got[0][1] > 0.2


@pytest.mark.parametrize("name", ["flat70000", "uneven"])
def test_envelope_vocabularies_parity(M, mt, oracle, rv, name):
    """The flat (70,000 words under the root) and uneven trees of tests/bow_envelope.py, each set against its noisy copy."""
    a = BE.vocabulary(name)
    voc = M.ORBVocabulary.from_arrays(a["parent"], a["is_leaf"], a["desc"], a["weight"], a["k"], a["L"])
    descs = list(BE.descriptors(name).values())
    rng = np.random.default_rng(4)
    descs += [flip_bits(rng, d, 0.01) for d in descs]
    frames, bows = frames_with_bow(M, mt, voc, descs, levelsup=BE.LEVELSUP[name][-1], seed=5)
    items = items_of(M, mt, frames, bows, [M.KeyFrameDatabase(mt)])
    got = check_all_pairs(oracle, rv, mt, items)
    k = len(descs) // 2
    assert any(got[i][i + k] > 0.05 for i in range(k))                 # a set against its noisy copy


@pytest.fixture(scope="module")
def world(M, mt):
    """Frames of a random k=10 L=4 tree: five EuRoC-shaped scenes, eight noisy re-observations each, resident with BoW."""
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 4, 9), 10, 4)
    rng = np.random.default_rng(6)
    base = [np.load(os.path.join(ROOT, "tests", "golden", n + ".npz"))["descriptors"][:1200] for n in GOLDEN]
    base += [rng.integers(0, 256, (1200, 32), dtype=np.uint8) for _ in range(2)]
    descs = [flip_bits(rng, base[i % 5], 0.03 + 0.01 * (i // 5 % 4)) for i in range(40)]
    frames, bows = frames_with_bow(M, mt, voc, descs, levelsup=2, seed=7)
    return voc, frames, bows


def test_edges(M, mt, oracle, rv, world):
    """Disjoint vectors give -0.0f; a self-score; the query among its own targets; repeated targets; 2,000 targets of one job spread
    over three databases and frames."""
    _, frames, bows = world
    dbs = [M.KeyFrameDatabase(mt) for _ in range(3)]
    items = items_of(M, mt, frames[:12], bows[:12], dbs)
    kv = M.KeyFrameView(mvKeysUn=random_keys(np.random.default_rng(0), 0), mDescriptors=np.zeros((0, 32), np.uint8),
                        mFeatVec=M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32)))
    top = max(max(b) for b in bows) + 1
    disjoint = [{top + 1: 0.25, top + 5: 0.75}, {top + 2: 1.0}]
    items += [((dbs[1], dbs[1].add(kv, b)), b) for b in disjoint]
    rng = np.random.default_rng(8)
    pick = rng.integers(0, len(items), 2000)
    pick[:3] = [0, 0, len(items) - 1]
    q = items[3]
    got, selfs, dis = mt.BowScoreBatch([(q[0], [items[i][0] for i in pick]), (items[0][0], [items[0][0]]),
                                        (items[-1][0], [items[-2][0], items[-1][0], items[5][0]])])
    assert len(got) == 2000
    memo = {}
    for t, i in enumerate(pick):
        if i not in memo:
            memo[i] = want(oracle, rv, q[1], items[i][1])
        assert bits(got[t]) == bits(memo[i]), (t, i)
    assert bits(got[0]) == bits(got[1])                               # a repeated target
    assert bits(selfs[0]) == bits(want(oracle, rv, bows[0], bows[0]))
    assert (bits(dis[[0, 2]]) == 0x80000000).all() and dis[1] == want(oracle, rv, disjoint[1], disjoint[1])
    # a query among its own targets, as a frame and as its slot
    own = mt.BowScoreBatch([(items[2][0], [items[2][0], items[14][0], items[7][0]])])[0]
    assert bits(own[0]) == bits(own[1]) == bits(want(oracle, rv, bows[2], bows[2]))


def test_scores_equal_the_database_query(M, mt, world):
    """For every live slot, the score of borb_kfdb_query_batch for a frame equals borb_bow_score_batch's for the same pair."""
    _, frames, bows = world
    db = M.KeyFrameDatabase(mt)
    mt.KfdbAddFramesBatch(db, frames[:30], None)
    db.erase(4); db.erase(17)
    live = [s for s in range(30) if s not in (4, 17)]
    queries = frames[28:40]
    got = mt.BowScoreBatch([(F, [(db, s) for s in live]) for F in queries])
    for (cw, sc, fw), g in zip(mt.KfdbQueryBatch(db, queries), got):
        assert np.array_equal(bits(sc[live]), bits(g))
    assert max(float(g.max()) for g in got) > 0.2


def test_detect_loop_replay(M, mt, oracle, rv, world):
    """LoopClosing::DetectLoop of 8 streams over 40 keyframes, each stream with its own database.  At every step: minScore from one
    borb_bow_score_batch over the covisible keyframes that are not bad (1.0f, then the float minimum; some covisible keyframes are
    resident frames LoopClosing has not added yet, some are bad and skipped by the caller), the query of every stream in one
    KfdbQueryBatch, loop_candidates, and the keyframe added with KfdbAddFramesBatch.  The candidate lists equal the verbatim
    KeyFrameDatabase::DetectLoopCandidates fed with the verbatim DBoW2 minScore of host copies."""
    if rv is None:
        pytest.skip("oracle/_ref/libdbowref.so not built (reference tree absent)")
    _, frames, bows = world
    S, N = 8, 40
    rng = np.random.default_rng(10)
    order = [rng.permutation(N) for _ in range(S)]                    # each stream meets the 40 keyframes in its own order
    dbs = [M.KeyFrameDatabase(mt) for _ in range(S)]
    slot_of = [dict() for _ in range(S)]                              # keyframe -> slot, per stream
    neigh = [[] for _ in range(S)]                                    # per slot: up to 10 covisible slots, best first
    total, differs = 0, 0
    for i in range(N):
        jobs, covis_kf, connected = [], [], []
        for s in range(S):
            kf = order[s][i]
            cov = [order[s][x] for x in (i - 1, i - 2, i - 3, i + 1, i + 2) if 0 <= x < N]    # i + 1, i + 2: not added yet
            bad = set(cov[1:2])
            good = [c for c in cov if c not in bad]
            jobs.append((frames[kf], [(dbs[s], slot_of[s][c]) if c in slot_of[s] else frames[c] for c in good]))
            covis_kf.append(good)
            connected.append({slot_of[s][c] for c in cov if c in slot_of[s]})
        scores = mt.BowScoreBatch(jobs)
        query = mt.KfdbQueryBatch(dbs, [frames[order[s][i]] for s in range(S)])
        for s in range(S):
            kf = order[s][i]
            minScore, ref_min, slotted_min = np.float32(1.0), np.float32(1.0), np.float32(1.0)
            for c, sc in zip(covis_kf[s], scores[s]):
                r = np.float32(rv.score(bows[kf], bows[c]))
                assert bits(sc) == bits(r)
                minScore, ref_min = min(minScore, sc), min(ref_min, r)
                if c in slot_of[s]:
                    slotted_min = min(slotted_min, r)
            assert bits(minScore) == bits(ref_min)
            differs += slotted_min != ref_min
            cw, sc, fw = query[s]
            n_kf = len(slot_of[s])
            got = M.loop_candidates(cw, sc, fw, dbs[s]._seq, connected[s], lambda x, s=s: neigh[s][x], minScore)
            if n_kf:
                kf_bows = [None] * n_kf
                for k, sl in slot_of[s].items():
                    kf_bows[sl] = bows[k]
                ng = np.full((n_kf, 10), -1, np.int32)
                for sl in range(n_kf):
                    ng[sl, :len(neigh[s][sl])] = neigh[s][sl]
                cn = np.zeros(n_kf, np.uint8)
                cn[list(connected[s])] = 1
                assert got == rv.detect_candidates(True, kf_bows, bows[kf], cn, ng, ref_min), (i, s)
            else:
                assert got == []
            total += len(got)
        slots = mt.KfdbAddFramesBatch(dbs, [frames[order[s][i]] for s in range(S)], None)
        for s, sl in enumerate(slots):
            assert sl == i
            slot_of[s][order[s][i]] = sl
            neigh[s].append([slot_of[s][order[s][x]] for x in (i - 1, i - 2, i - 3) if x >= 0][:10])
    assert total > 20 and differs > 0                                 # loops are found, and the unslotted keyframes matter


def test_launch_count(M, mt, world):
    _, frames, _ = world
    db = M.KeyFrameDatabase(mt)
    mt.KfdbAddFramesBatch(db, frames[:4], None)
    for n in (1, 8, 32):
        c0 = launches(mt)
        out = mt.BowScoreBatch([(frames[j % 40], [frames[(j + 1) % 40], (db, j % 4)]) for j in range(n)])
        assert launches(mt) - c0 == 1 and len(out) == n
    c0 = launches(mt)
    assert [len(x) for x in mt.BowScoreBatch([(frames[0], []), ((db, 1), [])])] == [0, 0]
    assert mt.BowScoreBatch([]) == []
    assert launches(mt) == c0


def test_refusals_name_the_reference(M, mt):
    """Each refusal is BORB_ERR_INVALID_ARG before any launch, naming "job j target t:" (or "job j query:", "job j:")."""
    rng = np.random.default_rng(11)
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 3, 5), 10, 3)
    good = [resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8)) for _ in range(3)]
    mt.ComputeBoWBatch(voc, good, 1, want_host=False)
    db = M.KeyFrameDatabase(mt)
    mt.KfdbAddFramesBatch(db, good, None)
    db.erase(1)
    no_bow = resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
    old = resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
    mt.ComputeBoWBatch(voc, [old], 1, want_host=False)
    old.resident.close()
    recycled = resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
    nowhere = M.FrameView(None, None, SCALE, (0, 0, 1, 1))

    def refused(jobs, prefix, what):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            mt.BowScoreBatch(jobs)
        detail = str(ei.value).split(": ", 2)[2]
        assert ei.value.status == 1 and detail.startswith(prefix) and what in detail, str(ei.value)
        assert launches(mt) == c0

    ok = (good[0], [good[1], (db, 0)])
    refused([ok, (good[0], [good[1], (db, 1)])], "job 1 target 1:", "not a live keyframe")
    refused([ok, (good[0], [(db, 2), (db, 3)])], "job 1 target 1:", "not a live keyframe")
    refused([(good[0], [(db, -1)])], "job 0 target 0:", "not a live keyframe")
    refused([ok, ok, (good[2], [good[0], good[1], no_bow])], "job 2 target 2:", "has no BoW")
    refused([ok, (recycled, [good[0]])], "job 1 query:", "has no BoW")
    refused([ok, ((db, 1), [good[0]])], "job 1 query:", "not a live keyframe")
    refused([(good[0], [good[1], nowhere])], "job 0 target 1:", "neither a frame nor a database")
    refused([(good[0], [(None, 0)])], "job 0 target 0:", "neither a frame nor a database")
    # n_targets < 0, NULL targets, NULL score: through the C structs
    jobs = (M._BowScoreJobC * 2)()
    refs = (M._BowRefC * 1)(M.ORBmatcher._bow_ref(good[1]))
    sc = np.zeros(1, np.float32)
    for j in range(2):
        jobs[j].query, jobs[j].targets, jobs[j].n_targets, jobs[j].score = M.ORBmatcher._bow_ref(good[0]), C.addressof(refs), 1, sc.ctypes.data
    for field, value, text in (("n_targets", -1, "n_targets"), ("targets", None, "null"), ("score", None, "null")):
        saved = getattr(jobs[1], field)
        setattr(jobs[1], field, value)
        c0 = launches(mt)
        st = mt._lib.borb_bow_score_batch(mt._h, jobs, 2)
        assert st == 1 and mt._lib.borb_last_error().decode().startswith("job 1:") and text in mt._lib.borb_last_error().decode()
        assert launches(mt) == c0
        setattr(jobs[1], field, saved)
    assert mt._lib.borb_bow_score_batch(mt._h, jobs, 2) == 0 and sc[0] == mt.BowScoreBatch([(good[0], [good[1]])])[0][0]
    assert mt._lib.borb_bow_score_batch(mt._h, None, 0) == 0
    assert mt._lib.borb_bow_score_batch(mt._h, None, 1) == 1
    assert mt._lib.borb_bow_score_batch(mt._h, jobs, -1) == 1
    # a frame on another device than the matcher cannot be built on a one-GPU machine
    if _lib.device_count() > 1:
        m1 = M.ORBmatcher(0.75, True, device=1)
        voc1 = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 3, 5), 10, 3, device=1)
        far = resident(M, m1, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
        m1.ComputeBoWBatch(voc1, [far], 1, want_host=False)
        refused([(good[0], [far])], "job 0 target 0:", "different devices")


def test_poisoned_buffers_change_nothing(M, mt, world):
    _, frames, _ = world
    so = _lib.load()
    db = M.KeyFrameDatabase(mt)
    mt.KfdbAddFramesBatch(db, frames[:10], None)
    jobs = [(frames[j], [frames[(j + k) % 40] if k % 2 else (db, (j + k) % 10) for k in range(12)]) for j in range(20)]
    so.borb_debug_set_poison(-1)
    base = mt.BowScoreBatch(jobs)
    try:
        for p in (0x00, 0xFF, 0x7F):
            so.borb_debug_set_poison(p)
            m2 = M.ORBmatcher(0.75, True)                              # fresh buffers, grown (and poisoned) by the call
            for m in (mt, m2):
                for x, y in zip(m.BowScoreBatch(jobs), base):
                    assert np.array_equal(bits(x), bits(y)), p
    finally:
        so.borb_debug_set_poison(-1)


def test_concurrent_add_erase_and_scores(M, world):
    """One thread adds keyframes, erases one of the scored slots and rewrites MapPoint masks on its own matcher, while another scores
    against the database on a second matcher: every call returns the scores of the state before the erase (which are those of any
    state, slots never change) or is refused for the erased slot, and after the erase it is refused."""
    _, frames, _ = world
    ma, mb = M.ORBmatcher(0.75, True), M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(ma)
    ma.KfdbAddFramesBatch(db, frames[:10], None)
    targets = [(db, s) for s in range(10)] + [frames[12], frames[13]]
    jobs = [(frames[j], targets) for j in (20, 21, 22)]
    before = mb.BowScoreBatch(jobs)
    erased = threading.Event()
    done = threading.Event()
    seen, errors = [], []

    def writer():
        try:
            for i in range(10, 40, 5):
                ma.KfdbAddFramesBatch(db, frames[i:i + 5], None)
                if i == 20:
                    db.erase(7)
                    erased.set()
                db.set_has_mp(0, np.zeros(frames[0].resident.n, np.uint8))
        except Exception as e:                                        # noqa: BLE001 - reported by the main thread
            errors.append(e)
        finally:
            done.set()

    def scorer():
        try:
            while True:
                last = done.is_set()
                was_erased = erased.is_set()
                try:
                    seen.append((was_erased, mb.BowScoreBatch(jobs)))
                except BorbError as e:
                    seen.append((was_erased, str(e)))
                if last:
                    break
        except Exception as e:                                        # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=writer), threading.Thread(target=scorer)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert len(seen) >= 2 and db.size()[0] == 40
    for was_erased, r in seen:
        if isinstance(r, str):
            assert "job 0 target 7: slot 7 is not a live keyframe" in r
        else:
            assert not was_erased
            for x, y in zip(r, before):
                assert np.array_equal(bits(x), bits(y))
    assert isinstance(seen[-1][1], str)
