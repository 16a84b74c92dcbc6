"""The library driven the way ORB-SLAM2 drives it: from the Tracking, LocalMapping and LoopClosing threads at once, sharing one
ORBVocabulary and one KeyFrameDatabase (src/Tracking.cc:760,1344,1348, src/LocalMapping.cc:137, src/LoopClosing.cc:116-215,
src/KeyFrame.cc:544).  Every thread is a Python thread calling the C ABI through ctypes (which releases the GIL, so the calls
overlap), with its own ORBmatcher as the adapters keep one per thread.  Every expected value is computed on the main thread before
any worker starts, from the port (oracle/) and from a single-threaded run of the library; workers collect their failures into a
list that the main thread asserts."""
import ctypes as C
import threading

import numpy as np
import pytest

from orb_slam2_b200 import synth

pytestmark = pytest.mark.gpu

JOIN_TIMEOUT = 180.0
LEVELSUP = 2
NNRATIO = 0.75
SCALE = (1.2 ** np.arange(8)).astype(np.float32)


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


def run_threads(targets):
    """Starts one daemon thread per (callable, args), joins each with a timeout; returns the failures they reported."""
    errors = []

    def wrap(fn, args):
        try:
            fn(*args)
        except Exception as ex:                                            # reported on the main thread
            errors.append(repr(ex))

    threads = [threading.Thread(target=wrap, args=(fn, args), daemon=True) for fn, args in targets]
    for th in threads:
        th.start()
    for th in threads:
        th.join(JOIN_TIMEOUT)
    hung = [i for i, th in enumerate(threads) if th.is_alive()]
    assert not hung, f"threads {hung} did not finish within {JOIN_TIMEOUT} s"
    return errors


def voc_of(M, pv):
    e = pv.export()
    return M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])


def same_bow(got, want):
    (bg, fg), (bw, fw) = got, want
    return (list(bg.items()) == list(bw.items()) and np.array_equal(fg.node_id, fw.node_id) and np.array_equal(fg.start, fw.start)
            and np.array_equal(fg.feat_idx, fw.feat_idx))


def same_raw(got, want):
    return all(np.array_equal(g, w) for g, w in zip(got, want))


def resident(M, mt, keys, desc):
    return M.FrameView(keys, np.ascontiguousarray(desc, np.uint8), SCALE, (0.0, 0.0, 640.0, 480.0)).make_resident(mt)


def noisy(rng, img, a):
    return np.clip(img.astype(np.int32) + rng.integers(-a, a + 1, img.shape), 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def descriptor_sets():
    """Six extracted 640x480 frames of 2000 features, one per thread: its descriptor sets are prefixes of 200 to 2000 rows."""
    from orb_slam2_b200.extractor import ORBextractor
    outs = ORBextractor(2000).extract_batch([synth.mono_frame(400 + i, 0, 0, 640, 480) for i in range(6)])
    assert all(len(d) >= 1500 for _, d in outs)
    return outs


# ------------------------------------------------------------------------------------------------------ 1. one shared vocabulary
def bow_race(M, oracle, voc, pv, descs, sizes_of):
    """Thread t calls ComputeBoW and transform_raw on descs[t][:sizes_of(t, r)] for r in its repetitions; both must equal the port
    and the single-threaded result.  Returns the failures and the number of mismatched calls."""
    from orb_slam2_b200.matcher import bow_and_featvec
    plan = [[sizes_of(t, r) for r in range(40)] for t in range(len(descs))]
    want = {}
    for t, d in enumerate(descs):
        for n in sorted(set(plan[t])):
            raw = pv.transform_raw(d[:n], LEVELSUP)
            want[t, n] = (raw, bow_and_featvec(*raw))
    mismatched = []

    def worker(t):
        got = [(n, voc.ComputeBoW(descs[t][:n], LEVELSUP), voc.transform_raw(descs[t][:n], LEVELSUP)) for n in plan[t]]
        for r, (n, bow, raw) in enumerate(got):                           # compared after the race, so the calls stay dense
            mismatched.extend([(t, r, n, "ComputeBoW")] if not same_bow(bow, want[t, n][1]) else [])
            mismatched.extend([(t, r, n, "transform_raw")] if not same_raw(raw, want[t, n][0]) else [])

    errors = run_threads([(worker, (t,)) for t in range(len(descs))])
    return errors, mismatched, 2 * sum(len(p) for p in plan), want


def test_shared_vocabulary_fixed_scratch(M, oracle, descriptor_sets):
    """Six threads transform on one vocabulary whose buffers were sized beforehand by both calls on the largest set, so nothing is
    reallocated during the race: without the vocabulary's lock the calls overwrite each other's descriptors and results in the
    one set of buffers."""
    from orb_slam2_b200.matcher import bow_and_featvec
    pv = oracle.PortVocabulary.random(10, 4, 5)
    voc = voc_of(M, pv)
    descs = [d for _, d in descriptor_sets]
    big = max(range(len(descs)), key=lambda t: len(descs[t]))
    sizes = lambda t, r: min(len(descs[t]), 200 + ((7 * t + 3 * r) % 10) * 200)
    raw = pv.transform_raw(descs[big], LEVELSUP)
    assert same_raw(voc.transform_raw(descs[big], LEVELSUP), raw)          # these two size the buffers for every call below
    assert same_bow(voc.ComputeBoW(descs[big], LEVELSUP), bow_and_featvec(*raw))
    errors, mismatched, total, want = bow_race(M, oracle, voc, pv, descs, sizes)
    assert not errors, errors
    assert not mismatched, f"{len(mismatched)} of {total} calls differ from the port, e.g. {mismatched[:6]}"
    for (t, n), (raw, bow) in list(want.items())[:8]:                    # the single-threaded library after the race
        assert same_raw(voc.transform_raw(descs[t][:n], LEVELSUP), raw) and same_bow(voc.ComputeBoW(descs[t][:n], LEVELSUP), bow)


def test_shared_vocabulary_growing_scratch(M, oracle, descriptor_sets):
    """A fresh vocabulary (empty scratch); every thread steps its sets up from 200 rows to 2000, so the scratch is regrown while
    other threads are in the middle of their calls."""
    pv = oracle.PortVocabulary.random(10, 4, 5)
    voc = voc_of(M, pv)
    descs = [d for _, d in descriptor_sets]
    sizes = lambda t, r: min(len(descs[t]), 200 + 45 * r + 7 * t)
    errors, mismatched, total, _ = bow_race(M, oracle, voc, pv, descs, sizes)
    assert not errors, errors
    assert not mismatched, f"{len(mismatched)} of {total} calls differ from the port, e.g. {mismatched[:6]}"


def test_shared_vocabulary_host_and_resident_paths(M, oracle, descriptor_sets):
    """One thread runs the host path (borb_compute_bow, on the vocabulary's buffers and stream) while the others run
    ComputeBoWBatch on their own resident frames with their own matchers; both paths equal the port."""
    from orb_slam2_b200.matcher import bow_and_featvec
    pv = oracle.PortVocabulary.random(10, 4, 5)
    voc = voc_of(M, pv)
    sets = [(k[:n], d[:n]) for (k, d), n in zip(descriptor_sets, (2000, 1500, 1100, 700, 300, 1800))]
    want = [bow_and_featvec(*pv.transform_raw(d, LEVELSUP)) for _, d in sets]
    bad = []

    def host(reps):
        for r in range(reps):
            for t, (_, d) in enumerate(sets):
                if not same_bow(voc.ComputeBoW(d, LEVELSUP), want[t]):
                    bad.append(("host", r, t))

    def batch(t, reps):
        mt = M.ORBmatcher(NNRATIO, True)
        mine = [(t + i) % len(sets) for i in range(3)]
        frames = [resident(M, mt, *sets[i]) for i in mine]
        for r in range(reps):
            for i, g in zip(mine, mt.ComputeBoWBatch(voc, frames, LEVELSUP)):
                if not same_bow(g, want[i]):
                    bad.append(("batch", t, r, i))

    errors = run_threads([(host, (25,))] + [(batch, (t, 40)) for t in range(4)])
    assert not errors, errors
    assert not bad, f"{len(bad)} results differ from the port, e.g. {bad[:6]}"


# ------------------------------------------------------------------------------------------------------ 2. one shared database
N_KF, N_ADD, N_CONTENT = 48, 264, 32
GROUP, VOLATILE = list(range(24, 32)), list(range(32, 48))     # slots 0-23 are stable


@pytest.fixture(scope="module")
def world(M, oracle):
    """The keyframes of test_gpu_kfdb.py's world (triples of frames share a scene), the contents LocalMapping adds, and the query
    frames of Tracking; FeatureVectors and BowVectors from the port's descent."""
    from orb_slam2_b200.extractor import ORBextractor
    from orb_slam2_b200.matcher import bow_and_featvec
    pv = oracle.PortVocabulary.random(10, 4, 5)
    X = ORBextractor(800)
    rng = np.random.default_rng(3)
    base = [synth.mono_frame(200 + i // 3, 0, 0, 640, 480) for i in range(N_KF)]
    kf_out = X.extract_batch([noisy(rng, b, 6) for b in base])
    add_out = X.extract_batch([noisy(rng, synth.mono_frame(500 + i // 2, 0, 0, 640, 480), 6) for i in range(N_CONTENT)])
    q_out = X.extract_batch([noisy(rng, base[i], 8) for i in (7, 20, 26, 40)])

    def views(outs, p_mp):
        vs, bows = [], []
        for k, d in outs:
            bow, fv = bow_and_featvec(*pv.transform_raw(d, LEVELSUP))
            vs.append(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < p_mp).astype(np.uint8)))
            bows.append(bow)
        return vs, bows

    kfs, bows = views(kf_out, 0.7)
    adds, add_bows = views(add_out, 0.7)
    qs, q_bows = views(q_out, 0.0)
    masks = [{s: (rng.random(len(kfs[s].mvKeysUn)) < 0.7).astype(np.uint8) for s in GROUP} for _ in range(2)]
    for s in GROUP:
        kfs[s] = M.KeyFrameView(kfs[s].mvKeysUn, kfs[s].mDescriptors, kfs[s].mFeatVec, has_mp=masks[0][s])
    return dict(pv=pv, kfs=kfs, bows=bows, adds=adds, add_bows=add_bows, qs=qs, q_bows=q_bows, masks=masks)




def with_mask(M, kf, hm):
    return M.KeyFrameView(kf.mvKeysUn, kf.mDescriptors, kf.mFeatVec, has_mp=hm)


def blocks(res):
    """(nmatches, pair_offset, pairs) -> the pair block of every keyframe."""
    nm, off, pairs = res
    return [pairs[off[k]:off[k] + nm[k]].copy() for k in range(len(nm))]


def dense(block, n):
    out = np.full(n, -1, np.int32)
    out[(block & 0xFFFF).astype(np.int64)] = (block >> 16).astype(np.int32)
    return out


def mask_state(got, want):
    """got = {slot: block}, want = [{slot: block} under mask set 0, ... under set 1] for the slots whose result may depend on the
    group's masks: None when all of them show the same mask set, else why not (a slot that matches neither set, or slots that show
    different sets).  A slot whose block is the same under both sets only has to match it."""
    seen = {s: [i for i in (0, 1) if np.array_equal(got[s], want[i][s])] for s in want[0]}
    if any(not v for v in seen.values()):
        return f"slots {[s for s, v in seen.items() if not v]} match neither mask set"
    if len({v[0] for v in seen.values() if len(v) == 1}) > 1:
        return f"one search saw both mask sets: {[v for v in seen.values()]}"
    return None


def telling(want, key):
    """The group slots whose block differs between the two mask sets in the search `key` = (query, .)."""
    return [s for s in GROUP if not np.array_equal(want[0][key, s], want[1][key, s])]


TRACK_SLOTS = list(range(0, 24, 3)) + GROUP                       # Tracking's SearchByBoW candidates: stable slots and the group
LOOP_QUERIES = [6, 25]                                             # LoopClosing's keyframes (one stable, one of the group) ...
LOOP_SLOTS = [7, 8, 19, 21, 0] + GROUP                             # ... and their candidates


def test_keyframe_database_three_threads(M, oracle, world):
    """A replay of ORB-SLAM2's three threads on one KeyFrameDatabase.  Slots 0-23 are never modified; LoopClosing switches the
    MapPoint masks of the group 24-31 between two sets with one set_has_mp_batch and searches loop candidates; LocalMapping computes
    the BoW of 264 new keyframes on the shared vocabulary, adds them (the slot table is reallocated twice during the run: it grows
    past 136 and past 269 slots) and erases slots 32-47 one by one; Tracking computes its frames' BoW with ComputeBoWBatch and
    queries and searches the database.  Every search must see each add, erase and mask batch whole."""
    pv, kfs, bows, masks, qs, q_bows = (world[k] for k in ("pv", "kfs", "bows", "masks", "qs", "q_bows"))
    voc = voc_of(M, pv)
    mt_track = M.ORBmatcher(NNRATIO, True)                         # the database's own matcher: used by Tracking only during the run
    db = M.KeyFrameDatabase(mt_track)
    assert [db.add(kf, b) for kf, b in zip(kfs, bows)] == list(range(N_KF))
    all_views, all_bows = kfs + world["adds"], bows + world["add_bows"]
    content = lambda s: s if s < N_KF else N_KF + (s - N_KF) % N_CONTENT     # slot -> index into all_views / all_bows
    n_final = N_KF + N_ADD

    # expected values: every score from the port; the pair blocks of a single-threaded run under each mask set, checked against the port
    exp = []
    for qb in q_bows:
        r = [oracle.port_bow_score(qb, all_bows[content(s)]) for s in range(n_final)]
        exp.append((np.array([x[1] for x in r], np.int32), np.array([x[0] for x in r], np.float32), np.array([x[2] for x in r], np.uint32)))
    mt_loop = M.ORBmatcher(NNRATIO, True)
    track_want, loop_want = [], []                                 # [mask set] -> {(query, slot): block}
    for ms in (0, 1):
        db.set_has_mp_batch(GROUP, [masks[ms][s] for s in GROUP])
        kv = lambda s: with_mask(M, kfs[s], masks[ms][s]) if s in GROUP else kfs[s]
        tw, lw = {}, {}
        for q, F in enumerate(qs):
            for s, b in zip(TRACK_SLOTS, blocks(db.SearchByBoWPairs(TRACK_SLOTS, F))):
                n_o, m_o = oracle.port_search_by_bow(kv(s), F, NNRATIO, True)
                assert len(b) == n_o and np.array_equal(dense(b, len(F.mvKeysUn)), m_o), (ms, q, s)
                tw[q, s] = b
        for q in LOOP_QUERIES:
            for s, b in zip(LOOP_SLOTS, blocks(mt_loop.SearchByBoWKFDbBatch(db, [q], [LOOP_SLOTS])[0])):
                n_o, m_o = oracle.port_search_by_bow_kf(kv(q), kv(s), NNRATIO, True)
                assert len(b) == n_o and np.array_equal(dense(b, len(kfs[q].mvKeysUn)), m_o), (ms, q, s)
                lw[q, s] = b
        track_want.append(tw); loop_want.append(lw)
    # a search that saw half a mask batch is told apart: each of Tracking's searches by four group slots or more (every group slot
    # by one of them at least), the group keyframe's loop search (its own mask switches with the batch) by its scene neighbours
    tell = [telling(track_want, q) for q in range(len(qs))]
    assert min(map(len, tell)) >= 4 and set().union(*tell) == set(GROUP), tell
    assert {24, 26} <= set(telling(loop_want, 25)), telling(loop_want, 25)
    state = [1]                                                    # the mask set the group holds now
    erased_where = []
    done = threading.Event()
    bad = []

    def check_scores(where, q, res, seen, last_n):
        cw, sc, fw = res
        n = len(cw)
        if n < last_n[0] or not N_KF <= n <= n_final:
            bad.append((where, "slot count went from", last_n[0], "to", n))
            return
        last_n[0] = n
        ok = (cw == exp[q][0][:n]) & (sc == exp[q][1][:n]) & (fw == exp[q][2][:n])
        erased = (cw == 0) & (sc == 0) & (fw == 0xFFFFFFFF)
        for s in VOLATILE:
            if erased[s] and not ok[s]:
                seen.add(s)
            elif not ok[s]:
                bad.append((where, "volatile slot is neither itself nor erased", s))
            elif s in seen and not erased[s]:
                bad.append((where, "erased slot came back", s))
        ok[VOLATILE] = True
        if not ok.all():
            bad.append((where, "slots differ from the port", np.nonzero(~ok)[0][:8].tolist()))

    def tracking():
        frames = [resident(M, mt_track, F.mvKeysUn, F.mDescriptors) for F in qs]
        seen, last_n, it = set(), [0], 0
        while not done.is_set() or it < 20:
            for q, g in enumerate(mt_track.ComputeBoWBatch(voc, frames, LEVELSUP)):
                if not same_bow(g, (q_bows[q], qs[q].mFeatVec)):
                    bad.append(("tracking bow", it, q))
            for q, res in enumerate(mt_track.KfdbQueryBatch(db, frames)):
                check_scores(("tracking query batch", it, q), q, res, seen, last_n)
            q = it % len(qs)
            check_scores(("tracking query", it, q), q, db.query(q_bows[q]), seen, last_n)
            F = M.KeyFrameView(qs[q].mvKeysUn, qs[q].mDescriptors, qs[q].mFeatVec)
            for where, res in (("tracking search", db.SearchByBoWPairs(TRACK_SLOTS, F)),
                               ("tracking resident search", mt_track.SearchByBoWDbBatch(db, [TRACK_SLOTS], [frames[q]])[0])):
                got = dict(zip(TRACK_SLOTS, blocks(res)))
                if any(not np.array_equal(got[s], track_want[0][q, s]) for s in TRACK_SLOTS if s not in GROUP):
                    bad.append((where, it, q, "stable slots differ"))
                msg = mask_state(got, [{s: w[q, s] for s in GROUP} for w in track_want])
                if msg:
                    bad.append((where, it, q, msg))
            it += 1

    def local_mapping():
        for i in range(N_ADD):
            c = i % N_CONTENT
            k, d = world["adds"][c].mvKeysUn, world["adds"][c].mDescriptors
            bow, fv = voc.ComputeBoW(d, LEVELSUP)
            if not same_bow((bow, fv), (world["add_bows"][c], world["adds"][c].mFeatVec)):
                bad.append(("local mapping bow", i))
            slot = db.add(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=world["adds"][c].has_mp), bow)
            if slot != N_KF + i:
                bad.append(("local mapping slot", i, slot))
            if i % 16 == 8:
                db.erase(VOLATILE[i // 16])
                erased_where.append(db.size()[0])
        done.set()

    def loop_closing():
        it = 0
        while not done.is_set() or it < 20:
            q = LOOP_QUERIES[it % 2]
            one = mt_loop.SearchByBoWKFDbBatch(db, [q], [LOOP_SLOTS])[0]
            both = mt_loop.SearchByBoWKFDbBatch(db, LOOP_QUERIES, [LOOP_SLOTS] * 2)
            for qq, res in [(q, one)] + list(zip(LOOP_QUERIES, both)):
                got = dict(zip(LOOP_SLOTS, blocks(res)))
                masked = LOOP_SLOTS if qq in GROUP else GROUP              # a group keyframe's own mask reaches every candidate
                if any(not np.array_equal(got[s], loop_want[0][qq, s]) for s in LOOP_SLOTS if s not in masked):
                    bad.append(("loop search", it, qq, "stable slots differ"))
                msg = mask_state(got, [{s: w[qq, s] for s in masked} for w in loop_want])
                if msg:
                    bad.append(("loop search", it, qq, msg))
            state[0] ^= 1
            db.set_has_mp_batch(GROUP, [masks[state[0]][s] for s in GROUP])
            it += 1

    errors = run_threads([(tracking, ()), (local_mapping, ()), (loop_closing, ())])
    assert not errors, errors
    assert not bad, f"{len(bad)} failures, e.g. {bad[:6]}"
    assert len(erased_where) == len(VOLATILE) and erased_where[-1] > 270

    # the final state equals a database rebuilt serially
    ref = M.KeyFrameDatabase(mt_track)
    for s in range(n_final):
        kv = all_views[content(s)]
        ref.add(with_mask(M, kv, masks[state[0]][s]) if s in GROUP else kv, all_bows[content(s)])
    for s in VOLATILE:
        ref.erase(s)
    assert db.size()[0] == ref.size()[0] == n_final
    live = list(range(32)) + list(range(N_KF, n_final, 5))
    for q, F in enumerate(qs):
        for a, b in zip(db.query(q_bows[q]), ref.query(q_bows[q])):
            assert np.array_equal(a, b), q
        for a, b in zip(blocks(db.SearchByBoWPairs(live, F)), blocks(ref.SearchByBoWPairs(live, F))):
            assert np.array_equal(a, b), q
    for q in LOOP_QUERIES + [25, N_KF + 3, n_final - 1]:
        for a, b in zip(blocks(db.SearchByBoWKFPairs(q, live)), blocks(ref.SearchByBoWKFPairs(q, live))):
            assert np.array_equal(a, b), q


def test_batches_over_two_databases_in_opposite_order(M, oracle, world):
    """Two threads run KfdbQueryBatch and SearchByBoWDbBatch over the same two databases, one with the jobs in the order [D1, D2],
    the other [D2, D1]: both finish (the databases are locked in address order) and every result is exact."""
    pv, kfs, bows, qs = world["pv"], world["kfs"], world["bows"], world["qs"]
    voc = voc_of(M, pv)
    mt0 = M.ORBmatcher(NNRATIO, True)
    dbs = [M.KeyFrameDatabase(mt0), M.KeyFrameDatabase(mt0)]
    for s, (kf, b) in enumerate(zip(kfs, bows)):
        dbs[s % 2].add(kf, b)
    slots = [[0, 3, 5, 8, 11, 3], [1, 2, 4, 10, 13, 22]]
    frames0 = [resident(M, mt0, qs[q].mvKeysUn, qs[q].mDescriptors) for q in (0, 1)]
    mt0.ComputeBoWBatch(voc, frames0, LEVELSUP, want_host=False)
    want_q = mt0.KfdbQueryBatch(dbs, frames0)
    want_s = [blocks(r) for r in mt0.SearchByBoWDbBatch(dbs, slots, frames0)]
    for j in (0, 1):
        so = [oracle.port_bow_score(world["q_bows"][j], bows[s]) for s in range(j, N_KF, 2)]
        assert np.array_equal(want_q[j][0], [x[1] for x in so]) and np.array_equal(want_q[j][1], np.float32([x[0] for x in so]))
        for s, b in zip(slots[j], want_s[j]):
            n_o, m_o = oracle.port_search_by_bow(kfs[2 * s + j], qs[j], NNRATIO, True)
            assert len(b) == n_o and np.array_equal(dense(b, len(qs[j].mvKeysUn)), m_o), (j, s)
    bad = []

    def worker(order, reps):
        mt = M.ORBmatcher(NNRATIO, True)
        frames = [resident(M, mt, qs[q].mvKeysUn, qs[q].mDescriptors) for q in (0, 1)]
        mt.ComputeBoWBatch(voc, frames, LEVELSUP, want_host=False)
        for r in range(reps):
            got_q = mt.KfdbQueryBatch([dbs[j] for j in order], [frames[j] for j in order])
            got_s = mt.SearchByBoWDbBatch([dbs[j] for j in order], [slots[j] for j in order], [frames[j] for j in order])
            for j, gq, gs in zip(order, got_q, got_s):
                if not all(np.array_equal(a, b) for a, b in zip(gq, want_q[j])):
                    bad.append(("query", order, r, j))
                if not all(np.array_equal(a, b) for a, b in zip(blocks(gs), want_s[j])):
                    bad.append(("search", order, r, j))

    errors = run_threads([(worker, ((0, 1), 200)), (worker, ((1, 0), 200))])
    assert not errors, errors
    assert not bad, f"{len(bad)} results differ, e.g. {bad[:6]}"


# ------------------------------------------------------------------------------------------------------ 3. single-threaded contracts
def test_set_has_mp_batch(M, oracle, world):
    """borb_kfdb_set_has_mp_batch equals the same updates made one at a time, the last mask of a repeated slot wins, n = 0 changes
    nothing, and a batch with one bad entry anywhere (an erased slot, a slot out of range, a NULL mask) is refused whole."""
    from orb_slam2_b200._lib import BorbError
    kfs, bows, qs = world["kfs"][:12], world["bows"][:12], world["qs"]
    rng = np.random.default_rng(9)
    mt = M.ORBmatcher(NNRATIO, True)
    a, b = M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt)
    for kf, bow in zip(kfs, bows):
        a.add(kf, bow); b.add(kf, bow)
    mask = lambda s, p=0.5: (rng.random(len(kfs[s].mvKeysUn)) < p).astype(np.uint8)
    F = M.KeyFrameView(qs[0].mvKeysUn, qs[0].mDescriptors, qs[0].mFeatVec)
    every = list(range(12))

    def searches(db):
        return blocks(db.SearchByBoWPairs(every, F)) + blocks(db.SearchByBoWKFPairs(7, every)) + blocks(db.SearchByBoWKFPairs(4, every))

    def same(x, y):
        return len(x) == len(y) and all(np.array_equal(p, q) for p, q in zip(x, y))

    current = {s: kfs[s].has_mp for s in every}
    upd = {3: mask(3), 7: mask(7), 8: mask(8), 11: mask(11)}
    a.set_has_mp_batch(list(upd), list(upd.values()))
    for s, m in upd.items():
        b.set_has_mp(s, m)
    current.update(upd)
    assert same(searches(a), searches(b))
    got = blocks(a.SearchByBoWPairs(every, F))
    for s in every:
        n_o, m_o = oracle.port_search_by_bow(with_mask(M, kfs[s], current[s]), F, NNRATIO, True)
        assert len(got[s]) == n_o and np.array_equal(dense(got[s], len(F.mvKeysUn)), m_o), s
    assert sum(len(x) for x in got) > 50
    # repeated slots: the last mask wins
    m1, m2 = mask(4), mask(4)
    a.set_has_mp_batch([4, 9, 4], [m1, kfs[9].has_mp, m2])
    b.set_has_mp(4, m2)
    current[4] = m2
    assert same(searches(a), searches(b))
    # n = 0 is a no-op
    before = searches(a)
    a.set_has_mp_batch([], [])
    assert same(searches(a), before)
    # one bad entry anywhere refuses the whole batch; the good entries (all-empty masks) would change every search
    a.erase(2); b.erase(2)
    every = [s for s in every if s != 2]
    before = searches(a)
    assert same(before, searches(b))
    zero = {s: np.zeros(len(kfs[s].mvKeysUn), np.uint8) for s in range(12)}
    for bad_slot, bad_mask in ((2, zero[2]), (12, zero[0]), (-1, zero[0]), (5, None)):
        for pos in (0, 2, 4):
            sl, ms = [3, 7, 11, 4], [zero[3], zero[7], zero[11], zero[4]]
            sl.insert(pos, bad_slot); ms.insert(pos, bad_mask)
            with pytest.raises(BorbError) as ei:
                a.set_has_mp_batch(sl, ms)
            assert ei.value.status == 1, (bad_slot, pos)
            assert same(searches(a), before), (bad_slot, pos)
    a.set_has_mp_batch([3, 7, 11, 4], [zero[3], zero[7], zero[11], zero[4]])
    assert not same(searches(a), before)


def test_last_error_is_per_thread(M, world):
    """Two threads trigger different argument refusals, made before any launch, over and over: each reads its own
    borb_last_error text."""
    from orb_slam2_b200 import _lib
    lib = _lib.load()
    mt = M.ORBmatcher(NNRATIO, True)
    db = M.KeyFrameDatabase(mt)
    db.add(world["kfs"][0], world["bows"][0])
    bad = []

    def erase(reps):
        for r in range(reps):
            st = lib.borb_kfdb_erase(db._h, 1000 + r)
            if st != 1 or lib.borb_last_error() != b"bad keyframe slot":
                bad.append(("erase", r, st, lib.borb_last_error()))

    def add(reps):
        kf = world["kfs"][1]
        kc = kf._c()
        w, v, slot = np.array([9, 5], np.uint32), np.array([0.5, 0.5]), C.c_int32(-1)
        for r in range(reps):
            st = lib.borb_kfdb_add(db._h, C.byref(kc), w.ctypes.data, v.ctypes.data, 2, C.byref(slot))
            if st != 1 or lib.borb_last_error() != b"BowVector words must ascend (std::map order)":
                bad.append(("add", r, st, lib.borb_last_error()))

    errors = run_threads([(erase, (3000,)), (add, (3000,))])
    assert not errors, errors
    assert not bad, f"{len(bad)} calls read another thread's error, e.g. {bad[:4]}"
    assert db.size()[0] == 1


def test_frames_from_extractor_between_enqueues(M):
    """borb_extract_batch_enqueue of batch A, borb_frames_from_extractor on a matcher, then batch B enqueued on the same extractor,
    with no borb_sync in between: the frames hold batch A (the matcher's stream waits for A, B's kernels wait for the frame build)
    and the extractor's outputs are batch B's."""
    from orb_slam2_b200 import _lib as L
    from orb_slam2_b200.extractor import ORBextractor
    K = (517.3, 516.5, 318.6, 255.3)
    lib = L.load()
    w, h, n = 640, 480, 3
    A = np.stack([synth.mono_frame(700 + i, 0, 0, w, h) for i in range(n)])
    B = np.stack([synth.mono_frame(800 + i, 0, 0, w, h) for i in range(n)])
    X0, mt0 = ORBextractor(1000), M.ORBmatcher(NNRATIO, True)
    want_a = X0.extract_batch(list(A))
    frames0, _ = M.frames_from_extractor(mt0, X0, list(range(n)), [len(k) for k, _ in want_a], K)
    read_a = [f.resident.read(stereo=False) for f in frames0]
    want_b = X0.extract_batch(list(B))
    assert all(len(k) > 500 for k, _ in want_a + want_b)

    X, mt = ORBextractor(1000), M.ORBmatcher(NNRATIO, True)
    cap = X.capacity(w, h)
    held = []

    def pinned(shape, dtype):
        p = C.c_void_p()
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        L.check(lib.borb_host_alloc(C.byref(p), nbytes), "borb_host_alloc")
        held.append(p)
        return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p.value)).view(dtype).reshape(shape)

    try:
        outs = [(pinned((n, cap), L.KP_DTYPE), pinned((n, cap, 32), np.uint8), pinned((n,), np.int32)) for _ in range(2)]
        for rounds in range(3):
            for o in outs:
                for a in o:
                    a[...] = 0
            for (kps, desc, cnt), imgs in zip(outs, (A, B)):
                ptrs = (C.c_void_p * n)(*[imgs[i].ctypes.data for i in range(n)])
                L.check(lib.borb_extract_batch_enqueue(X._h, ptrs, n, w, h, w, L.ptr(kps), L.ptr(desc), cap, L.ptr(cnt)),
                        "borb_extract_batch_enqueue")
                if imgs is A:
                    frames, _ = M.frames_from_extractor(mt, X, list(range(n)), [len(k) for k, _ in want_a], K, want_host=False)
            L.check(lib.borb_sync(X._h), "borb_sync")
            for i, f in enumerate(frames):
                got = f.resident.read(stereo=False)
                for key in ("keys_un", "desc", "cell_start", "cell_idx"):
                    assert np.array_equal(got[key], read_a[i][key]), (rounds, i, key)
                f.resident.close()
            for (kps, desc, cnt), want in zip(outs, (want_a, want_b)):
                for i, (k, d) in enumerate(want):
                    assert cnt[i] == len(k) and np.array_equal(kps[i, :cnt[i]], k) and np.array_equal(desc[i, :cnt[i]], d), i
    finally:
        for p in held:
            lib.borb_host_free(p)
