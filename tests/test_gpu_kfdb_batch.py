"""GPU parity of the relocalisation step of Tracking::Track() for many camera streams on resident frames:
borb_kfdb_query_batch (KeyFrameDatabase query) must equal borb_kfdb_query and the oracle's score, job by job, bit for bit, and
borb_search_by_bow_db_batch (SearchByBoW(KeyFrame*, Frame&) against database keyframes) must equal borb_search_by_bow_db_pairs
on host views of the same frames, keyframe by keyframe.  Both are a fixed number of launches whatever the batch size, and
argument errors are refused before anything is launched, naming the job."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from orb_slam2_b200 import synth

pytestmark = pytest.mark.gpu

SCALE = (1.2 ** np.arange(8)).astype(np.float32)


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def resident(M, mt, keys, desc):
    hi_x = float(max(640.0, keys["x"].max() + 1)) if len(keys) else 640.0
    hi_y = float(max(480.0, keys["y"].max() + 1)) if len(keys) else 480.0
    return M.FrameView(keys, np.ascontiguousarray(desc, np.uint8), SCALE, (0.0, 0.0, hi_x, hi_y)).make_resident(mt)


def flip_bits(rng, d, p):
    flip = rng.random((len(d), 32, 8)) < p
    return d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)


def random_keys(rng, n):
    from orb_slam2_b200._lib import KP_DTYPE
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(20, 600, n).astype(np.float32); k["y"] = rng.uniform(20, 440, n).astype(np.float32)
    k["angle"] = rng.uniform(0, 360, n).astype(np.float32); k["size"] = 31.0; k["octave"] = 0; k["class_id"] = -1
    return k


def host_view(M, keys, desc, fv):
    return M.KeyFrameView(mvKeysUn=keys, mDescriptors=desc, mFeatVec=fv)


def same_blocks(got, want):
    """(nmatches, pair_offset, pairs) of two searches: equal counts and equal per-keyframe pair blocks."""
    (nm, off, pairs), (nm2, off2, pairs2) = got, want
    assert np.array_equal(nm, nm2)
    assert int(nm.sum()) == len(pairs)
    for k in range(len(nm)):
        assert np.array_equal(pairs[off[k]:off[k] + nm[k]], pairs2[off2[k]:off2[k] + nm2[k]]), k


def dense(nm, off, pairs, n_f):
    out = np.full((len(nm), n_f), -1, np.int32)
    for k in range(len(nm)):
        pr = pairs[off[k]:off[k] + nm[k]]
        out[k, (pr & 0xFFFF).astype(np.int64)] = (pr >> 16).astype(np.int32)
    return out


@pytest.fixture(scope="module")
def scenes():
    """Extracted 640x480 frames: triples share a scene (the keyframes), and noisy re-observations of some scenes (the queries)."""
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(800)
    rng = np.random.default_rng(3)
    base = [synth.mono_frame(200 + i // 3, 0, 0, 640, 480) for i in range(36)]
    imgs = [np.clip(b.astype(np.int32) + rng.integers(-6, 7, b.shape), 0, 255).astype(np.uint8) for b in base]
    kf = X.extract_batch(imgs)
    qimgs = [np.clip(base[i].astype(np.int32) + rng.integers(-8, 9, base[i].shape), 0, 255).astype(np.uint8) for i in (7, 20, 31, 4)]
    q = X.extract_batch(qimgs)
    return dict(kf=kf, q=q, base=base)


def voc_of(M, pv):
    e = pv.export()
    return M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])


def build_db(M, mt, voc, outs, levelsup, rng, erase=()):
    db = M.KeyFrameDatabase(mt)
    kfs, bows = [], []
    for k, d in outs:
        bow, fv = voc.transform(d, levelsup)
        kv = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.7).astype(np.uint8))
        db.add(kv, bow)
        kfs.append(kv); bows.append(bow)
    for s in erase:
        db.erase(s)
    return db, kfs, bows


def test_query_batch_equals_single_queries_and_oracle(M, oracle, scenes):
    pv = oracle.PortVocabulary.random(10, 4, 5)
    voc = voc_of(M, pv)
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(5)
    dbA, _, bowsA = build_db(M, mt, voc, scenes["kf"][:24], 2, rng)
    dbB, _, bowsB = build_db(M, mt, voc, scenes["kf"][18:36], 2, rng, erase=(3, 10))
    dbE = M.KeyFrameDatabase(mt)
    big_d = flip_bits(rng, np.concatenate([d for _, d in scenes["kf"][:12]])[:8192], 0.03)
    assert len(big_d) == 8192
    sets = [(k, d) for k, d in scenes["q"]] + [(scenes["q"][0][0][:0], scenes["q"][0][1][:0]), (random_keys(rng, 8192), big_d)]
    frames = [resident(M, mt, k, d) for k, d in sets]
    host = mt.ComputeBoWBatch(voc, frames, 2)
    assert len(host[4][0]) == 0 and len(host[5][1].feat_idx) == 8192
    jobs = [(dbA, 0), (dbA, 1), (dbB, 2), (dbA, 3), (dbE, 0), (dbA, 4), (dbB, 5), (dbB, 0)]
    c0 = launches(mt)
    got = mt.KfdbQueryBatch([d for d, _ in jobs], [frames[f] for _, f in jobs])
    assert launches(mt) - c0 == 1
    for j, ((db, f), (cw, sc, fw)) in enumerate(zip(jobs, got)):
        cw1, sc1, fw1 = db.query(host[f][0])
        assert np.array_equal(cw, cw1) and np.array_equal(sc, sc1) and np.array_equal(fw, fw1), j
        bows = bowsA if db is dbA else (bowsB if db is dbB else [])
        assert len(cw) == len(bows)
        for s, b in enumerate(bows):
            if db is dbB and s in (3, 10):
                assert cw[s] == 0 and fw[s] == 0xFFFFFFFF
                continue
            so, co, fo = oracle.port_bow_score(host[f][0], b)
            assert cw[s] == co and fw[s] == fo and sc[s] == np.float32(so), (j, s)
    assert len(got[4][0]) == 0 and np.all(got[5][0] == 0) and got[0][0].max() > 20
    # one launch whatever the number of jobs
    many = [frames[i % 4] for i in range(32)]
    c0 = launches(mt)
    assert len(mt.KfdbQueryBatch(dbA, many)) == 32
    assert launches(mt) - c0 == 1


def test_relocalization_candidates_in_job_order(M, oracle, scenes, tmp_path):
    """relocalization_candidates applied to the jobs in job order with the database's persistent mRelocScore dict gives what the
    same queries give as sequential DetectRelocalizationCandidates calls, and what the verbatim KeyFrameDatabase.cc gives."""
    pv = oracle.PortVocabulary.random(10, 3, 5)
    voc = voc_of(M, pv)
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(11)
    outs = scenes["kf"][:30]
    db, _, bows = build_db(M, mt, voc, outs, 2, rng)
    db_seq, _, _ = build_db(M, mt, voc, outs, 2, np.random.default_rng(11))
    n_kf = len(outs)
    neigh = np.full((n_kf, 10), -1, np.int32)
    for s in range(n_kf):
        nb = [x for x in (s - 2, s - 1, s + 1, s + 2) if 0 <= x < n_kf] + rng.integers(0, n_kf, 4).tolist()
        nb = [x for x in dict.fromkeys(nb) if x != s][:10]
        neigh[s, :len(nb)] = nb
    covis = lambda s: [int(x) for x in neigh[s] if x >= 0]
    qsets = list(scenes["q"]) + [(k, flip_bits(rng, d, 0.05)) for k, d in scenes["kf"][2:30:4]]
    frames = [resident(M, mt, k, d) for k, d in qsets]
    host = mt.ComputeBoWBatch(voc, frames, 2)
    got = mt.KfdbQueryBatch(db, frames)
    lists = [M.relocalization_candidates(cw, sc, fw, db._seq, covis, db._reloc_score) for cw, sc, fw in got]
    want = [db_seq.DetectRelocalizationCandidates(h[0], covis) for h in host]
    assert lists == want and sum(len(x) for x in lists) > 10
    if oracle.have_dbowref():
        path = tmp_path / "voc.txt"
        pv.save_text(str(path))
        path.write_text(path.read_text().rstrip("\n"))      # see tests/test_oracle_dbow_ref.py: the reference loader's trailing-newline quirk
        rv = oracle.RefVocabulary(path)
        assert rv.reloc_sequence(bows, [h[0] for h in host], neigh) == lists


def search_world(M, oracle, scenes, ori):
    """Databases at levelsup 1-4, a 6000-feature frame whose block does not fit in shared memory, and the search jobs of one call."""
    pv = oracle.PortVocabulary.random(10, 4, 5)
    voc = voc_of(M, pv)
    mt = M.ORBmatcher(0.75, ori)
    rng = np.random.default_rng(17)
    dbs = {L: build_db(M, mt, voc, scenes["kf"][:9], L, rng) for L in (1, 2, 3, 4)}   # scenes 0-2
    # the large frame: random descriptors, keyframes derived from it by bit flips so that real matches exist
    qd = rng.integers(0, 256, (6000, 32), dtype=np.uint8)
    qk = random_keys(rng, 6000)
    big_db = M.KeyFrameDatabase(mt)
    big_kfs = []
    for n, p in ((1500, 0.03), (900, 0.06), (2400, 0.02)):
        src = rng.choice(6000, n, replace=False)
        k = random_keys(rng, n)
        k["angle"] = (qk["angle"][src] + rng.choice([0.0, 0.0, 0.0, 95.0], n)).astype(np.float32) % np.float32(360)
        d = flip_bits(rng, qd[src], p)
        bow, fv = voc.transform(d, 2)
        kv = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(n) < 0.7).astype(np.uint8))
        big_db.add(kv, bow); big_kfs.append(kv)
    q = scenes["q"]
    # (levelsup, frame keys, frame desc, database, slots)
    specs = [(2, q[0][0], q[0][1], "2", [6, 3, 3, 7, 1, 6]),        # repeated slots (q[0] re-observes scene 2, q[3] scene 1)
             (2, q[3][0], q[3][1], "2", None),                      # full sweep
             (1, q[0][0], q[0][1], "1", None),                      # ~1000 single-feature nodes
             (3, q[3][0], q[3][1], "3", [2, 4, 7]),                 # ~10 nodes of ~80: buckets wider than 32
             (4, q[0][0], q[0][1], "4", None),                      # one node with every feature
             (2, q[0][0][:0], q[0][1][:0], "2", [1, 2]),             # a frame without features
             (2, q[0][0], q[0][1], "2", []),                        # n_kf == 0
             (2, qk, qd, "big", None)]                              # frame block in global memory
    frames_by_L = {}
    for j, (L, k, d, _, _) in enumerate(specs):
        frames_by_L.setdefault(L, []).append((j, resident(M, mt, k, d)))
    frames, host_F = [None] * len(specs), [None] * len(specs)
    for L, lst in frames_by_L.items():
        bows = mt.ComputeBoWBatch(voc, [f for _, f in lst], L)
        for (j, f), (_, fv) in zip(lst, bows):
            frames[j] = f
            host_F[j] = host_view(M, specs[j][1], specs[j][2], fv)
    db_of = lambda key: big_db if key == "big" else dbs[int(key)][0]
    kfs_of = lambda key: big_kfs if key == "big" else dbs[int(key)][1]
    return mt, specs, frames, host_F, db_of, kfs_of


@pytest.mark.parametrize("ori", [True, False])
def test_search_batch_equals_single_calls_and_oracle(M, oracle, scenes, ori):
    mt, specs, frames, host_F, db_of, kfs_of = search_world(M, oracle, scenes, ori)
    dbs = [db_of(s[3]) for s in specs]
    slots = [s[4] for s in specs]
    c0 = launches(mt)
    got = mt.SearchByBoWDbBatch(dbs, slots, frames)
    assert launches(mt) - c0 == 3
    for j, (g, db, sl, F) in enumerate(zip(got, dbs, slots, host_F)):
        single = db.SearchByBoWPairs(sl, F)
        same_blocks(g, single)
        kfs = kfs_of(specs[j][3])
        sl_all = list(range(len(kfs))) if sl is None else sl
        assert len(g[0]) == len(sl_all)
        if j in (0, 3, 7) or (j == 2 and not ori):                   # a sample against the restated SearchByBoW
            dn = dense(*g, len(F.mvKeysUn))
            for i, s in enumerate(sl_all):
                n_o, m_o = oracle.port_search_by_bow(kfs[s], F, 0.75, ori)
                assert g[0][i] == n_o and np.array_equal(dn[i], m_o), (j, s)
        if oracle.have_matchref() and j == 1:
            dn = dense(*g, len(F.mvKeysUn))
            for i, s in enumerate(sl_all):
                n_r, m_r = oracle.ref_search_by_bow(kfs[s], F, 0.75, ori)
                assert g[0][i] == n_r and np.array_equal(dn[i], m_r), (j, s)
    assert np.all(got[5][0] == 0) and len(got[5][0]) == 2 and len(got[6][0]) == 0
    assert got[0][0][1] == got[0][0][2] and got[0][0].max() > 10 and got[7][0][0] > 100 and got[4][0].max() > 10
    # 3 launches whatever the number of jobs
    for n in (1, 32):
        c0 = launches(mt)
        mt.SearchByBoWDbBatch([dbs[1]] * n, [None] * n, [frames[1]] * n)
        assert launches(mt) - c0 == 3


def test_set_has_mp_and_erase_between_batches(M, oracle, scenes):
    mt, specs, frames, host_F, db_of, kfs_of = search_world(M, oracle, scenes, True)
    db, kfs = db_of("2"), kfs_of("2")
    before = mt.SearchByBoWDbBatch([db, db], [None, [7, 5]], [frames[1], frames[0]])
    hm = np.zeros(len(kfs[7].mvKeysUn), np.uint8); hm[::2] = 1
    db.set_has_mp(7, hm)
    db.erase(5)
    after = mt.SearchByBoWDbBatch([db, db], [None, [7]], [frames[1], frames[0]])
    kf7 = dataclasses.replace(kfs[7], has_mp=hm)
    for g, F in ((after[0], host_F[1]),):
        same_blocks(g, db.SearchByBoWPairs(None, F))
        assert g[0][5] == 0
    n_o, m_o = oracle.port_search_by_bow(kf7, host_F[0], 0.75, True)
    assert after[1][0][0] == n_o and np.array_equal(dense(*after[1], len(host_F[0].mvKeysUn))[0], m_o)
    assert after[1][0][0] != before[1][0][0] and before[0][0][5] > 0


def test_relocalisation_chain_on_resident_stereo_frames(M, oracle):
    """stereo_frames -> frames_from_extractor (mode 1) -> frames_compute_bow -> kfdb_query_batch -> host candidates ->
    search_by_bow_db_batch, against the same chain through the single calls on host views and the oracle."""
    from orb_slam2_b200.extractor import ORBextractor
    from orb_slam2_b200 import sharding
    arrs = sharding.random_vocabulary_arrays(10, 6, 7)
    voc = M.ORBVocabulary.from_arrays(*arrs, 10, 6)
    X = ORBextractor(1200)
    bf, fx = 47.9, 435.2
    K = (fx, fx, 376.0, 240.0)
    pairs = [synth.stereo_pair(80 + i, 0, 0, 752, 480) for i in range(10)]
    res = X.stereo_frames([p[0] for p in pairs[:6]], [p[1] for p in pairs[:6]], bf, fx)
    rng = np.random.default_rng(23)
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    kfs = []
    for r in res:                                              # keyframes: the first six left views, twice with bit noise
        for p in (0.0, 0.04):
            d = flip_bits(rng, r["mDescriptors"], p)
            bow, fv = voc.transform(d, 4)
            kv = M.KeyFrameView(mvKeysUn=r["mvKeys"], mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(d)) < 0.8).astype(np.uint8))
            db.add(kv, bow); kfs.append(kv)
    n_kf = len(kfs)
    covis = lambda s: [x for x in (s - 1, s + 1, s + 2) if 0 <= x < n_kf]
    lost = X.stereo_frames([p[0] for p in pairs[1:5]], [p[1] for p in pairs[1:5]], bf, fx)
    frames, host = M.frames_from_extractor(mt, X, [0, 2, 4, 6], [len(r["mvKeys"]) for r in lost], K, bf=bf, mode=1)
    bows = mt.ComputeBoWBatch(voc, frames, 4)
    q = mt.KfdbQueryBatch(db, frames)
    state = {}
    cands = [M.relocalization_candidates(cw, sc, fw, db._seq, covis, state) for cw, sc, fw in q]
    assert all(len(c) > 0 for c in cands)
    got = mt.SearchByBoWDbBatch(db, cands, frames)
    for j, (r, (bow, fv)) in enumerate(zip(lost, bows)):
        F = host_view(M, host["keys_un"][j], r["mDescriptors"], fv)
        assert np.array_equal(host["keys_un"][j], r["mvKeys"])
        assert db.DetectRelocalizationCandidates(bow, covis) == cands[j]
        same_blocks(got[j], db.SearchByBoWPairs(cands[j], F))
        dn = dense(*got[j], len(F.mvKeysUn))
        for i, s in enumerate(cands[j]):
            n_o, m_o = oracle.port_search_by_bow(kfs[s], F, 0.75, True)
            assert got[j][0][i] == n_o and np.array_equal(dn[i], m_o), (j, s)
    assert max(int(g[0].max()) for g in got) > 100


def test_refusals_name_the_job_and_launch_nothing(M, oracle, scenes):
    from orb_slam2_b200 import _lib
    from orb_slam2_b200._lib import BorbError
    pv = oracle.PortVocabulary.random(10, 4, 5)
    voc = voc_of(M, pv)
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(29)
    db, kfs, _ = build_db(M, mt, voc, scenes["kf"][:9], 2, rng, erase=(4,))
    q = scenes["q"][0]
    good = resident(M, mt, q[0], q[1])
    (_, fv), = mt.ComputeBoWBatch(voc, [good], 2)
    F = host_view(M, q[0], q[1], fv)

    def refused(call, job, status=1):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        assert ei.value.status == status and str(ei.value).split(": ", 2)[2].startswith(f"job {job}:"), str(ei.value)
        assert launches(mt) == c0

    no_bow = resident(M, mt, q[0], q[1])
    for fr, job in ((no_bow, 1), (None, 2)):
        refused(lambda: mt.KfdbQueryBatch([db] * 3, [good, fr if job == 1 else good, fr if job == 2 else good]), job)
        refused(lambda: mt.SearchByBoWDbBatch([db] * 3, [[0, 1]] * 3, [good, fr if job == 1 else good, fr if job == 2 else good]), job)
    refused(lambda: mt.KfdbQueryBatch([db, None], [good, good]), 1)
    refused(lambda: mt.SearchByBoWDbBatch([db, None], [None, None], [good, good]), 1)
    # a recycled frame block starts without BoW
    old = resident(M, mt, q[0], q[1])
    mt.ComputeBoWBatch(voc, [old], 2, want_host=False)
    old.resident.close()
    recycled = resident(M, mt, q[0], q[1])
    refused(lambda: mt.SearchByBoWDbBatch([db, db], [[0], [0]], [good, recycled]), 1)
    refused(lambda: mt.KfdbQueryBatch([db, db], [good, recycled]), 1)
    # slots: erased, out of range, NULL with the wrong count
    refused(lambda: mt.SearchByBoWDbBatch([db] * 2, [[0, 1], [2, 4]], [good, good]), 1)
    refused(lambda: mt.SearchByBoWDbBatch([db] * 3, [[0], [0], [9]], [good] * 3), 2)
    jobs = (M._BowDbJobC * 2)()
    nm = np.zeros(16, np.int32); off = np.zeros(16, np.int32); pairs = np.zeros(64, np.uint32); tot = np.zeros(1, np.int32)
    for j in range(2):
        jobs[j].db, jobs[j].frame, jobs[j].n_kf = db._h.value, good.resident._h.value, 9
        jobs[j].n_matches, jobs[j].pair_offset, jobs[j].pairs, jobs[j].pairs_cap, jobs[j].n_pairs_total = nm.ctypes.data, off.ctypes.data, pairs.ctypes.data, 64, tot.ctypes.data
    jobs[1].n_kf = 8                                           # slots == NULL: n_kf must be the slot count
    refused(lambda: _lib.check(mt._lib.borb_search_by_bow_db_batch(mt._h, jobs, 2, mt.mfNNratio, 1), "batch"), 1)
    jobs[1].n_kf = 9
    jobs[1].pair_offset = None                                 # pairs without pair_offset
    refused(lambda: _lib.check(mt._lib.borb_search_by_bow_db_batch(mt._h, jobs, 2, mt.mfNNratio, 1), "batch"), 1)
    # capacity: a query output smaller than the database, and pairs beyond one job's pairs_cap
    qjobs = (M._KfdbQueryJobC * 2)()
    cw = np.zeros(9, np.int32); sc = np.zeros(9, np.float32); fw = np.zeros(9, np.uint32); ns = np.zeros(1, np.int32)
    for j in range(2):
        qjobs[j].db, qjobs[j].frame = db._h.value, good.resident._h.value
        qjobs[j].common_words, qjobs[j].score, qjobs[j].first_word, qjobs[j].cap, qjobs[j].n_slots = cw.ctypes.data, sc.ctypes.data, fw.ctypes.data, 9, ns.ctypes.data
    qjobs[1].cap = 8
    refused(lambda: _lib.check(mt._lib.borb_kfdb_query_batch(mt._h, qjobs, 2), "query"), 1, status=5)
    want_nm = db.SearchByBoWPairs(None, F)[0]
    assert want_nm.sum() > 4
    outs = [(np.zeros(9, np.int32), np.zeros(9, np.int32), np.zeros(512 * 9, np.uint32), np.zeros(1, np.int32)) for _ in range(3)]
    cjobs = (M._BowDbJobC * 3)()
    for j, (nm_j, off_j, pairs_j, tot_j) in enumerate(outs):
        cjobs[j].db, cjobs[j].frame, cjobs[j].n_kf = db._h.value, good.resident._h.value, 9
        cjobs[j].n_matches, cjobs[j].pair_offset, cjobs[j].pairs, cjobs[j].n_pairs_total = nm_j.ctypes.data, off_j.ctypes.data, pairs_j.ctypes.data, tot_j.ctypes.data
        cjobs[j].pairs_cap = [512 * 9, int(want_nm.sum()) - 1, int(want_nm.sum()) - 2][j]
    c0 = launches(mt)
    with pytest.raises(BorbError) as ei:
        _lib.check(mt._lib.borb_search_by_bow_db_batch(mt._h, cjobs, 3, mt.mfNNratio, 1), "batch")
    assert ei.value.status == 5 and "job 1:" in str(ei.value) and launches(mt) - c0 == 3
    for nm_j, off_j, pairs_j, tot_j in outs:                   # counts and offsets are valid for every job
        assert np.array_equal(nm_j, want_nm) and tot_j[0] == want_nm.sum()
    same_blocks((outs[0][0], outs[0][1], outs[0][2][:tot_j[0]]), db.SearchByBoWPairs(None, F))
    # the handle still gives correct results
    got = mt.SearchByBoWDbBatch(db, [None, [0, 3]], [good, good])
    same_blocks(got[0], db.SearchByBoWPairs(None, F))
    same_blocks(got[1], db.SearchByBoWPairs([0, 3], F))
    cw1, sc1, fw1 = mt.KfdbQueryBatch(db, [good])[0]
    cw2, sc2, fw2 = db.query(mt.ComputeBoWBatch(voc, [good], 2)[0][0])
    assert np.array_equal(cw1, cw2) and np.array_equal(sc1, sc2) and np.array_equal(fw1, fw2)
