"""GPU parity of the device-resident keyframe database (KeyFrameDatabase + SearchByBoW against resident keyframes)
with the restatements in oracle/orb_port_match.cpp: shared-word counts, L1 scores (bit-exact as float), candidate
lists of DetectRelocalizationCandidates, and SearchByBoW results."""
import numpy as np
import pytest

from orb_slam2_b200 import synth

pytestmark = pytest.mark.gpu

N_KF = 48


@pytest.fixture(scope="module")
def world(oracle):
    from orb_slam2_b200 import matcher as M
    from orb_slam2_b200.extractor import ORBextractor
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    X = ORBextractor(800)
    rng = np.random.default_rng(3)
    base = [synth.mono_frame(200 + i // 3, 0, 0, 640, 480) for i in range(N_KF)]      # triples of frames share a scene
    imgs = [np.clip(b.astype(np.int32) + rng.integers(-6, 7, b.shape), 0, 255).astype(np.uint8) for b in base]
    outs = X.extract_batch(imgs)
    kfs, bows = [], []
    for k, d in outs:
        bow, fv = voc.transform(d, 2)
        kfs.append(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.7).astype(np.uint8)))
        bows.append(bow)
    qimg = np.clip(base[7].astype(np.int32) + rng.integers(-8, 9, base[7].shape), 0, 255).astype(np.uint8)
    qk, qd = X(qimg)
    qbow, qfv = voc.transform(qd, 2)
    F = M.KeyFrameView(mvKeysUn=qk, mDescriptors=qd, mFeatVec=qfv)
    return dict(M=M, voc=voc, kfs=kfs, bows=bows, F=F, qbow=qbow, n_words=int(e["is_leaf"].sum()) + len(e["is_leaf"]))


def test_query_counts_and_scores_match_oracle(world, oracle):
    M = world["M"]
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    slots = [db.add(kf, bow) for kf, bow in zip(world["kfs"], world["bows"])]
    assert slots == list(range(N_KF)) and db.size()[0] == N_KF and db.size()[1] > 0
    cw, sc, fw = db.query(world["qbow"])
    for s in range(N_KF):
        so, co, fo = oracle.port_bow_score(world["qbow"], world["bows"][s])
        assert cw[s] == co and fw[s] == fo, s
        assert sc[s] == np.float32(so), (s, sc[s], so)                    # bit-exact: terms are added in word order
    assert cw.max() > 20 and int(np.argmax(sc)) in (6, 7, 8)                # the query's own scene scores highest
    # erase: the slot stops matching, the others are unchanged
    db.erase(7)
    cw2, sc2, fw2 = db.query(world["qbow"])
    assert cw2[7] == 0 and fw2[7] == 0xFFFFFFFF
    keep = np.arange(N_KF) != 7
    assert np.array_equal(cw2[keep], cw[keep]) and np.array_equal(sc2[keep], sc[keep])
    with pytest.raises(Exception):
        db.erase(7)
    # empty query, empty database
    cw3, sc3, _ = db.query({})
    assert np.all(cw3 == 0) and np.all(sc3 == 0)
    db.clear()
    assert db.size()[0] == 0 and len(db.query(world["qbow"])[0]) == 0


def test_relocalization_candidates_match_oracle(world, oracle):
    M = world["M"]
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    for kf, bow in zip(world["kfs"], world["bows"]):
        db.add(kf, bow)
    rng = np.random.default_rng(11)
    neigh = np.full((N_KF, 10), -1, np.int32)
    for s in range(N_KF):
        nb = [x for x in (s - 2, s - 1, s + 1, s + 2) if 0 <= x < N_KF] + rng.integers(0, N_KF, 3).tolist()
        nb = [x for x in dict.fromkeys(nb) if x != s][:10]
        neigh[s, :len(nb)] = nb
    covis = lambda s: [int(x) for x in neigh[s] if x >= 0]
    for q in (world["qbow"], world["bows"][20], world["bows"][41]):
        got = db.DetectRelocalizationCandidates(q, covis)
        want = oracle.port_detect_reloc_candidates(world["bows"], world["n_words"], q, neigh)
        assert got == want.tolist() and len(got) >= 1, (got, want)


def test_loop_candidates_match_oracle(world, oracle):
    """KeyFrameDatabase::DetectLoopCandidates (src/KeyFrameDatabase.cc:76-197) from the GPU query + the host logic."""
    M = world["M"]
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    for kf, bow in zip(world["kfs"], world["bows"]):
        db.add(kf, bow)
    rng = np.random.default_rng(13)
    neigh = np.full((N_KF, 10), -1, np.int32)
    for s in range(N_KF):
        nb = [x for x in (s - 1, s + 1, s + 2) if 0 <= x < N_KF] + rng.integers(0, N_KF, 2).tolist()
        nb = [x for x in dict.fromkeys(nb) if x != s][:10]
        neigh[s, :len(nb)] = nb
    covis = lambda s: [int(x) for x in neigh[s] if x >= 0]
    for q, conn, min_score in ((world["qbow"], [6, 30], 0.0), (world["bows"][20], [19, 20, 21], 0.02), (world["bows"][41], [], 0.15)):
        connected = np.zeros(N_KF, np.uint8); connected[conn] = 1
        got = db.DetectLoopCandidates(q, conn, covis, min_score)
        want = oracle.port_detect_loop_candidates(world["bows"], world["n_words"], q, connected, neigh, min_score).tolist()
        assert got == want, (got, want)


def test_search_by_bow_against_resident_keyframes(world, oracle):
    M = world["M"]
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    for kf, bow in zip(world["kfs"], world["bows"]):
        db.add(kf, bow)
    F = world["F"]
    slots = [6, 7, 8, 20, 7, 47, 0]
    nm, match = db.SearchByBoW(slots, F)
    nm_h, match_h = mt.SearchByBoW([world["kfs"][s] for s in slots], F)          # same kernel, keyframes staged from the host
    assert np.array_equal(nm, nm_h) and np.array_equal(match, match_h)
    for i, s in enumerate(slots):
        n_o, m_o = oracle.port_search_by_bow(world["kfs"][s], F, 0.75, True)
        assert nm[i] == n_o and np.array_equal(match[i], m_o), s
    assert nm[1] > 30
    # MapPoint mask updated in place
    hm = np.zeros(len(world["kfs"][7].mvKeysUn), np.uint8); hm[::2] = 1
    db.set_has_mp(7, hm)
    kf7 = M.KeyFrameView(world["kfs"][7].mvKeysUn, world["kfs"][7].mDescriptors, world["kfs"][7].mFeatVec, has_mp=hm)
    nm2, match2 = db.SearchByBoW([7], F)
    n_o, m_o = oracle.port_search_by_bow(kf7, F, 0.75, True)
    assert nm2[0] == n_o and np.array_equal(match2[0], m_o)


def _pairs_to_dense(nm, off, pairs, n_f):
    out = np.full((len(nm), n_f), -1, np.int32)
    for k in range(len(nm)):
        pr = pairs[off[k]:off[k] + nm[k]]
        j, r = (pr & 0xFFFF).astype(np.int64), (pr >> 16).astype(np.int32)
        assert len(np.unique(j)) == len(j)
        out[k, j] = r
    return out


@pytest.mark.parametrize("levelsup", [1, 2, 3, 4])
def test_search_by_bow_pairs_all_bucket_shapes(oracle, levelsup):
    """The compact database search against the restated SearchByBoW for every bucket geometry of the kernel: levelsup 1 = ~1000
    single-feature nodes, 2 = ~100 nodes of ~8, 3 = 10 nodes of ~80 (multi-tile matrix), 4 = one node with every feature
    (direct evaluation); with and without the orientation cull."""
    from orb_slam2_b200 import matcher as M
    from orb_slam2_b200.extractor import ORBextractor
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    X = ORBextractor(800)
    rng = np.random.default_rng(17 + levelsup)
    base = [synth.mono_frame(300 + i // 3, 0, 0, 640, 480) for i in range(9)]
    imgs = [np.clip(b.astype(np.int32) + rng.integers(-6, 7, b.shape), 0, 255).astype(np.uint8) for b in base]
    outs = X.extract_batch(imgs)
    kfs, bows = [], []
    for k, d in outs:
        bow, fv = voc.transform(d, levelsup)
        kfs.append(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.6).astype(np.uint8)))
        bows.append(bow)
    qk, qd = X(np.clip(base[4].astype(np.int32) + rng.integers(-8, 9, base[4].shape), 0, 255).astype(np.uint8))
    qbow, qfv = voc.transform(qd, levelsup)
    F = M.KeyFrameView(mvKeysUn=qk, mDescriptors=qd, mFeatVec=qfv)
    for ori in (True, False):
        mt = M.ORBmatcher(0.75, ori)
        db = M.KeyFrameDatabase(mt)
        for kf, bow in zip(kfs, bows):
            db.add(kf, bow)
        nm, off, pairs = db.SearchByBoWPairs(None, F)
        dense = _pairs_to_dense(nm, off, pairs, len(qk))
        nm_d, dense_d = db.SearchByBoW(np.arange(len(kfs), dtype=np.int32), F)
        assert np.array_equal(nm, nm_d) and np.array_equal(dense, dense_d)
        for s in range(len(kfs)):
            n_o, m_o = oracle.port_search_by_bow(kfs[s], F, 0.75, ori)
            assert nm[s] == n_o and np.array_equal(dense[s], m_o), (levelsup, ori, s)
        assert nm.max() > 10
        # counts only, a slot subset with a repeat, and an erased slot
        nm2, _, none = db.SearchByBoWPairs([3, 4, 4, 0], F, want_pairs=False)
        assert none is None and np.array_equal(nm2, nm[[3, 4, 4, 0]])
        db.erase(2)
        nm3, off3, pairs3 = db.SearchByBoWPairs(None, F)
        assert nm3[2] == 0 and np.array_equal(np.delete(nm3, 2), np.delete(nm, 2))
        assert np.array_equal(_pairs_to_dense(nm3, off3, pairs3, len(qk))[[0, 1, 3, 8]], dense[[0, 1, 3, 8]])


def test_config4_real_size_2000_keyframes(oracle):
    """BASELINE configs[4] at its own size: EuRoC-shaped 752x480 @1200 features, k=10 L=6 vocabulary, 2000 resident keyframes.
    KeyFrameDatabase query (common words, L1 scores) and SearchByBoW against ALL keyframes equal the restated reference."""
    from orb_slam2_b200 import matcher as M, sharding
    from orb_slam2_b200.extractor import ORBextractor
    n_kf, n_src = 2000, 40
    arrs = sharding.random_vocabulary_arrays(10, 6, 7)
    voc = M.ORBVocabulary.from_arrays(*arrs, 10, 6)
    X = ORBextractor(1200)
    rng = np.random.default_rng(1)
    outs = X.extract_batch([synth.mono_frame(50 + i, 0, 0, 752, 480) for i in range(n_src)])
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    kfs, bows = [], []
    for j in range(n_kf):
        k, d = outs[j % n_src]
        if j >= n_src:
            flip = (rng.random((len(d), 32, 8)) < 0.04)
            d = d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)
        bow, fv = voc.transform(d, 4)
        kf = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.8).astype(np.uint8))
        db.add(kf, bow)
        kfs.append(kf); bows.append(bow)
    qk, qd = outs[3]
    flip = (rng.random((len(qd), 32, 8)) < 0.02)
    qd = qd ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(qd), 32)
    qbow, qfv = voc.transform(qd, 4)
    F = M.KeyFrameView(mvKeysUn=qk, mDescriptors=qd, mFeatVec=qfv)
    assert len(qk) >= 1200 and all(len(k.mvKeysUn) >= 1200 for k in kfs[:n_src])
    cw, sc, fw = db.query(qbow)
    for s in rng.choice(n_kf, 64, replace=False).tolist() + [3, 43]:
        so, co, fo = oracle.port_bow_score(qbow, bows[s])
        assert cw[s] == co and fw[s] == fo and sc[s] == np.float32(so), s
    nm, off, pairs = db.SearchByBoWPairs(None, F)
    assert int(nm.sum()) == len(pairs)
    dense = _pairs_to_dense(nm, off, pairs, len(qk))
    for s in range(n_kf):
        n_o, m_o = oracle.port_search_by_bow(kfs[s], F, 0.75, True)
        assert nm[s] == n_o and np.array_equal(dense[s], m_o), s
    assert nm[3] > 300 and nm.max() == nm[3::n_src].max()


@pytest.mark.parametrize("n_frame,levelsup", [(6000, 2), (8192, 3), (3000, 2)])
def test_search_by_bow_large_query_frames(oracle, n_frame, levelsup):
    """Query frames at and beyond what fits next to the per-warp scratch in one SM's shared memory: 3000 features still use the
    shared-memory frame block with fewer warps per CTA, 6000 / 8192 (the library's limit) read the block through L1 from global
    memory (bowdb_match_kernel<., false>), with buckets far wider than 32 columns (claim bitset path).  Random descriptors, keyframes
    derived from the frame by bit flips so that real matches exist; every keyframe against the restated SearchByBoW."""
    from orb_slam2_b200 import matcher as M
    from orb_slam2_b200._lib import KP_DTYPE
    rng = np.random.default_rng(n_frame + levelsup)
    pv = oracle.PortVocabulary.random(10, 4, 9)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])

    def keys(n):
        k = np.zeros(n, KP_DTYPE)
        k["x"] = rng.uniform(20, 600, n).astype(np.float32); k["y"] = rng.uniform(20, 440, n).astype(np.float32)
        k["angle"] = rng.uniform(0, 360, n).astype(np.float32); k["size"] = 31.0; k["octave"] = 0; k["class_id"] = -1
        return k
    qd = rng.integers(0, 256, (n_frame, 32), dtype=np.uint8)
    qk = keys(n_frame)
    qbow, qfv = voc.transform(qd, levelsup)
    F = M.KeyFrameView(mvKeysUn=qk, mDescriptors=qd, mFeatVec=qfv)
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    kfs = []
    for j in range(5):
        n = [1500, 900, 2400, 1, 700][j]
        src = rng.choice(n_frame, n, replace=False)
        flip = rng.random((n, 32, 8)) < [0.03, 0.06, 0.02, 0.0, 0.10][j]
        d = qd[src] ^ np.packbits(flip, axis=2, bitorder="little").reshape(n, 32)
        k = keys(n)
        k["angle"] = (qk["angle"][src] + rng.choice([0.0, 0.0, 0.0, 95.0], n)).astype(np.float32) % np.float32(360)
        bow, fv = voc.transform(d, levelsup)
        kf = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(n) < 0.7).astype(np.uint8))
        db.add(kf, bow); kfs.append(kf)
    nm, off, pairs = db.SearchByBoWPairs(None, F)
    dense = _pairs_to_dense(nm, off, pairs, n_frame)
    for s, kf in enumerate(kfs):
        n_o, m_o = oracle.port_search_by_bow(kf, F, 0.75, True)
        assert nm[s] == n_o and np.array_equal(dense[s], m_o), s
    assert nm[0] > 100 and nm[2] > 100
