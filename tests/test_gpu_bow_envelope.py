"""GPU: the place-recognition envelope (tests/bow_envelope.py) through the CUDA library, bit for bit against the port:
borb_bow_transform, borb_compute_bow and borb_frames_compute_bow on every vocabulary shape (text loader and array upload);
borb_kfdb_query and _batch on every query size; borb_search_by_bow_db, _pairs and _batch on every search case and on batches of
2 * n_SM + 1 small jobs and of mixed shared / global frame blocks with empty jobs — each database search under the three Hamming
modes and four scheduling settings (item targets 1, 8192 and 2^20, and the static schedule)."""
import functools

import numpy as np
import pytest

from orb_slam2_b200 import _lib
from orb_slam2_b200 import matcher as M
from orb_slam2_b200._lib import BorbError
from tests import bow_envelope as BE

pytestmark = pytest.mark.gpu

SCALE = (1.2 ** np.arange(8)).astype(np.float32)
CSA_MODES = [0, 1, 2]
ITEM_TARGETS = [1, 8192, 2 ** 20, -8192]          # negative: the static schedule with target 8192
DEFAULT_CSA, DEFAULT_TARGET = 2, 8192             # borb_match_host.cu:1652-1653


@pytest.fixture(scope="module")
def mt():
    return M.ORBmatcher(0.75, True)


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def knobs():
    """Every (Hamming mode, item target) setting; both knobs are restored when the generator is closed."""
    lib = _lib.load()
    try:
        for csa in CSA_MODES:
            for tgt in ITEM_TARGETS:
                _lib.check(lib.borb_debug_set_bow_csa(csa), "set_bow_csa")
                _lib.check(lib.borb_debug_set_bow_item_target(tgt), "set_bow_item_target")
                yield csa, tgt
    finally:
        lib.borb_debug_set_bow_csa(DEFAULT_CSA)
        lib.borb_debug_set_bow_item_target(DEFAULT_TARGET)


@pytest.fixture(scope="module")
def vocs(oracle, tmp_path_factory):
    d = tmp_path_factory.mktemp("bow_envelope")
    out = {}
    for name in BE.VOCABS:
        a = BE.vocabulary(name)
        path = BE.write_voc(a, str(d / f"{name}.txt"))
        out[name] = (a, oracle.PortVocabulary.load_text(path), M.ORBVocabulary.loadFromTextFile(path),
                     M.ORBVocabulary.from_arrays(a["parent"], a["is_leaf"], a["desc"], a["weight"], a["k"], a["L"]))
    return out


def _keys(n, seed=0):
    return BE._keys(np.random.default_rng(seed), n)


def resident(mt, keys, desc):
    return M.FrameView(keys, np.ascontiguousarray(desc, np.uint8), SCALE, (0.0, 0.0, 640.0, 480.0)).make_resident(mt)


def same_bow(got, want):
    (bg, fg), (bw, fw) = got, want
    assert list(bg) == list(bw)
    assert np.array_equal(np.fromiter(bg.values(), np.float64, len(bg)), np.fromiter(bw.values(), np.float64, len(bw)))
    assert np.array_equal(fg.node_id, fw.node_id) and np.array_equal(fg.start, fw.start) and np.array_equal(fg.feat_idx, fw.feat_idx)


@pytest.mark.parametrize("name", BE.VOCABS)
def test_transform_and_compute_bow_equal_port(oracle, vocs, mt, name):
    a, pv, vt, va = vocs[name]
    sets = BE.descriptors(name)
    for levelsup in BE.LEVELSUP[name]:
        frames = [resident(mt, _keys(len(d), i), d) for i, d in enumerate(sets.values())]
        batch = mt.ComputeBoWBatch(vt, frames, levelsup)
        for (sname, d), got_b in zip(sets.items(), batch):
            bow_p, fv_p, w, wt, nd = BE.port_transform(oracle, pv, d, levelsup)
            for voc in (vt, va):
                gw, gwt, gnd = voc.transform_raw(d, levelsup)
                assert np.array_equal(gw, w) and np.array_equal(gwt, wt) and np.array_equal(gnd, nd), (levelsup, sname)
            same_bow(vt.ComputeBoW(d, levelsup), (bow_p, fv_p))
            same_bow(got_b, (bow_p, fv_p))


def test_compute_bow_sizes_equal_port(oracle, vocs, mt):
    """Every ComputeBoW size up to 8192 features; past it the descent alone still equals the port, and borb_compute_bow refuses
    the frame (bow_build_kernel's keys of 8193 features would need 256 KB of shared memory)."""
    a, pv, vt, va = vocs["weights"]
    sets = [BE.compute_set(n) for n in BE.COMPUTE_SIZES] + [BE.compute_set(n, True) for n in (1, 1025, 8192)]
    frames = [resident(mt, _keys(len(d), i), d) for i, d in enumerate(sets)]
    big = BE.compute_set(10000)
    for levelsup in (0, 1, 2):
        got = mt.ComputeBoWBatch(vt, frames, levelsup)
        for d, g in zip(sets, got):
            want = BE.port_transform(oracle, pv, d, levelsup)[:2]
            same_bow(g, want)
            same_bow(vt.ComputeBoW(d, levelsup), want)
        want_raw = pv.transform_raw(big, levelsup)
        for voc in (vt, va):
            assert all(np.array_equal(g, w) for g, w in zip(voc.transform_raw(big, levelsup), want_raw)), levelsup
    with pytest.raises(BorbError) as ei:
        vt.ComputeBoW(BE.compute_set(BE.MATCH_MAX_FEATURES + 1), 0)
    assert ei.value.status == 1 and f"limit {BE.MATCH_MAX_FEATURES}" in str(ei.value), str(ei.value)


def test_child_rank_limit_is_refused_naming_the_node():
    n = (1 << BE.CHILD_RANK_BITS) + 1                        # the root with 2^23 children
    parent = np.zeros(n, np.int32)
    leaf = np.ones(n, np.uint8); leaf[0] = 0
    with pytest.raises(BorbError) as ei:
        M.ORBVocabulary.from_arrays(parent, leaf, np.zeros((n, 32), np.uint8), np.ones(n, np.float64), 10, 1)
    assert ei.value.status == 1 and "node 0:" in str(ei.value), str(ei.value)


# ---------------------------------------------------------------------------------------------------------------------------
# keyframe-database queries
def _empty_kf():
    return M.KeyFrameView(mvKeysUn=np.zeros(0, BE.KP_DTYPE), mDescriptors=np.zeros((0, 32), np.uint8),
                          mFeatVec=M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32)))


def test_query_equals_port(oracle, mt):
    kfs, queries, _ = BE.query_world()
    db = M.KeyFrameDatabase(mt)
    for b in kfs:
        db.add(_empty_kf(), b)
    for qname, q in queries.items():
        cw, sc, fw = db.query(q)
        assert len(cw) == len(kfs)
        for s, b in enumerate(kfs):
            so, co, fo = oracle.port_bow_score(q, b)
            assert cw[s] == co and fw[s] == fo and sc[s] == np.float32(so), (qname, s)
    q = queries["order_first"]
    assert db.query(q)[1][len(kfs) - 2] == np.float32(1.0)


def test_query_batch_equals_port(oracle, vocs, mt):
    """Resident frames' BowVectors on the order-sensitive vocabulary against keyframes of the same vocabulary, one launch."""
    a, pv, vt, _ = vocs["weights"]
    sets = [BE.compute_set(n) for n in (0, 1, 33, 1025, 8192)] + [BE.compute_set(8192, True), BE.descriptors("weights")["order"]]
    frames = [resident(mt, _keys(len(d), i), d) for i, d in enumerate(sets)]
    host = mt.ComputeBoWBatch(vt, frames, 1)
    db = M.KeyFrameDatabase(mt)
    kf_bows = []
    for i, d in enumerate(sets[1:] + [BE.compute_set(4097), BE.compute_set(32)]):
        bow = BE.port_transform(oracle, pv, d, 1)[0]
        db.add(_empty_kf(), bow); kf_bows.append(bow)
    got = mt.KfdbQueryBatch(db, frames)
    for j, (cw, sc, fw) in enumerate(got):
        for s, b in enumerate(kf_bows):
            so, co, fo = oracle.port_bow_score(host[j][0], b)
            assert cw[s] == co and fw[s] == fo and sc[s] == np.float32(so), (j, s)
        cw1, sc1, fw1 = db.query(host[j][0])
        assert np.array_equal(cw, cw1) and np.array_equal(sc, sc1) and np.array_equal(fw, fw1)


# ---------------------------------------------------------------------------------------------------------------------------
# database searches
@functools.lru_cache(maxsize=None)
def _port_search(name):
    from oracle import oracle_lib
    return BE.port_search(oracle_lib, BE.search_case(name))


def _db_of(mt, kfs):
    db = M.KeyFrameDatabase(mt)
    for k in kfs:
        db.add(k, {0: 1.0})
    return db


@pytest.mark.parametrize("name", BE.SEARCH_NAMES)
def test_database_search_equals_port_in_every_mode(oracle, mt, name):
    c = BE.search_case(name)
    port = _port_search(name)
    want_nm = np.array([n for n, _ in port], np.int32)
    want = np.stack([m for _, m in port])
    n_f = len(c["F"].mvKeysUn)
    db = _db_of(mt, c["kfs"])
    slots = np.arange(len(c["kfs"]), dtype=np.int32)
    for csa, tgt in knobs():
        nm, dn = db.SearchByBoW(slots, c["F"])
        assert np.array_equal(nm, want_nm) and np.array_equal(dn, want), (csa, tgt)
        nm, off, pairs = db.SearchByBoWPairs(None, c["F"])
        assert np.array_equal(nm, want_nm) and np.array_equal(BE.dense_from_pairs(nm, off, pairs, n_f), want), (csa, tgt)
    assert want_nm.sum() > 0


def test_pairs_cap_equal_to_the_total_and_one_below(mt):
    c = BE.search_case("edges")
    port = _port_search("edges")
    total = sum(n for n, _ in port)
    db = _db_of(mt, c["kfs"])
    nm, off, pairs = db.SearchByBoWPairs(None, c["F"], pairs_cap=total)
    assert len(pairs) == total and np.array_equal(BE.dense_from_pairs(nm, off, pairs, len(c["F"].mvKeysUn)), np.stack([m for _, m in port]))
    with pytest.raises(BorbError) as ei:
        db.SearchByBoWPairs(None, c["F"], pairs_cap=total - 1)
    assert ei.value.status == 5


@pytest.fixture(scope="module")
def batch_world(oracle, vocs, mt, n_sm):
    """12 small frames near the 40-wide vocabulary's leaves (blocks in shared memory), one 6000-feature frame (global memory), a
    database of keyframes that are noisy, permuted copies of them, and the port's SearchByBoW of every (frame, keyframe) pair."""
    a, pv, vt, _ = vocs["k40"]
    rng = np.random.default_rng(77)
    small = [BE.near_leaves(a, rng, int(n), flips=(0, 1, 2, 4)) for n in rng.integers(40, 200, 12)]
    big = BE.near_leaves(a, rng, 6000, flips=(0, 1, 3))
    descs = small + [big]
    keys = [_keys(len(d), 100 + i) for i, d in enumerate(descs)]
    frames = [resident(mt, k, d) for k, d in zip(keys, descs)]
    host = mt.ComputeBoWBatch(vt, frames, 1)
    Fh = [M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=h[1]) for k, d, h in zip(keys, descs, host)]
    for d, h in zip(descs, host):
        same_bow(h, BE.port_transform(oracle, pv, d, 1)[:2])
    db = M.KeyFrameDatabase(mt)
    kfs = []
    for i, d in enumerate(descs):
        p = rng.permutation(len(d))
        flip = rng.random((len(d), 256)) < rng.choice([0.0, 0.03, 0.1], len(d))[:, None]
        kd = np.packbits(np.unpackbits(d[p], axis=1) ^ flip, axis=1)
        kk = keys[i][p].copy()
        kk["angle"] = (kk["angle"] + rng.choice([0.0, 0.0, 60.0], len(d))).astype(np.float32) % np.float32(360)
        bow, fv = BE.port_transform(oracle, pv, kd, 1)[:2]
        kv = M.KeyFrameView(mvKeysUn=kk, mDescriptors=kd, mFeatVec=fv, has_mp=(rng.random(len(d)) < 0.8).astype(np.uint8))
        db.add(kv, bow); kfs.append(kv)
    port = {}
    for f in range(len(descs)):
        for s in range(len(kfs)):
            port[f, s] = oracle.port_search_by_bow(kfs[s], Fh[f], 0.75, True)
    assert BE.frame_fits_smem(len(host[0][1].node_id), len(host[0][1].feat_idx))
    assert not BE.frame_fits_smem(len(host[12][1].node_id), len(host[12][1].feat_idx))
    return dict(frames=frames, Fh=Fh, db=db, port=port, n_sm=n_sm)


def _check_jobs(W, jobs, got, tag):
    for j, ((f, sl), (nm, off, pairs)) in enumerate(zip(jobs, got)):
        assert len(nm) == len(sl), (tag, j)
        dn = BE.dense_from_pairs(nm, off, pairs, len(W["Fh"][f].mvKeysUn))
        for i, s in enumerate(sl):
            n_p, m_p = W["port"][f, s]
            assert nm[i] == n_p and np.array_equal(dn[i], m_p), (tag, j, s)


def test_table_batch_of_2_nsm_plus_1_small_jobs(mt, batch_world):
    """More jobs than twice the CTAs: some CTA loads three or more shared-memory frame blocks in turn."""
    W = batch_world
    n = 2 * W["n_sm"] + 1
    jobs = [(j % 12, [j % 12, (j + 1) % 12, (j + 5) % 12][: 1 + j % 3]) for j in range(n)]
    for csa, tgt in knobs():
        got = mt.SearchByBoWDbBatch(W["db"], [sl for _, sl in jobs], [W["frames"][f] for f, _ in jobs])
        _check_jobs(W, jobs, got, (csa, tgt))


def test_mixed_batch_with_empty_jobs(mt, batch_world):
    """Shared-memory and global frame blocks in one launch, with n_kf == 0 jobs in the middle and at the end."""
    W = batch_world
    jobs = [(0, [0, 3, 12]), (12, [12, 0, 1, 12]), (5, []), (1, [1]), (12, [4, 12]), (7, list(range(13))), (2, [])]
    for csa, tgt in knobs():
        got = mt.SearchByBoWDbBatch(W["db"], [sl for _, sl in jobs], [W["frames"][f] for f, _ in jobs])
        _check_jobs(W, jobs, got, (csa, tgt))
        assert len(got[2][0]) == 0 and len(got[6][0]) == 0
    assert W["port"][12, 12][0] > 100
