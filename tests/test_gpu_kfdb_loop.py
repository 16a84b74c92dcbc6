"""GPU parity of loop closure's first search, SearchByBoW(KeyFrame*, KeyFrame*) (src/ORBmatcher.cc:522-655), run on the resident
keyframe database: borb_search_by_bow_kf_db_pairs / _batch must give, for every (query slot, candidate slot), the count and the
match12 of borb_search_by_bow_kf on host views, of the port and of the verbatim ORBmatcher.cc — across EuRoC-shaped keyframes,
the real vocabulary's FeatureVectors, wide buckets, ties, the strict TH_LOW gate, empty MapPoint masks, 8192-feature keyframes,
whole databases and many streams per launch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from orb_slam2_b200._lib import BorbError

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def flip(rng, d, p):
    f = rng.random((len(d), 32, 8)) < p
    return d ^ np.packbits(f, axis=2, bitorder="little").reshape(len(d), 32)


def match12(nm, off, pairs, k, n1):
    out = np.full(n1, -1, np.int32)
    pr = pairs[off[k]:off[k] + nm[k]]
    out[(pr & 0xFFFF).astype(np.int64)] = (pr >> 16).astype(np.int32)
    return out


def euroc():
    g = np.load(os.path.join(ROOT, "tests", "golden", "extract_euroc_1200.npz"))
    return g["keypoints"], g["descriptors"]


def noisy_views(M, rng, keys, desc, fvs, n, p_bits=0.06, p_mp=0.7):
    """n keyframes of one scene: bit noise on the descriptors, jittered angles, a random MapPoint mask; fvs(desc) -> FeatureVector."""
    out = []
    for _ in range(n):
        d = flip(rng, desc, p_bits)
        k = keys.copy()
        k["angle"] = np.mod(k["angle"] + rng.normal(0, 8, len(k)), 360).astype(np.float32)
        out.append(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fvs(d), has_mp=(rng.random(len(k)) < p_mp).astype(np.uint8)))
    return out


def make_db(M, mt, views):
    db = M.KeyFrameDatabase(mt)
    for v in views:
        db.add(v, {})
    return db


def check_against_refs(M, oracle, mt, views, q, slots, got, nnratio, ori):
    """got = (nm, off, pairs) of the database search of views[q] against views[slots]."""
    nm, off, pairs = got
    assert len(nm) == len(slots) and int(nm.sum()) == len(pairs)
    n1 = len(views[q].mvKeysUn)
    for k, s in enumerate(slots):
        m12 = match12(nm, off, pairs, k, n1)
        n_h, m_h = mt.SearchByBoW_KF(views[q], views[s])
        n_p, m_p = oracle.port_search_by_bow_kf(views[q], views[s], nnratio, ori)
        assert int(nm[k]) == n_h == n_p, (q, s, int(nm[k]), n_h, n_p)
        assert np.array_equal(m12, m_h) and np.array_equal(m12, m_p), (q, s)
        if oracle.have_ref():
            n_r, m_r = oracle.ref_search_by_bow_kf(views[q], views[s], nnratio, ori)
            assert n_r == n_p and np.array_equal(m_r, m_p), (q, s)


@pytest.fixture(scope="module")
def euroc_world(M, oracle):
    """EuRoC-shaped 752x480 @1200 keyframes of one scene, FeatureVectors of a random k=10, L=6 vocabulary at levelsup 4."""
    pv = oracle.PortVocabulary.random(10, 6, 11)
    keys, desc = euroc()
    rng = np.random.default_rng(21)
    return noisy_views(M, rng, keys, desc, lambda d: M.bow_and_featvec(*pv.transform_raw(d, 4))[1], 8)


@pytest.mark.parametrize("ori", [0, 1])
@pytest.mark.parametrize("nnratio", [0.6, 0.75, 1.0])
def test_euroc_parity(M, oracle, euroc_world, ori, nnratio):
    mt = M.ORBmatcher(nnratio, bool(ori))
    views = euroc_world
    db = make_db(M, mt, views)
    slots = [1, 2, 3, 0, 7, 2, 5]                        # repeats and the query itself among its candidates
    got = db.SearchByBoWKFPairs(0, slots)
    assert got[0].sum() > 100                            # the fixture matches
    check_against_refs(M, oracle, mt, views, 0, slots, got, nnratio, ori)
    got = db.SearchByBoWKFPairs(6, None)                 # every slot
    check_against_refs(M, oracle, mt, views, 6, list(range(len(views))), got, nnratio, ori)


@pytest.mark.parametrize("ori", [0, 1])
def test_real_vocabulary_featvecs(M, oracle, ori):
    """The FeatureVectors the reference's own ORBvoc.txt gives the three golden descriptor sets (tests/golden/voc_real.npz)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "voc_real.npz"))
    rng = np.random.default_rng(4)
    mt = M.ORBmatcher(0.75, bool(ori))
    for name in ("extract_euroc_1200", "extract_kitti_2000", "extract_tum_1000"):
        e = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
        fv = M.FeatureVector(g[name + "_fv_node"], g[name + "_fv_start"], g[name + "_fv_idx"])
        views = noisy_views(M, rng, e["keypoints"], e["descriptors"], lambda d: fv, 5)
        db = make_db(M, mt, views)
        got = db.SearchByBoWKFPairs(2, [0, 1, 2, 3, 4])
        assert got[0].sum() > 100, name
        check_against_refs(M, oracle, mt, views, 2, [0, 1, 2, 3, 4], got, 0.75, ori)


def synth_view(M, rng, n, nodes, base=None, p_bits=0.0, angles=None, has_mp=None):
    from orb_slam2_b200._lib import KP_DTYPE
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(10, 740, n); k["y"] = rng.uniform(10, 470, n); k["size"] = 31.0; k["class_id"] = -1
    k["angle"] = rng.uniform(0, 360, n) if angles is None else angles
    d = rng.integers(0, 256, (n, 32), dtype=np.uint8) if base is None else flip(rng, base, p_bits)
    fv = M.FeatureVector.from_nodes(np.asarray(nodes, np.int64))
    hm = np.ones(n, np.uint8) if has_mp is None else np.asarray(has_mp, np.uint8)
    return M.KeyFrameView(mvKeysUn=k, mDescriptors=np.ascontiguousarray(d), mFeatVec=fv, has_mp=hm)


@pytest.mark.parametrize("ori", [0, 1])
def test_wide_buckets_and_ties(M, oracle, ori):
    """Buckets of 20, 40, 70 and 300 features on both sides; candidates with duplicated descriptors (first minimum wins, best equal
    to second best)."""
    rng = np.random.default_rng(8)
    widths = [20, 40, 70, 300]
    nodes = np.repeat(np.arange(len(widths)) * 7 + 3, widths)
    n = len(nodes)
    base = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    views = [synth_view(M, rng, n, nodes, base, 0.05, has_mp=rng.random(n) < 0.8) for _ in range(4)]
    dup = views[3].mDescriptors.copy()
    dup[1::2] = dup[0::2][:len(dup[1::2])]                 # pairs of identical rows: ties everywhere
    views[3] = M.KeyFrameView(mvKeysUn=views[3].mvKeysUn, mDescriptors=dup, mFeatVec=views[3].mFeatVec, has_mp=views[3].has_mp)
    views.append(synth_view(M, rng, n, nodes, dup, 0.0, has_mp=np.ones(n)))   # exact copies: best == second best for many rows
    mt = M.ORBmatcher(0.75, bool(ori))
    db = make_db(M, mt, views)
    for q in (0, 3):
        slots = [0, 1, 2, 3, 4]
        check_against_refs(M, oracle, mt, views, q, slots, db.SearchByBoWKFPairs(q, slots), 0.75, ori)
    mt1 = M.ORBmatcher(1.0, bool(ori))
    db1 = make_db(M, mt1, views)
    check_against_refs(M, oracle, mt1, views, 0, [1, 4], db1.SearchByBoWKFPairs(0, [1, 4]), 1.0, ori)


def test_strict_th_low_and_bin_sign(M, oracle):
    """A best distance of 49 matches and one of exactly 50 does not (the relocalisation overload accepts 50); and rotation bins whose
    sign decides the rotation cull."""
    rng = np.random.default_rng(2)
    q = rng.integers(0, 256, (2, 32), dtype=np.uint8)
    c = q.copy()
    bits = np.unpackbits(c, axis=1, bitorder="little")
    bits[0, :49] ^= 1                                      # distance 49
    bits[1, :50] ^= 1                                      # distance 50
    c = np.packbits(bits, axis=1, bitorder="little")
    angles_q = np.array([10.0, 20.0], np.float32)
    vq = synth_view(M, rng, 2, [5, 9], q, angles=angles_q)
    vc = synth_view(M, rng, 2, [5, 9], c, angles=angles_q)
    vq = M.KeyFrameView(mvKeysUn=vq.mvKeysUn, mDescriptors=q, mFeatVec=vq.mFeatVec, has_mp=vq.has_mp)
    vc = M.KeyFrameView(mvKeysUn=vc.mvKeysUn, mDescriptors=c, mFeatVec=vc.mFeatVec, has_mp=vc.has_mp)
    mt = M.ORBmatcher(1.0, False)
    db = make_db(M, mt, [vq, vc])
    nm, off, pairs = db.SearchByBoWKFPairs(0, [1])
    assert int(nm[0]) == 1 and np.array_equal(match12(nm, off, pairs, 0, 2), [0, -1])
    check_against_refs(M, oracle, mt, [vq, vc], 0, [1], (nm, off, pairs), 1.0, 0)
    # the relocalisation overload (:228, bestDist1 <= TH_LOW) on the same data matches both
    nm_r, _, _ = db.SearchByBoWPairs([1], vq)
    assert int(nm_r[0]) == 2
    # bin sign: rotations +5 and -5 degrees fall into bins 0 and 12, and ComputeThreeMaxima keeps the first of two equal counts;
    # with 12 rows at +60 and 11 at +120 the cull keeps the +5 rows and drops the -5 rows (candidate - query would do the opposite)
    groups = [(5.0, 10), (-5.0, 10), (60.0, 12), (120.0, 11)]
    rot = np.concatenate([np.full(c, r, np.float32) for r, c in groups])
    n = len(rot)
    nodes = np.arange(n) % 6
    base = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    aq = rng.uniform(0, 360, n).astype(np.float32)
    v1 = synth_view(M, rng, n, nodes, base, 0.0, angles=aq)
    v2 = synth_view(M, rng, n, nodes, base, 0.02, angles=np.mod(aq - rot, 360).astype(np.float32))
    mt1 = M.ORBmatcher(0.75, True)
    db1 = make_db(M, mt1, [v1, v2])
    got = db1.SearchByBoWKFPairs(0, [1])
    m12 = match12(*got, 0, n)
    assert int(got[0][0]) == n - 10 and (m12[:10] >= 0).all() and (m12[10:20] < 0).all()
    check_against_refs(M, oracle, mt1, [v1, v2], 0, [1], got, 0.75, 1)
    got = db1.SearchByBoWKFPairs(1, [0])                   # the other direction: the -5 rows survive
    m21 = match12(*got, 0, n)
    assert (m21[:10] < 0).all() and (m21[10:20] >= 0).all()
    check_against_refs(M, oracle, mt1, [v1, v2], 1, [0], got, 0.75, 1)


def test_masks_empty_and_set_has_mp(M, oracle, euroc_world):
    views = list(euroc_world[:4])
    n = len(views[0].mvKeysUn)
    mt = M.ORBmatcher(0.75, True)
    db = make_db(M, mt, views)
    zero = np.zeros(n, np.uint8)
    db.set_has_mp(0, zero)                                  # a query without MapPoints: nothing can match
    nm, _, pairs = db.SearchByBoWKFPairs(0, [1, 2, 3])
    assert nm.sum() == 0 and len(pairs) == 0
    db.set_has_mp(0, views[0].has_mp)
    db.set_has_mp(2, zero)                                  # a candidate without MapPoints
    nm, _, _ = db.SearchByBoWKFPairs(0, [1, 2, 3])
    assert nm[0] > 0 and nm[1] == 0 and nm[2] > 0
    new = (np.random.default_rng(1).random(n) < 0.4).astype(np.uint8)
    db.set_has_mp(1, new)                                   # a changed mask is honoured
    v1 = M.KeyFrameView(mvKeysUn=views[1].mvKeysUn, mDescriptors=views[1].mDescriptors, mFeatVec=views[1].mFeatVec, has_mp=new)
    views2 = [views[0], v1, M.KeyFrameView(mvKeysUn=views[2].mvKeysUn, mDescriptors=views[2].mDescriptors, mFeatVec=views[2].mFeatVec,
                                           has_mp=zero), views[3]]
    check_against_refs(M, oracle, mt, views2, 0, [1, 2, 3], db.SearchByBoWKFPairs(0, [1, 2, 3]), 0.75, 1)
    check_against_refs(M, oracle, mt, views2, 1, [0, 3], db.SearchByBoWKFPairs(1, [0, 3]), 0.75, 1)


def test_8192_feature_keyframes(M, oracle):
    """The largest keyframes: the query block no longer fits in shared memory and is read from global memory."""
    rng = np.random.default_rng(9)
    n = 8192
    nodes = rng.integers(0, 90, n)
    base = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    views = [synth_view(M, rng, n, nodes, base, 0.08, has_mp=rng.random(n) < 0.7) for _ in range(3)]
    mt = M.ORBmatcher(0.75, True)
    db = make_db(M, mt, views)
    got = db.SearchByBoWKFPairs(0, [1, 2, 0])
    assert got[0][0] > 1000
    check_against_refs(M, oracle, mt, views, 0, [1, 2, 0], got, 0.75, 1)


def test_all_2000_slots(M, oracle):
    """slots = NULL over a 2000-keyframe database (erased slots give zeros), checked against the single host-view search."""
    rng = np.random.default_rng(12)
    pv = oracle.PortVocabulary.random(10, 6, 3)
    keys, desc = euroc()
    keys, desc = keys[:300], desc[:300]
    fv0 = M.bow_and_featvec(*pv.transform_raw(desc, 4))[1]
    views = noisy_views(M, rng, keys, desc, lambda d: fv0, 2000, p_bits=0.08)
    mt = M.ORBmatcher(0.75, True)
    db = make_db(M, mt, views)
    db.erase(17)
    nm, off, pairs = db.SearchByBoWKFPairs(5, None)
    assert len(nm) == 2000 and nm[17] == 0 and nm.sum() > 2000 * 20
    for k in range(2000):
        if k == 17:
            continue
        n_h, m_h = mt.SearchByBoW_KF(views[5], views[k])
        assert int(nm[k]) == n_h and np.array_equal(match12(nm, off, pairs, k, 300), m_h), k
    for k in (0, 5, 999, 1999):
        n_p, m_p = oracle.port_search_by_bow_kf(views[5], views[k], 0.75, 1)
        assert int(nm[k]) == n_p and np.array_equal(match12(nm, off, pairs, k, 300), m_p)


def test_batch_equals_single_calls(M, oracle):
    """32 streams with their own 300-keyframe databases and 15 candidates each, plus four jobs on one shared database: every job
    equals its single call; the launch count does not depend on the number of jobs; overflow names the first job that overflowed."""
    rng = np.random.default_rng(30)
    pv = oracle.PortVocabulary.random(10, 6, 5)
    keys, desc = euroc()
    keys, desc = keys[:200], desc[:200]
    fv0 = M.bow_and_featvec(*pv.transform_raw(desc, 4))[1]
    mt = M.ORBmatcher(0.75, True)
    dbs, qs, sls = [], [], []
    for s in range(32):
        views = noisy_views(M, rng, keys, desc, lambda d: fv0, 300, p_bits=0.07)
        dbs.append(make_db(M, mt, views))
        qs.append(int(rng.integers(0, 300)))
        sls.append(rng.integers(0, 300, 15).astype(np.int32))
    shared = dbs[0]
    for _ in range(4):
        dbs.append(shared); qs.append(int(rng.integers(0, 300))); sls.append(rng.integers(0, 300, 15).astype(np.int32))
    l0 = launches(mt)
    got = mt.SearchByBoWKFDbBatch(dbs, qs, sls)
    l1 = launches(mt)
    one = mt.SearchByBoWKFDbBatch(dbs[:1], qs[:1], sls[:1])
    l2 = launches(mt)
    assert l1 - l0 == l2 - l1 == 3
    total = 0
    for j, (db, q, sl) in enumerate(zip(dbs, qs, sls)):
        nm, off, pairs = got[j]
        nm2, off2, pairs2 = db.SearchByBoWKFPairs(q, sl)
        assert np.array_equal(nm, nm2), j
        for k in range(len(sl)):
            assert np.array_equal(pairs[off[k]:off[k] + nm[k]], pairs2[off2[k]:off2[k] + nm2[k]]), (j, k)
        total += int(nm.sum())
    assert np.array_equal(one[0][0], got[0][0]) and total > 32 * 15 * 20
    # overflow: jobs 1 and 2 have too little room; the error names job 1, every count stays valid
    caps = [None, 3, 2] + [None] * 3
    with pytest.raises(BorbError, match="job 1:"):
        mt.SearchByBoWKFDbBatch(dbs[:6], qs[:6], sls[:6], pairs_cap=caps)


def test_refusals_name_the_job_and_launch_nothing(M, oracle, euroc_world):
    from orb_slam2_b200.matcher import _BowKfDbJobC
    mt = M.ORBmatcher(0.75, True)
    views = list(euroc_world[:3])
    db = make_db(M, mt, views)
    db.add(M.KeyFrameView(mvKeysUn=views[0].mvKeysUn[:0], mDescriptors=views[0].mDescriptors[:0],
                          mFeatVec=M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32))), {})   # slot 3: no features
    db.erase(1)
    good = (db, 0, [2], None)
    cases = [
        ((None, 0, [2], None), "null database"),
        ((db, 1, [2], None), "query slot 1"),                   # erased
        ((db, 9, [2], None), "query slot 9"),                   # out of range
        ((db, -1, [2], None), "query slot -1"),
        ((db, 3, [2], None), "query slot 3"),                   # added without features
        ((db, 0, [1], None), "slot 1 is not a live keyframe"),  # erased candidate
        ((db, 0, [7], None), "slot 7 is not a live keyframe"),
    ]
    for bad, text in cases:
        l0 = launches(mt)
        with pytest.raises(BorbError, match="job 1: .*" + text):
            mt.SearchByBoWKFDbBatch([good[0], bad[0]], [good[1], bad[1]], [good[2], bad[2]], pairs_cap=[100, 100])
        assert launches(mt) == l0, text
    # slots == NULL with a wrong n_kf (only the C ABI can say so)
    jobs = (_BowKfDbJobC * 1)()
    nm = np.zeros(8, np.int32); off = np.zeros(8, np.int32); pairs = np.zeros(8, np.uint32); tot = np.zeros(1, np.int32)
    J = jobs[0]
    J.db, J.query_slot, J.slots, J.n_kf = db._h.value, 0, None, 2
    J.n_matches, J.pair_offset, J.pairs, J.pairs_cap, J.n_pairs_total = nm.ctypes.data, off.ctypes.data, pairs.ctypes.data, 8, tot.ctypes.data
    st = mt._lib.borb_search_by_bow_kf_db_batch(mt._h, jobs, 1, C.c_float(0.75), 1)
    assert st != 0 and mt._lib.borb_last_error().decode().startswith("job 0: slots == NULL")


def test_overflow_keeps_counts_and_offsets(M, euroc_world):
    """BORB_ERR_CAPACITY after the run: every job's counts and offsets equal those of a run with room for every pair, and the pairs
    that fit are the uncapped run's."""
    from orb_slam2_b200.matcher import _BowKfDbJobC
    mt = M.ORBmatcher(0.75, True)
    db = make_db(M, mt, list(euroc_world))
    qs, sls = [0, 3, 5], [np.array([1, 2, 3], np.int32), np.array([0, 4], np.int32), np.array([6, 7, 1], np.int32)]
    full = mt.SearchByBoWKFDbBatch(db, qs, sls)
    caps = [100000, 7, 5]
    jobs = (_BowKfDbJobC * 3)()
    keep = []
    for j in range(3):
        nm = np.full(len(sls[j]), -9, np.int32); off = np.full(len(sls[j]), -9, np.int32)
        pairs = np.zeros(caps[j], np.uint32); tot = np.zeros(1, np.int32)
        J = jobs[j]
        J.db, J.query_slot, J.slots, J.n_kf = db._h.value, qs[j], sls[j].ctypes.data, len(sls[j])
        J.n_matches, J.pair_offset, J.pairs, J.pairs_cap, J.n_pairs_total = nm.ctypes.data, off.ctypes.data, pairs.ctypes.data, caps[j], tot.ctypes.data
        keep.append((nm, off, pairs, tot))
    st = mt._lib.borb_search_by_bow_kf_db_batch(mt._h, jobs, 3, C.c_float(0.75), 1)
    assert st != 0 and mt._lib.borb_last_error().decode().startswith("job 1:")
    for j, (nm, off, pairs, tot) in enumerate(keep):
        nm2, off2, pairs2 = full[j]
        assert np.array_equal(nm, nm2) and int(tot[0]) == int(nm2.sum()) > caps[1]
        nz = np.nonzero(nm)[0]
        order = nz[np.argsort(off[nz])]
        assert np.array_equal(off[order], np.concatenate([[0], np.cumsum(nm[order])[:-1]]))        # the blocks tile the pair list
        for k in range(len(nm)):
            if off[k] + nm[k] <= caps[j]:
                assert np.array_equal(pairs[off[k]:off[k] + nm[k]], pairs2[off2[k]:off2[k] + nm2[k]]), (j, k)


@pytest.fixture(scope="module")
def loop_adapter(tmp_path_factory):
    """tests/loop_adapter_wrap.cpp: the ComputeSim3 adapter on stand-in KeyFrame / MapPoint types, linked against libborb.so."""
    out = str(tmp_path_factory.mktemp("loop_adapter") / "libloopadapt.so")
    lib_dir = os.path.join(ROOT, "orb_slam2_b200")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "oracle", "cvmini"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "loop_adapter_wrap.cpp"), "-o", out, "-L", lib_dir,
                           "-l:libborb.so", "-Wl,-rpath," + lib_dir])
    lib = C.CDLL(out)
    lib.loop_adapter_run.restype = C.c_int
    lib.loop_adapter_run.argtypes = [C.c_int, C.c_void_p] + [C.c_void_p] * 2 + [C.c_void_p] + [C.c_void_p] * 3 + [C.c_void_p] * 2 + \
        [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def run_adapter(lib, views, add_state, now_state, query, cands, erase, nnratio, ori):
    n = len(views)
    keep = []

    def ptrs(arrs, dtype):
        a = [np.ascontiguousarray(x, dtype) for x in arrs]
        keep.append(a)
        return (C.c_void_p * n)(*[x.ctypes.data for x in a])
    from orb_slam2_b200._lib import KP_DTYPE
    nf = np.array([len(v.mvKeysUn) for v in views], np.int32)
    nn = np.array([len(v.mFeatVec.node_id) for v in views], np.int32)
    cand = np.ascontiguousarray(cands, np.int32)
    counts = np.zeros(len(cands), np.int32)
    match = np.full((len(cands), nf[query]), -7, np.int32)
    err = C.create_string_buffer(512)
    rc = lib.loop_adapter_run(n, nf.ctypes.data, ptrs([v.mvKeysUn for v in views], KP_DTYPE), ptrs([v.mDescriptors for v in views], np.uint8),
                              nn.ctypes.data, ptrs([v.mFeatVec.node_id for v in views], np.uint32), ptrs([v.mFeatVec.start for v in views], np.int32),
                              ptrs([v.mFeatVec.feat_idx for v in views], np.uint32), ptrs(add_state, np.uint8), ptrs(now_state, np.uint8),
                              int(query), len(cand), cand.ctypes.data, int(erase), float(nnratio), int(ori), counts.ctypes.data, match.ctypes.data,
                              err, 512)
    assert rc == 0, err.value.decode()
    return counts, match


@pytest.mark.parametrize("ori", [0, 1])
def test_loop_adapter_matches_verbatim_search(M, oracle, euroc_world, loop_adapter, ori):
    """kfdb_search_loop_candidates as ComputeSim3 uses it: the masks the database got at add() are stale (MapPoints culled, added and
    set bad since), the query is among its candidates, a candidate repeats and one has been erased from the database.  Each
    candidate's count and vpMatches12 equal the verbatim SearchByBoW(KeyFrame*, KeyFrame*) on the MapPoints as they are at the
    call (0 matches for the erased candidate)."""
    rng = np.random.default_rng(40 + ori)
    views = list(euroc_world[:6])
    add_state = [rng.choice(3, len(v.mvKeysUn), p=[0.3, 0.6, 0.1]).astype(np.uint8) for v in views]
    now_state = []
    for a in add_state:
        b = a.copy()
        flip_ = rng.random(len(b)) < 0.25
        b[flip_] = rng.choice(3, int(flip_.sum()), p=[0.3, 0.6, 0.1])
        now_state.append(b)
    cands = [1, 2, 0, 4, 2, 5, 3]
    counts, match = run_adapter(loop_adapter, views, add_state, now_state, 0, cands, 5, 0.75, ori)
    now = [M.KeyFrameView(mvKeysUn=v.mvKeysUn, mDescriptors=v.mDescriptors, mFeatVec=v.mFeatVec, has_mp=(s == 1).astype(np.uint8))
           for v, s in zip(views, now_state)]
    for c, s in enumerate(cands):
        if s == 5:
            assert counts[c] == 0 and (match[c] == -1).all()
            continue
        if oracle.have_ref():
            n_r, m_r = oracle.ref_search_by_bow_kf(now[0], now[s], 0.75, ori)
        else:
            n_r, m_r = oracle.port_search_by_bow_kf(now[0], now[s], 0.75, ori)
        assert counts[c] == n_r and np.array_equal(match[c], m_r), (c, s)
    assert counts.sum() > 100
