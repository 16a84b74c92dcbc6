"""CPU: the place-recognition envelope (tests/bow_envelope.py) — vocabulary shapes, ComputeBoW sizes, keyframe-database queries
and database SearchByBoW jobs — through the port and the verbatim reference: DBoW2's loadFromTextFile / transform / score,
KeyFrameDatabase.cc's candidate detection and ORBmatcher.cc's SearchByBoW, on every case where the reference is defined.  The
cases together reach every coverage class."""
import numpy as np
import pytest

from orb_slam2_b200 import matcher as M
from tests import bow_envelope as BE


@pytest.fixture(scope="module")
def O(oracle):
    if not oracle.have_dbowref():
        pytest.skip("oracle/_ref/libdbowref.so not built (reference tree absent)")
    return oracle


@pytest.fixture(scope="module")
def vocs(O, tmp_path_factory):
    d = tmp_path_factory.mktemp("bow_envelope")
    out = {}
    for name in BE.VOCABS:
        a = BE.vocabulary(name)
        path = BE.write_voc(a, str(d / f"{name}.txt"))
        out[name] = (a, O.PortVocabulary.load_text(path), O.RefVocabulary(path))
    return out


_hits = {}


@pytest.mark.parametrize("name", BE.VOCABS)
def test_loaders_agree_and_leaf_flags_are_child_lists(vocs, name):
    a, pv, rv = vocs[name]
    assert not BE.voc_text(a).endswith("\n")
    pe, re_ = pv.export(), rv.export()
    leaf_by_children = (BE.child_counts(a) == 0).astype(np.uint8)
    leaf_by_children[0] = 0
    for e in (pe, re_):
        assert np.array_equal(e["is_leaf"], leaf_by_children)
        assert np.array_equal(e["desc"], a["desc"]) and np.array_equal(e["weight"], a["weight"])
        assert np.array_equal(e["parent"][1:], a["parent"][1:])
    assert np.array_equal(a["is_leaf"], leaf_by_children)
    assert rv.words == int(leaf_by_children.sum())


@pytest.mark.parametrize("name", BE.VOCABS)
def test_transform_equals_reference_dbow2(O, vocs, name):
    a, pv, rv = vocs[name]
    hits = _hits.setdefault("voc", set())
    compared = 0
    for levelsup in BE.LEVELSUP[name]:
        for sname, d in BE.descriptors(name).items():
            bow_p, fv_p, w, wt, nd = BE.port_transform(O, pv, d, levelsup)
            hits |= BE.descent_coverage(a, levelsup, w) | BE.bow_coverage(a, w, wt, len(d))
            bw, bv, (fn, fs, fi) = O.port_compute_bow(pv, d, levelsup)
            assert list(bow_p) == bw.tolist() and np.array_equal(np.fromiter(bow_p.values(), np.float64, len(bow_p)), bv)
            assert np.array_equal(fv_p.node_id, fn) and np.array_equal(fv_p.start, fs) and np.array_equal(fv_p.feat_idx, fi)
            if not BE.reference_defined(a, levelsup, w):
                continue                                     # DBoW2 reads an uninitialised NodeId there: port and library only
            bow_r, node_r, start_r, idx_r = rv.transform(d, levelsup)
            assert list(bow_r) == list(bow_p), (levelsup, sname)
            assert np.array_equal(np.fromiter(bow_r.values(), np.float64, len(bow_r)), np.fromiter(bow_p.values(), np.float64, len(bow_p)))
            assert np.array_equal(node_r, fv_p.node_id) and np.array_equal(start_r, fv_p.start) and np.array_equal(idx_r, fv_p.feat_idx)
            compared += 1
    assert compared > 0


@pytest.mark.parametrize("n", BE.COMPUTE_SIZES)
@pytest.mark.parametrize("one_word", [False, True])
def test_compute_bow_sizes_equal_reference(O, vocs, n, one_word):
    if one_word and n not in (1, 1025, 8192):
        pytest.skip("one-word runs at three sizes")
    a, pv, rv = vocs["weights"]
    d = BE.compute_set(n, one_word)
    bow_p, fv_p, w, wt, _ = BE.port_transform(O, pv, d, 1)
    _hits.setdefault("voc", set()).update(BE.bow_coverage(a, w, wt, n))
    bow_r, node_r, start_r, idx_r = rv.transform(d, 1)
    assert list(bow_r) == list(bow_p)
    assert np.array_equal(np.fromiter(bow_r.values(), np.float64, len(bow_r)), np.fromiter(bow_p.values(), np.float64, len(bow_p)))
    assert np.array_equal(node_r, fv_p.node_id) and np.array_equal(start_r, fv_p.start) and np.array_equal(idx_r, fv_p.feat_idx)


def test_scores_and_candidates_equal_reference(O, vocs):
    _, _, rv = vocs["flat70000"]                             # the inverted file of the verbatim database spans the query words
    kfs, queries, neigh = BE.query_world()
    n_kf = len(kfs)
    covis = lambda s: [int(x) for x in neigh[s] if x >= 0]
    seq = list(range(n_kf))
    hits = _hits.setdefault("query", set())
    total = 0
    for qname, q in queries.items():
        hits |= BE.query_coverage(kfs, qname, q)
        per = [O.port_bow_score(q, b) for b in kfs]
        for b, p in zip(kfs, per):
            assert rv.score(q, b) == p[0]                    # identical doubles
        sc = np.array([np.float32(p[0]) for p in per], np.float32)
        cw = np.array([p[1] for p in per], np.int32)
        fw = np.array([p[2] for p in per], np.uint32)
        ref = rv.detect_candidates(False, kfs, q, None, neigh)
        assert O.port_detect_reloc_candidates(kfs, BE.FLAT_WORDS, q, neigh).tolist() == ref
        assert M.relocalization_candidates(cw, sc, fw, seq, covis) == ref
        for min_score, conn in [(0.0, []), (0.01, [3, 24])]:
            connected = np.zeros(n_kf, np.uint8); connected[conn] = 1
            ref = rv.detect_candidates(True, kfs, q, connected, neigh, min_score)
            assert O.port_detect_loop_candidates(kfs, BE.FLAT_WORDS, q, connected, neigh, min_score).tolist() == ref
            assert M.loop_candidates(cw, sc, fw, seq, set(conn), covis, min_score) == ref
            total += len(ref)
    assert total > 5
    # the order-sensitive pair: the sequential sum keeps the float score at 1.0f, a pairwise one would not
    q = queries["order_first"]
    s = np.float32(O.port_bow_score(q, kfs[-2])[0])
    assert s == np.float32(1.0) and BE.float_score_orders(q, kfs[-2])[1] != s


@pytest.mark.parametrize("name", BE.SEARCH_NAMES)
def test_database_search_equals_reference(O, name):
    if not O.have_matchref():
        pytest.skip("oracle/_ref/libmatchref.so not built")
    c = BE.search_case(name)
    port = BE.port_search(O, c)
    port_all = BE.port_search(O, c, ori=False)
    for k, (n_p, m_p) in zip(c["kfs"], port):
        n_r, m_r = O.ref_search_by_bow(k, c["F"], c["ratio"], c["ori"])
        assert n_r == n_p and np.array_equal(m_r, m_p)
    assert sum(n for n, _ in port) > 0
    _hits.setdefault("search", set()).update(BE.search_coverage(c, port, port_all))


def test_coverage_reaches_every_class():
    """Runs after the case tests of this module: every class of BE.CLASSES is reached by some case."""
    got = set().union(*_hits.values()) if _hits else set()
    if not {"voc", "query", "search"} <= set(_hits):
        pytest.skip("the case tests of this module did not all run")
    missing = sorted(set(BE.CLASSES) - got)
    assert not missing, missing
