"""CPU: the matcher port (oracle/orb_port_match.cpp) equals the verbatim ORBmatcher.cc on the descriptor-distance gate cases of
tests/match_gates.py, the verbatim build decides the two members of every pair differently, and the cases reach every class of
match_gates.CLASSES."""
import operator

import numpy as np
import pytest

from tests import match_gates as MG
from tests import proj_geometry as G


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_matchref() and oracle.have_frameref()):
        pytest.skip("oracle/_ref/libmatchref.so or libframeref.so not built (reference tree absent)")
    return oracle


def _ids():
    return [f"{c['cls']}-{c['member']}" for c in MG.cases()]


def port_equals_reference(O, c, method):
    """Asserts that the port and the verbatim build agree on one method of case c."""
    got, want = MG.run_port(O, c, method), MG.run_ref(O, c, method)
    if method == "local":
        fr_p, n_p, match = got
        fr_r, (n_r, owner), mps = want
        assert G.frustum_equal(fr_p, fr_r), (fr_p, fr_r)
        assert n_p == n_r and np.array_equal(O.owner_from_matches(c["F"], mps, match), owner)
    elif method in ("last", "kf", "sim3proj"):
        occ = c["F"].occupied if method != "last" else None
        assert got[0] == want[0] and np.array_equal(O.owner_from_state(occ, got[1]), want[1]), (got, want)
    elif method == "proj":
        assert got[0] == want[0] and np.array_equal(O.owner_from_matches(c["F"], c["mps"], got[1]), want[1]), (got, want)
    elif method == "init":
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), (got, want)
    elif method == "tri":
        assert np.array_equal(got, want), (got, want)
    else:
        assert got[0] == want[0] and np.array_equal(got[1], want[1]), (got, want)


@pytest.mark.parametrize("i", range(len(MG.cases())), ids=_ids())
def test_port_equals_reference(O, i):
    c = MG.cases()[i]
    for method in MG.methods(c):
        port_equals_reference(O, c, method)


@pytest.mark.parametrize("cls", sorted(MG.CLASSES))
def test_pair_members_are_decided_differently(O, cls):
    pair = {c["member"]: c for c in MG.cases() if c["cls"] == cls}
    assert sorted(pair) == [0, 1]
    assert MG.decided(O, pair[0]) is True and MG.decided(O, pair[1]) is False, cls


def test_every_class_is_reached():
    assert {c["cls"] for c in MG.cases()} == set(MG.CLASSES)
    assert set(MG.DECIDER) | {c["cls"] for c in MG.cases() if "kind" in c} == set(MG.CLASSES)
    assert not set(MG.CLASSES) & set(MG.NOT_COVERED)


def test_descriptors_sit_at_their_distances():
    """The Hamming distances the cases are built on, recomputed from the descriptors."""
    for c in MG.cases():
        if "kind" not in c:
            d12, d21 = c["dists"]
            assert MG.hamming(c["P"].descriptors[0], c["F"].mDescriptors[0]) == d12
            assert MG.hamming(c["P2"].descriptors[0], c["F"].mDescriptors[0]) == (d12 if d21 is None else d21)
        elif c["kind"] == "proj" and "dists" in c:
            q = c["mps"].descriptors[0]
            assert [MG.hamming(q, k) for k in c["F"].mDescriptors] == list(c["dists"]), c["cls"]
        elif c["kind"] in ("bow0", "bow1") and "dists" in c:
            q, cols = c["kf"].mDescriptors[0], c["F"].mDescriptors[c["n_fill"]:]
            want = [d for d in c["dists"] if d is not None]
            assert [MG.hamming(q, k) for k in cols] == want, c["cls"]
            assert all(MG.hamming(q, k) >= 200 for k in c["F"].mDescriptors[:c["n_fill"]])
            assert c["n_fill"] == 0 or len(c["F"].mDescriptors) > MG.BOW_JCAP
        elif c["kind"] == "init" and "dists" in c:
            q = c["F1"].mDescriptors[0]
            assert [MG.hamming(q, k) for k in c["F2"].mDescriptors] == [d for d in c["dists"] if d is not None], c["cls"]


def test_gates_restated_decide_the_pairs():
    """The numpy restatement of each ratio / no-second gate keeps member 0 and drops member 1; where the class is a float product
    boundary, a product evaluated in double decides the member on the product the other way (member 0 of the projection's `>`,
    member 1 of the `<` of SearchByBoW and SearchForInitialization)."""
    gate = {"proj": lambda c, **k: MG.proj_gate(c["dists"][0], 0, c["dists"][1], c["F"].mvKeysUn["octave"][1], c["ratio"], **k),
            "bow0": lambda c, **k: MG.bow_gate(0, *c["dists"], c["ratio"], **k),
            "bow1": lambda c, **k: MG.bow_gate(1, *c["dists"], c["ratio"], **k),
            "init": lambda c, **k: MG.init_gate(*c["dists"], c["ratio"], **k)}
    n = 0
    for c in MG.cases():
        if c.get("kind") not in gate or "dists" not in c:
            continue
        assert gate[c["kind"]](c) is (c["member"] == 0), (c["cls"], c["member"])
        on_product = c["member"] == (0 if c["kind"] == "proj" else 1)
        if "_ratio_" in c["cls"] and c["cls"].endswith(("_06", "_07", "_08", "_09")) and on_product:
            assert gate[c["kind"]](c, prod=MG.double_product) is (c["member"] == 1), c["cls"]
            n += 1
    assert n == 9


def test_ratio_separations():
    """Where the float32 product and the exact one decide `d1 < r*d2` / `d1 > r*d2` differently (d2 = 1..256): `<` at 0.6 and
    0.8, `>` at 0.7 and 0.9, nowhere at 0.75 and 1.0.  Each ratio class is built on the first such pair."""
    lt, gt = operator.lt, operator.gt
    counts = {r: (len(MG.separating(r, lt)), len(MG.separating(r, gt))) for r in (0.6, 0.7, 0.75, 0.8, 0.9, 1.0)}
    assert counts == {0.6: (33, 0), 0.7: (0, 25), 0.75: (0, 0), 0.8: (51, 0), 0.9: (0, 25), 1.0: (0, 0)}
    assert MG.first_separating(0.6, lt) == (3, 5) and MG.first_separating(0.7, gt) == (7, 10)
    assert MG.first_separating(0.9, gt) == (9, 10) and MG.first_separating(0.8, lt) == (4, 5)
    assert np.float32(np.float32(25.0 * 2.0 ** -30) * MG.INT_MAX_F) == 50.0


def test_init_walk_case_runs_the_window_walk():
    """init_excl_walk: B's window holds more than INIT_K entries and its INIT_K nearest are the features the earlier queries took
    at B's own distance (member 0) or all but one (member 1), so init_replay_kernel's prefix yields fewer than two."""
    for c in MG.cases():
        if c["cls"] != "init_excl_walk":
            continue
        B = c["F1"].mDescriptors[MG.INIT_K]
        d = [MG.hamming(B, f) for f in c["F2"].mDescriptors]
        assert len(d) > MG.INIT_K and sorted(d)[:MG.INIT_K] == d[:MG.INIT_K]
        assert d[:MG.INIT_K] == ([5] if c["member"] == 0 else [4]) + [5] * (MG.INIT_K - 1)
        taken = [MG.hamming(c["F1"].mDescriptors[k], c["F2"].mDescriptors[k]) for k in range(MG.INIT_K)]
        assert taken == [5] * MG.INIT_K
