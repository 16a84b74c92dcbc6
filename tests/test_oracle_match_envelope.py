"""CPU: the matcher port (oracle/orb_port_match.cpp) equals the verbatim ORBmatcher.cc on the size-envelope cases of
tests/match_envelope.py — 8192-feature frames, contested claim chains over several waves, tied descriptors in every Search* /
Fuse method, wide FeatureVector nodes, rotation-histogram boundaries — and those cases reach every coverage class listed in
match_envelope.CLASSES.
tests/test_gpu_adapters.py re-collects test_port_equals_reference against the adapter library."""
import numpy as np
import pytest

from tests import match_envelope as E


@pytest.fixture(scope="module")
def O(oracle):
    if not oracle.have_matchref():
        pytest.skip("oracle/_ref/libmatchref.so not built (reference tree absent)")
    return oracle


@pytest.mark.parametrize("name", E.NAMES)
def test_port_equals_reference(O, name):
    c = E.case(O, name)
    res = E.port_equals_reference(O, c)
    assert E.match_count(c, res) > 20


def test_cases_reach_every_coverage_class(oracle):
    hit = {}
    for name in E.NAMES:
        c = E.case(oracle, name)
        for k in E.coverage(c, E.run_port(oracle, c)):
            hit.setdefault(k, name)
    assert set(hit) == set(E.CLASSES), sorted(set(E.CLASSES) - set(hit))


def test_envelope_views_hold_exactly_the_limit(oracle):
    for shape in (E.KITTI, E.EUROC):
        v = E.envelope_views(oracle, shape)
        assert len(v["kl"]) == len(v["kr"]) == E.MATCH_MAX_FEATURES
        assert E.in_grid(v["kl"], (0.0, 0.0, float(v["w"]), float(v["h"]))).all()
    assert len(E.envelope_views(oracle, E.KITTI, n=E.MATCH_MAX_FEATURES + 1)["kl"]) == E.MATCH_MAX_FEATURES + 1


def test_histogram_cases_sit_on_the_tenth_boundary(oracle):
    """max2 (resp. max3) equals 0.1 * max1 in float: the bin is kept, and a tied bin later in the order is culled."""
    for name, kept in (("hist_max2_tenth", (1, 3, 5)), ("hist_max3_tenth", (2, 4, 6))):
        c = E.case(oracle, name)
        n, state = E.run_port(oracle, c)
        Cur, Last = c["F"], c["Last"]
        bins = np.array([E._rot_bin(Last.mvKeysUn["angle"][q], Cur.mvKeysUn["angle"][f]) for f, q in enumerate(state) if q >= 0])
        assert set(bins.tolist()) == set(kept) and n == len(bins), (name, sorted(set(bins.tolist())))
