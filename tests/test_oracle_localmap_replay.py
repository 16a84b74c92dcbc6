"""CPU: the CreateNewMapPoints replay that borb_search_for_triangulation_batch documents, on the verbatim SearchForTriangulation
(src/ORBmatcher.cc:657-823, oracle/_ref/libmatchref.so).  LocalMapping searches the new keyframe against each neighbour in turn,
and every pair it triangulates gives a kf1 feature a MapPoint that later searches skip (:697-703).  Without the orientation check
each kf1 row depends only on its own MapPoint flag, so one search per neighbour with the entry mask, filtered by the flags the
earlier neighbours set, equals the sequential searches; with the orientation check the rotation histogram couples the rows and
it does not."""
import dataclasses

import numpy as np
import pytest

from tests import localmap_fixtures as lf
from tests import match_fixtures as mf

K2 = (525.0, 525.0, 319.5, 239.5)


@pytest.fixture(scope="module")
def O(oracle):
    if not oracle.have_matchref():
        pytest.skip("oracle/_ref/libmatchref.so not built (reference tree absent)")
    return oracle


@pytest.fixture(scope="module")
def world(oracle):
    v = mf.two_views(oracle, 7)
    kf1, kf2s = lf.neighbourhood(v, oracle.PortVocabulary.random(10, 4, 5))
    return kf1, kf2s


def searcher(O, ori):
    F12 = mf.rectified_F12(7)
    Ow1 = np.array([0.3, -0.05, -2.0], np.float32)                    # the epipole falls inside the image
    T2w = np.eye(4, dtype=np.float32)[:3]
    return lambda kf1, kf2: O.ref_search_for_triangulation(kf1, kf2, F12, Ow1, T2w, K2, False, ori)


def test_entry_mask_searches_replay_the_sequential_ones(O, world):
    kf1, kf2s = world
    search = searcher(O, False)
    seq = lf.sequential(search, kf1, kf2s)
    rep = lf.replay([search(kf1, kf2) for kf2 in kf2s], kf1.has_mp)
    for i, (a, b) in enumerate(zip(seq, rep)):
        assert np.array_equal(a, b), i
    assert all(len(p) > 10 for p in seq)
    # the mask matters: later neighbours lose rows that earlier ones triangulated
    assert sum(len(search(kf1, kf2)) - len(p) for kf2, p in zip(kf2s[1:], seq[1:])) > 20


def rotated(kf2s, frac=0.1, seed=1):
    """The neighbours with a tenth of their features turned by 90 degrees: a second rotation bin near the 10 % cut of
    ComputeThreeMaxima (:1601-1642), so that which rows an earlier neighbour masked decides whether the bin survives."""
    rng = np.random.default_rng(seed)
    out = []
    for k in kf2s:
        kp = k.mvKeysUn.copy()
        sel = rng.random(len(kp)) < frac
        kp["angle"][sel] = (kp["angle"][sel] + 90.0) % 360.0
        out.append(dataclasses.replace(k, mvKeysUn=kp))
    return out


def test_with_the_orientation_check_the_replay_is_not_exact(O, world):
    kf1, kf2s = world
    kf2s = rotated(kf2s)
    assert all(np.array_equal(a, b) for a, b in zip(lf.sequential(searcher(O, False), kf1, kf2s),
                                                     lf.replay([searcher(O, False)(kf1, k) for k in kf2s], kf1.has_mp)))
    search = searcher(O, True)
    seq = lf.sequential(search, kf1, kf2s)
    rep = lf.replay([search(kf1, kf2) for kf2 in kf2s], kf1.has_mp)
    assert any(not np.array_equal(a, b) for a, b in zip(seq, rep))
