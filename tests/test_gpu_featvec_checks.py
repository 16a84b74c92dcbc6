"""Every entry point that takes a borb_keyframe_view as a host view checks its FeatureVector before anything is staged or launched:
node ids strictly ascending, 0 <= start[0] <= start[1] <= ... <= start[n_nodes], every feat_idx[r] (r < start[n_nodes]) below n.
The kernels index shared and global memory with these values, so a violator must be refused with BORB_ERR_INVALID_ARG, the
batches naming the job, and no launch.  On valid input each SearchByBoW call, single, keyframe pair or batch, is one launch."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 64
SCALE = (1.2 ** np.arange(8)).astype(np.float32)
MALFORMED = ["equal_nodes", "descending_nodes", "decreasing_start", "negative_start0", "feat_idx_n"]


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def keyframe(M, seed, fv=None, flip=0.0):
    """N features in 4 FeatureVector nodes of N/4; the descriptors of seed 0 with a fraction `flip` of their bits flipped."""
    rng = np.random.default_rng(0)
    keys = np.zeros(N, M.KP_DTYPE)
    keys["x"], keys["y"] = rng.uniform(0, 640, N), rng.uniform(0, 480, N)
    keys["angle"], keys["octave"] = rng.uniform(0, 360, N), rng.integers(0, 8, N)
    desc = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    flips = np.random.default_rng(seed).random((N, 32, 8)) < flip
    desc ^= np.packbits(flips, axis=2, bitorder="little").reshape(N, 32)
    if fv is None:
        fv = M.FeatureVector(np.array([2, 5, 9, 14], np.uint32), np.arange(0, N + 1, N // 4, dtype=np.int32),
                             rng.permutation(N).astype(np.uint32))
    return M.KeyFrameView(mvKeysUn=keys, mDescriptors=desc, mFeatVec=fv, has_mp=np.ones(N, np.uint8), mvScaleFactors=SCALE,
                          mvLevelSigma2=SCALE * SCALE)


def malformed(M, kind):
    kf = keyframe(M, 1, flip=0.02)
    node, start, idx = kf.mFeatVec.node_id.copy(), kf.mFeatVec.start.copy(), kf.mFeatVec.feat_idx.copy()
    if kind == "equal_nodes":
        node[2] = node[1]
    elif kind == "descending_nodes":
        node[[1, 2]] = node[[2, 1]]
    elif kind == "decreasing_start":
        start[2] = start[1] - 1
    elif kind == "negative_start0":
        start[0] = -1
    else:
        idx[5] = N
    return dataclasses.replace(kf, mFeatVec=M.FeatureVector(node, start, idx))


@pytest.fixture(scope="module")
def world(M, oracle):
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    mt = M.ORBmatcher(0.7, True)
    good = keyframe(M, 1, flip=0.02)
    frames = [M.FrameView(good.mvKeysUn, good.mDescriptors, SCALE, (0.0, 0.0, 640.0, 480.0)).make_resident(mt) for _ in range(2)]
    bows = mt.ComputeBoWBatch(voc, frames, 2)
    good = dataclasses.replace(good, mFeatVec=bows[0][1])           # the host view of the resident frames
    assert len(good.mFeatVec.node_id) > 3
    db = M.KeyFrameDatabase(mt)
    db.add(good, {1: 0.5, 3: 0.25})
    return mt, db, good, frames


def entry_points(M, world, bad):
    """(name, call, job index of a batch or None) for every host-view side of every entry point that takes one."""
    mt, db, good, frames = world
    F12, ep = np.eye(3, dtype=np.float32), (320.0, 240.0)
    return [
        ("search_by_bow(keyframe)", lambda: mt.SearchByBoW([good, bad], good), None),
        ("search_by_bow(frame)", lambda: mt.SearchByBoW([good], bad), None),
        ("search_by_bow_kf(kf1)", lambda: mt.SearchByBoW_KF(bad, good), None),
        ("search_by_bow_kf(kf2)", lambda: mt.SearchByBoW_KF(good, bad), None),
        ("search_by_bow_batch(kf)", lambda: mt.SearchByBoWBatch([good, bad], frames), 1),
        ("search_for_triangulation(kf1)", lambda: mt.SearchForTriangulation(bad, good, F12, ep), None),
        ("search_for_triangulation(kf2)", lambda: mt.SearchForTriangulation(good, bad, F12, ep), None),
        ("search_for_triangulation_batch(kf1)", lambda: mt.SearchForTriangulationBatch([good, bad], [good, good], [F12] * 2, [ep] * 2), 1),
        ("search_for_triangulation_batch(kf2)", lambda: mt.SearchForTriangulationBatch([good, good], [good, bad], [F12] * 2, [ep] * 2), 1),
        ("kfdb_add", lambda: db.add(bad, {1: 0.5}), None),
        ("search_by_bow_db", lambda: db.SearchByBoW([0], bad), None),
        ("search_by_bow_db_pairs", lambda: db.SearchByBoWPairs(None, bad), None),
    ]


@pytest.mark.parametrize("kind", MALFORMED)
def test_malformed_featvec_is_refused_before_any_launch(M, world, kind):
    from orb_slam2_b200._lib import BorbError
    mt, db, good, frames = world
    bad = malformed(M, kind)
    slots = db.size()[0]
    for name, call, job in entry_points(M, world, bad):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        err = mt._lib.borb_last_error().decode()
        assert ei.value.status == 1, (name, str(ei.value))
        assert "FeatureVector" in err, (name, err)
        if job is not None:
            assert err.startswith(f"job {job}:"), (name, err)
        assert launches(mt) == c0, name
    assert db.size()[0] == slots                                      # the refused add took no slot
    # the handle still works
    assert mt.SearchByBoW_KF(good, good)[0] > 0


def test_one_launch_per_search_by_bow_call(M, world):
    mt, db, good, frames = world
    kfs = [keyframe(M, s, fv=good.mFeatVec, flip=f) for s, f in ((2, 0.02), (3, 0.05), (4, 0.3))]
    c0 = launches(mt)
    nm, match = mt.SearchByBoW(kfs, good)
    assert launches(mt) - c0 == 1
    for k, kf in enumerate(kfs):                                      # every keyframe against the one staged frame
        n1, m1 = mt.SearchByBoW(kf, good)
        assert n1 == nm[k] and np.array_equal(m1, match[k]), k
    assert nm[0] > N // 2 and nm[2] == 0
    c0 = launches(mt)
    n12, m12 = mt.SearchByBoW_KF(kfs[0], good)
    assert launches(mt) - c0 == 1 and n12 > N // 2
    c0 = launches(mt)
    got = mt.SearchByBoWBatch(kfs[:2], frames)
    assert launches(mt) - c0 == 1
    for k, (n, m) in enumerate(got):
        assert n == nm[k] and np.array_equal(m, match[k]), k
