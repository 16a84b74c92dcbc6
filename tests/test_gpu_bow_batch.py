"""GPU parity of the reference-keyframe step of Tracking::Track() for many camera streams on resident frames:
borb_frames_compute_bow (Frame::ComputeBoW, src/Frame.cc:395-402, on the device) must equal the oracle's transform and its
one-frame case borb_compute_bow bit for bit, and borb_search_by_bow_batch (SearchByBoW(KeyFrame*, Frame&), src/ORBmatcher.cc:159-288) must equal the
oracle and the single borb_search_by_bow on host views.  Both are a fixed number of launches whatever the batch size, and
argument errors are refused before anything is launched."""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest

from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCALE = (1.2 ** np.arange(8)).astype(np.float32)


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def views(oracle):
    return {s: mf.two_views(oracle, s) for s in (7, 8)}


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def resident(M, mt, keys, desc, has_mp=None):
    bounds = (0.0, 0.0, float(max(640.0, keys["x"].max() + 1 if len(keys) else 0)), float(max(480.0, keys["y"].max() + 1 if len(keys) else 0)))
    F = M.FrameView(keys, np.ascontiguousarray(desc, np.uint8), SCALE, bounds)
    return dataclasses.replace(F.make_resident(mt), has_mp=has_mp)


def flip_bits(rng, d, p):
    flip = rng.random((len(d), 32, 8)) < p
    return d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)


def same_bow(got, want):
    (bg, fg), (bw, fw) = got, want
    assert list(bg.items()) == list(bw.items())                    # same words, same order, bit-identical doubles
    assert np.array_equal(fg.node_id, fw.node_id) and np.array_equal(fg.start, fw.start) and np.array_equal(fg.feat_idx, fw.feat_idx)


def synthetic_frames(views):
    """(keys, desc) of ~1000, 1, 0 and 8192 features and of a frame whose descriptors repeat (word runs longer than one)."""
    rng = np.random.default_rng(5)
    kl, dl = views[7]["kl"], views[7]["dl"]
    big_k = np.concatenate([views[7]["kl"], views[7]["kr"], views[8]["kl"], views[8]["kr"]] * 3)[:8192]
    big_d = flip_bits(rng, np.concatenate([views[7]["dl"], views[7]["dr"], views[8]["dl"], views[8]["dr"]] * 3)[:8192], 0.03)
    assert len(big_d) == 8192
    rep = np.tile(np.arange(60), 9)
    return [(kl, dl), (kl[:1], dl[:1]), (kl[:0], dl[:0]), (big_k, big_d), (kl[rep], dl[rep])]


@pytest.mark.parametrize("levelsup", [4, 3])
def test_device_bow_equals_host_path_and_oracle(M, oracle, views, levelsup):
    from orb_slam2_b200.matcher import bow_and_featvec
    pv = oracle.PortVocabulary.random(10, 5, 21)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    mt = M.ORBmatcher(0.75, True)
    sets = synthetic_frames(views)
    frames = [resident(M, mt, k, d) for k, d in sets]
    c0 = launches(mt)
    got = mt.ComputeBoWBatch(voc, frames, levelsup)
    assert launches(mt) - c0 == 2
    for (k, d), g in zip(sets, got):
        same_bow(g, voc.ComputeBoW(d, levelsup))
        same_bow(g, bow_and_featvec(*pv.transform_raw(d, levelsup)))
    assert len(got[2][0]) == 0 and len(got[2][1].node_id) == 0 and list(got[2][1].start) == [0]
    assert len(got[3][1].feat_idx) == 8192
    assert len(got[4][0]) <= 60 and len(got[4][1].feat_idx) == 540            # every word run is at least 9 long
    # the same frames again, without host copies: still 2 launches; the device vectors stay searchable
    c0 = launches(mt)
    assert mt.ComputeBoWBatch(voc, frames[:1], levelsup, want_host=False) is None
    assert launches(mt) - c0 == 2


def test_stop_words_drop_out_of_both_vectors(M, oracle, views):
    from orb_slam2_b200.matcher import bow_and_featvec
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    w = e["weight"].copy()
    leaves = np.nonzero(e["is_leaf"])[0]
    w[leaves[::3]] = 0.0                                            # a third of the words are stop words
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], w, e["k"], e["L"])
    mt = M.ORBmatcher(0.75, True)
    d = views[8]["dr"]
    frames = [resident(M, mt, views[8]["kr"], d), resident(M, mt, views[7]["kl"], views[7]["dl"])]
    stop = e["word_id"][leaves[::3]]
    got = mt.ComputeBoWBatch(voc, frames, 2)
    for g, dd in zip(got, (d, views[7]["dl"])):
        same_bow(g, voc.ComputeBoW(dd, 2))
        wo, to, no = pv.transform_raw(dd, 2)                           # the oracle's descent, with the zeroed weights applied
        to = np.where(np.isin(wo, stop), 0.0, to)
        assert (to == 0).sum() > 50 and g[1].start[-1] == (to > 0).sum() and len(g[0]) < len(np.unique(wo))
        same_bow(g, bow_and_featvec(wo, to, no))


def test_frames_from_extractor_get_the_bow_of_their_descriptors(M, oracle):
    from orb_slam2_b200 import synth
    from orb_slam2_b200.matcher import bow_and_featvec
    from orb_slam2_b200.extractor import ORBextractor
    pv = oracle.PortVocabulary.random(10, 5, 21)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    X = ORBextractor(1000)
    outs = X.extract_batch([synth.mono_frame(60 + i, 0, 0, 640, 480) for i in range(3)])
    mt = M.ORBmatcher(0.75, True)
    frames, _ = M.frames_from_extractor(mt, X, [2, 0, 1], [len(outs[i][0]) for i in (2, 0, 1)], (517.3, 516.5, 318.6, 255.3), mode=0)
    got = mt.ComputeBoWBatch(voc, frames, 4)
    for i, g in zip((2, 0, 1), got):
        assert len(outs[i][1]) > 500
        same_bow(g, voc.ComputeBoW(outs[i][1], 4))
        same_bow(g, bow_and_featvec(*pv.transform_raw(outs[i][1], 4)))


def test_real_vocabulary_device_bow_equals_verbatim_dbow2(M):
    arr = os.path.join(ROOT, "oracle", "_ref", "orbvoc_arrays.npz")
    if not os.path.exists(arr):
        pytest.skip("oracle/_ref/orbvoc_arrays.npz absent (build() writes it where the reference tree is present)")
    a = np.load(arr)
    voc = M.ORBVocabulary.from_arrays(a["parent"], a["is_leaf"], a["desc"], a["weight"], int(a["k"][0]), int(a["L"][0]))
    g = np.load(os.path.join(ROOT, "tests", "golden", "voc_real.npz"))
    mt = M.ORBmatcher(0.75, True)
    names = ["extract_kitti_2000", "extract_euroc_1200", "extract_tum_1000"]
    sets = [np.load(os.path.join(ROOT, "tests", "golden", n + ".npz")) for n in names]
    frames = [resident(M, mt, s["keypoints"], s["descriptors"]) for s in sets]
    got = mt.ComputeBoWBatch(voc, frames, 4)
    for name, (bow, fv) in zip(names, got):
        assert np.array_equal(np.fromiter(bow.keys(), np.uint32, len(bow)), g[name + "_bow_word"]), name
        assert np.array_equal(np.fromiter(bow.values(), np.float64, len(bow)), g[name + "_bow_value"]), name
        assert np.array_equal(fv.node_id, g[name + "_fv_node"]) and np.array_equal(fv.start, g[name + "_fv_start"]), name
        assert np.array_equal(fv.feat_idx, g[name + "_fv_idx"]), name


def search_world(M, oracle, views):
    """Jobs of borb_search_by_bow_batch and, per job, the host views of the same data."""
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    mt = M.ORBmatcher(0.7, True)
    rng = np.random.default_rng(11)
    v7, v8 = views[7], views[8]
    mp = lambda n, frac=0.7: (rng.random(n) < frac).astype(np.uint8)
    # (frame keys, frame desc), then the keyframe: ("host", keys, desc, has_mp, empty_fv) or ("frame", index into frames, has_mp)
    frame_sets = [(v7["kl"], v7["dl"]), (v8["kl"], v8["dl"]), (v7["kr"][:300], v7["dr"][:300]), (v7["kl"][:0], v7["dl"][:0]),
                  (v8["kr"], v8["dr"]), (v7["kl"], v7["dl"])]
    kr8 = v8["kr"]
    specs = [
        ("host", v7["kr"], v7["dr"], mp(len(v7["kr"])), False),        # the other view of the scene
        ("frame", 6, mp(len(kr8))),                                   # resident keyframe: the right view of 8
        ("host", v7["kl"], v7["dl"], None, False),                    # has_mp NULL: nothing can match
        ("host", v8["kl"], v8["dl"], mp(len(v8["kl"])), False),        # a frame without features
        ("host", kr8, flip_bits(rng, v8["dr"], 0.02), mp(len(kr8)), False),   # a re-observation of the same frame: > 50 matches
        ("frame", 0, mp(len(v7["kl"]))),                              # the frame as its own reference keyframe: > 50 matches
        ("host", v8["kl"], v8["dl"], mp(len(v8["kl"])), True),         # a keyframe with an empty FeatureVector
        ("frame", 7, None),                                           # resident keyframe, has_mp NULL
    ]
    frame_sets += [(kr8, v8["dr"]), (v8["kl"], v8["dl"])]            # 6: resident keyframe of job 1, 7: of job 7
    job_frames = [0, 1, 2, 3, 4, 5, 0, 1]
    frames = [resident(M, mt, k, d) for k, d in frame_sets]
    bows = mt.ComputeBoWBatch(voc, frames, 2)
    jobs_kf, jobs_F, host_kf, host_F = [], [], [], []
    for spec, fi in zip(specs, job_frames):
        k, d = frame_sets[fi]
        jobs_F.append(frames[fi])
        host_F.append(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=bows[fi][1]))
        if spec[0] == "host":
            _, kk, kd, hm, empty = spec
            fv = M.FeatureVector(np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.uint32)) if empty else voc.ComputeBoW(kd, 2)[1]
            kv = M.KeyFrameView(mvKeysUn=kk, mDescriptors=kd, mFeatVec=fv, has_mp=hm)
            jobs_kf.append(kv); host_kf.append(kv)
        else:
            _, ri, hm = spec
            jobs_kf.append(dataclasses.replace(frames[ri], has_mp=hm))
            kk, kd = frame_sets[ri]
            host_kf.append(M.KeyFrameView(mvKeysUn=kk, mDescriptors=kd, mFeatVec=bows[ri][1], has_mp=hm))
    return mt, frames, jobs_kf, jobs_F, host_kf, host_F


@pytest.mark.parametrize("ori", [True, False])
def test_search_by_bow_batch_equals_oracle_and_single_calls(M, oracle, views, ori):
    mt0, frames, jobs_kf, jobs_F, host_kf, host_F = search_world(M, oracle, views)
    mt = M.ORBmatcher(0.7, ori)
    c0 = launches(mt)
    got = mt.SearchByBoWBatch(jobs_kf, jobs_F)
    assert launches(mt) - c0 == 1
    assert len(got) == len(jobs_F)
    for j, ((n_g, m_g), kv, Fv) in enumerate(zip(got, host_kf, host_F)):
        assert len(m_g) == len(Fv.mvKeysUn), j
        n_o, m_o = oracle.port_search_by_bow(kv, Fv, 0.7, ori)
        n_s, m_s = mt.SearchByBoW(kv, Fv)
        assert n_g == n_o == n_s and np.array_equal(m_g, m_o) and np.array_equal(m_g, m_s), (j, n_g, n_o, n_s)
    assert got[2][0] == 0 and got[3][0] == 0 and len(got[3][1]) == 0 and got[6][0] == 0 and np.all(got[6][1] == -1) and got[7][0] == 0
    assert got[4][0] > 50 and got[5][0] > 50 and got[0][0] > 0 and got[1][0] > 0
    # one launch whatever the number of jobs
    c0 = launches(mt)
    mt.SearchByBoWBatch(jobs_kf[:1], jobs_F[:1])
    assert launches(mt) - c0 == 1


def test_refusals_name_the_job_and_launch_nothing(M, oracle, views):
    from orb_slam2_b200._lib import BorbError
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    mt = M.ORBmatcher(0.7, True)
    v = views[7]
    kf = M.KeyFrameView(mvKeysUn=v["kr"], mDescriptors=v["dr"], mFeatVec=voc.ComputeBoW(v["dr"], 2)[1], has_mp=np.ones(len(v["kr"]), np.uint8))
    good = resident(M, mt, v["kl"], v["dl"])
    mt.ComputeBoWBatch(voc, [good], 2)

    def refused(call, job):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        assert ei.value.status == 1 and f"job {job}:" in str(ei.value), str(ei.value)
        assert launches(mt) == c0

    no_bow = resident(M, mt, v["kl"], v["dl"])
    refused(lambda: mt.SearchByBoWBatch([kf, kf], [good, no_bow]), 1)
    host = M.FrameView(v["kl"], v["dl"], SCALE, (0.0, 0.0, 640.0, 480.0))
    refused(lambda: mt.SearchByBoWBatch([kf, kf, kf], [good, good, host]), 2)
    refused(lambda: mt.SearchByBoWBatch([kf, dataclasses.replace(no_bow, has_mp=np.ones(len(v["kl"]), np.uint8))], [good, good]), 1)
    # a recycled frame block starts without BoW
    old = resident(M, mt, v["kl"], v["dl"])
    mt.ComputeBoWBatch(voc, [old], 2, want_host=False)
    assert mt.SearchByBoWBatch([kf], [old])[0][0] > 0
    old.resident.close()
    recycled = resident(M, mt, v["kl"], v["dl"])
    refused(lambda: mt.SearchByBoWBatch([kf, kf], [good, recycled]), 1)
    # the handle still works
    n, m = mt.SearchByBoWBatch([kf], [good])[0]
    n_s, m_s = mt.SearchByBoW(kf, M.KeyFrameView(mvKeysUn=v["kl"], mDescriptors=v["dl"], mFeatVec=voc.ComputeBoW(v["dl"], 2)[1]))
    assert n == n_s > 0 and np.array_equal(m, m_s)


def test_multistream_example_runs_its_reference_keyframe_step(tmp_path):
    so = os.path.join(ROOT, "orb_slam2_b200", "libborb.so")
    exe = tmp_path / "example_host"
    subprocess.check_call(["g++", "-std=c++14", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "integration", "example_multistream_host.cc"),
                           so, f"-Wl,-rpath,{os.path.dirname(so)}", "-o", str(exe)])
    r = subprocess.run([str(exe), "4"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "reference-keyframe search:" in r.stdout and r.stdout.strip().endswith("ok"), r.stdout[-3000:]
