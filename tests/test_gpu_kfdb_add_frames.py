"""GPU parity of borb_kfdb_add_frames, KeyFrameDatabase::add of many keyframes straight from their resident frames: every job must
leave its database exactly as borb_kfdb_add leaves it for a host view of the same frame - the same block bytes, slots, device bytes
and host row copies (borb_debug_kfdb_read) - so that every query and search of the database gives the same results whichever path
added a keyframe.  One launch whatever the number of jobs, argument errors refused before anything is allocated, and the new slots
independent of the frames they came from."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from orb_slam2_b200 import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCALE = (1.2 ** np.arange(8)).astype(np.float32)
LEVELSUP = 4
FIELDS = ("node", "start", "meta", "desc", "bow_word", "bow_value", "host_meta", "block")


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def voc(M):
    from orb_slam2_b200 import sharding
    return M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def random_keys(rng, n):
    from orb_slam2_b200._lib import KP_DTYPE
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(20, 600, n).astype(np.float32); k["y"] = rng.uniform(20, 440, n).astype(np.float32)
    k["angle"] = rng.uniform(0, 360, n).astype(np.float32); k["size"] = 31.0; k["octave"] = rng.integers(0, 8, n); k["class_id"] = -1
    return k


def flip_bits(rng, d, p):
    flip = rng.random((len(d), 32, 8)) < p
    return d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)


def resident(M, mt, keys, desc):
    return M.FrameView(keys, np.ascontiguousarray(desc, np.uint8), SCALE, (0.0, 0.0, 800.0, 600.0)).make_resident(mt)


def host_view(M, F, fv, has_mp):
    """The keyframe view borb_kfdb_add takes for a resident frame: its mvKeysUn and descriptors as the device holds them."""
    r = F.resident.read(stereo=False)
    return M.KeyFrameView(mvKeysUn=r["keys_un"], mDescriptors=r["desc"], mFeatVec=fv, has_mp=has_mp)


def same_db(dbA, dbB, slotsA=None, slotsB=None):
    """Equal slot counts and device bytes (whole databases), and for each compared slot pair the same block, arrays and host row
    copies."""
    if slotsA is None:
        assert dbA.size() == dbB.size()
    n = dbA.size()[0]
    for a, b in zip(slotsA if slotsA is not None else range(n), slotsB if slotsB is not None else range(n)):
        ra, rb = dbA.read_slot(a), dbB.read_slot(b)
        assert ra["n"] == rb["n"], (a, b)
        for k in FIELDS:
            assert ra[k].dtype == rb[k].dtype and np.array_equal(ra[k], rb[k]), (a, b, k)


def same_blocks(got, want):
    (nm, off, pairs), (nm2, off2, pairs2) = got, want
    assert np.array_equal(nm, nm2)
    for k in range(len(nm)):
        assert np.array_equal(pairs[off[k]:off[k] + nm[k]], pairs2[off2[k]:off2[k] + nm2[k]]), k


@pytest.fixture(scope="module")
def world(M, voc):
    """Resident frames with BoW at LEVELSUP: extractor frames of the synth, TUM (640x480) and EuRoC (752x480) shapes - monocular,
    stereo and RGB-D - and random frames of 1, 1000 and 8192 features.  Returns (matcher, [(name, FrameView, FeatureVector, bow)])."""
    from orb_slam2_b200.extractor import ORBextractor
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(61)
    frames, names = [], []
    X = ORBextractor(1000)
    imgs = [synth.mono_frame(300 + i, 0, 0, 640, 480) for i in range(3)]
    outs = X.extract_batch(imgs)
    K = (517.3, 516.5, 318.6, 255.3)
    fr, _ = M.frames_from_extractor(mt, X, [0, 1], [len(o[0]) for o in outs[:2]], K, (0.26, -0.95, -0.005, 0.002, 1.16))
    frames += fr; names += ["tum_mono_0", "tum_mono_1"]
    depth = [(1.0 + 2.0 * rng.random((480, 640))).astype(np.float32) for _ in range(2)]
    fr, _ = M.frames_from_extractor(mt, X, [1, 2], [len(o[0]) for o in outs[1:3]], K, bf=40.0, mode=2, depth=depth)
    frames += fr; names += ["tum_rgbd_1", "tum_rgbd_2"]
    XE = ORBextractor(1200)
    pairs = [synth.stereo_pair(90 + i, 0, 0, 752, 480) for i in range(2)]
    res = XE.stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], 47.9, 435.2)
    fr, _ = M.frames_from_extractor(mt, XE, [0, 2], [len(r["mvKeys"]) for r in res], (435.2, 435.2, 376.0, 240.0), bf=47.9, mode=1)
    frames += fr; names += ["euroc_stereo_0", "euroc_stereo_1"]
    Xs = ORBextractor(500)
    (k, d), = Xs.extract_batch([synth.mono_frame(7, 0, 0, 320, 240)])
    frames.append(resident(M, mt, k, d)); names.append("synth_320")
    for n in (1, 1000, 8192):
        frames.append(resident(M, mt, random_keys(rng, n), rng.integers(0, 256, (n, 32), dtype=np.uint8))); names.append(f"random_{n}")
    host = mt.ComputeBoWBatch(voc, frames, LEVELSUP)
    assert all(len(fv.feat_idx) > 0 for _, fv in host) and len(host[-1][1].feat_idx) == 8192
    return mt, [(nm, F, fv, bow) for nm, F, (bow, fv) in zip(names, frames, host)]


def masks(rng, n):
    return [None, np.ones(n, np.uint8), (rng.random(n) < 0.6).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8)]


def test_blocks_equal_the_host_path(M, world):
    """Every frame with has_mp NULL, all ones and random (nonzero bytes other than 1 included), added once through one
    borb_kfdb_add_frames and once through borb_kfdb_add on its host view: the same slots, blocks, arrays and host row copies."""
    mt, frames = world
    rng = np.random.default_rng(62)
    dbA, dbB = M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt)
    jobs = []
    for name, F, fv, bow in frames:
        for hm in masks(rng, F.resident.n):
            assert dbA.add(host_view(M, F, fv, hm), bow) == len(jobs)
            jobs.append((F, hm))
    c0 = launches(mt)
    slots = mt.KfdbAddFramesBatch(dbB, [F for F, _ in jobs], [hm for _, hm in jobs])
    assert launches(mt) - c0 == 1
    assert slots == list(range(len(jobs)))
    same_db(dbA, dbB)
    assert dbB._seq == dbA._seq and dbB._n == dbA._n
    r = dbB.read_slot(len(jobs) - 1)                         # random_8192, random mask
    assert len(r["meta"]) == 2 * 8192 and 0 < int(((r["meta"][0::2] >> 16) & 1).sum()) < 8192


def test_empty_and_stop_word_frames(M, voc):
    """A frame with 0 features, and frames whose every word is a stop word (empty BowVector and FeatureVector), get the slots,
    blocks and device bytes that borb_kfdb_add gives empty vectors."""
    from orb_slam2_b200 import sharding
    parent, is_leaf, desc, weight = sharding.random_vocabulary_arrays(10, 4, 9)
    stop = M.ORBVocabulary.from_arrays(parent, is_leaf, desc, np.zeros_like(weight), 10, 4)
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(63)
    empty = resident(M, mt, random_keys(rng, 0), np.zeros((0, 32), np.uint8))
    stopped = [resident(M, mt, random_keys(rng, n), rng.integers(0, 256, (n, 32), dtype=np.uint8)) for n in (1, 700)]
    (b0, f0), = mt.ComputeBoWBatch(voc, [empty], LEVELSUP)
    hs = mt.ComputeBoWBatch(stop, stopped, 2)
    assert all(len(b) == 0 and len(f.node_id) == 0 for b, f in [(b0, f0)] + hs)
    dbA, dbB = M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt)
    frames = [empty, stopped[0], stopped[1], stopped[1]]
    fvs = [f0, hs[0][1], hs[1][1], hs[1][1]]
    hms = [None, np.ones(1, np.uint8), None, np.ones(700, np.uint8)]
    for F, fv, hm in zip(frames, fvs, hms):
        dbA.add(host_view(M, F, fv, hm), {})
    assert mt.KfdbAddFramesBatch(dbB, frames, hms) == [0, 1, 2, 3]
    same_db(dbA, dbB)
    assert dbB.read_slot(2)["n"] == 700 and len(dbB.read_slot(2)["meta"]) == 0


def keyframes_300(M, mt, voc, world_frames, rng):
    """300 keyframes: bit-flipped re-observations of the world's extractor frames, resident with BoW; (frames, fvs, bows, masks)."""
    base = [(F.resident.read(stereo=False), F) for name, F, _, _ in world_frames if not name.startswith("random")]
    frames = []
    for i in range(300):
        r, _ = base[i % len(base)]
        frames.append(resident(M, mt, r["keys_un"], flip_bits(rng, r["desc"], 0.02 + 0.01 * (i % 5))))
    host = mt.ComputeBoWBatch(voc, frames, LEVELSUP)
    hms = [(rng.random(F.resident.n) < 0.7).astype(np.uint8) for F in frames]
    return frames, [fv for _, fv in host], [b for b, _ in host], hms


def test_databases_behave_the_same(M, voc, world):
    """Three 300-keyframe databases - through borb_kfdb_add, through one borb_kfdb_add_frames, and both paths interleaved - give the
    same queries (single and batched), SearchByBoW against the new slots, SearchByBoW(KeyFrame*, KeyFrame*) from a new slot, and
    DetectRelocalizationCandidates / DetectLoopCandidates sequences; again after set_has_mp_batch and after erasing new slots."""
    mt, wf = world
    rng = np.random.default_rng(64)
    frames, fvs, bows, hms = keyframes_300(M, mt, voc, wf, rng)
    n = len(frames)
    dbA, dbB, dbC = M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt)
    for i in range(n):
        dbA.add(host_view(M, frames[i], fvs[i], hms[i]), bows[i])
    c0 = launches(mt)
    assert mt.KfdbAddFramesBatch(dbB, frames, hms) == list(range(n))
    assert launches(mt) - c0 == 1
    i = 0
    while i < n:                                            # runs of 1-17 keyframes, alternating the two paths
        k = int(rng.integers(1, 18))
        if (i // 7) % 2:
            mt.KfdbAddFramesBatch(dbC, frames[i:i + k], hms[i:i + k])
        else:
            for j in range(i, min(n, i + k)):
                dbC.add(host_view(M, frames[j], fvs[j], hms[j]), bows[j])
        i += k
    same_db(dbA, dbB)
    same_db(dbA, dbC)
    dbs = (dbA, dbB, dbC)
    queries = [F for nm, F, _, _ in wf if not nm.startswith("random")][:6]
    q_host = mt.ComputeBoWBatch(voc, queries, LEVELSUP)
    qviews = [host_view(M, F, fv, None) for F, (_, fv) in zip(queries, q_host)]
    covis = lambda s: [x for x in (s - 2, s - 1, s + 1, s + 3, s + 7) if 0 <= x < n]

    def observe():
        out = []
        for db in dbs:
            o = {}
            o["query"] = [db.query(b) for b, _ in q_host]
            o["batch"] = mt.KfdbQueryBatch(db, queries)
            o["reloc"] = [db.DetectRelocalizationCandidates(b, covis) for b, _ in q_host]
            o["loop"] = [db.DetectLoopCandidates(bows[s], covis(s), covis, 0.01) for s in (5, 77, 150, 299)]
            live = [s for s in range(n) if s not in erased]
            o["bow"] = [db.SearchByBoWPairs(live[::3], F) for F in qviews[:3]]
            o["bow_batch"] = mt.SearchByBoWDbBatch(db, [live[1::4]] * 3, queries[3:6])
            o["kfkf"] = [db.SearchByBoWKFPairs(q, live[::5]) for q in (12, 150, 298) if q not in erased]
            out.append(o)
        a = out[0]
        for o in out[1:]:
            for (x, y) in zip(a["query"] + a["batch"], o["query"] + o["batch"]):
                assert all(np.array_equal(u, v) for u, v in zip(x, y))
            assert o["reloc"] == a["reloc"] and o["loop"] == a["loop"]
            for x, y in zip(a["bow"] + a["bow_batch"] + a["kfkf"], o["bow"] + o["bow_batch"] + o["kfkf"]):
                same_blocks(x, y)
        return a

    erased = set()
    a = observe()
    assert sum(len(r) for r in a["reloc"]) > 0 and max(int(x[0].max()) for x in a["bow"]) > 20 and max(int(x[0].max()) for x in a["kfkf"]) > 20
    new_masks = [(rng.random(frames[s].resident.n) < 0.4).astype(np.uint8) for s in (3, 12, 150, 151)]
    for db in dbs:
        db.set_has_mp_batch([3, 12, 150, 151], new_masks)
    same_db(dbA, dbB); same_db(dbA, dbC)
    b = observe()
    assert any(not np.array_equal(x[0], y[0]) for x, y in zip(a["kfkf"], b["kfkf"]))
    erased = {4, 150, 200}
    for db in dbs:
        for s in sorted(erased):
            db.erase(s)
    observe()
    c = mt.KfdbQueryBatch(dbB, queries[:1])[0]
    assert all(c[0][s] == 0 for s in erased)


def test_batch_semantics_and_frame_independence(M, voc, world):
    """32 jobs over 4 databases in interleaved order: per database the slots ascend in job order after its existing ones, one launch.
    The frames are then destroyed and their blocks recycled by new frames: the slots' blocks and searches do not change."""
    mt, wf = world
    rng = np.random.default_rng(65)
    frames, fvs, bows, hms = keyframes_300(M, mt, voc, wf, rng)
    dbs = [M.KeyFrameDatabase(mt) for _ in range(4)]
    for d, db in enumerate(dbs):
        for i in range(d):
            db.add(host_view(M, frames[40 + i], fvs[40 + i], hms[40 + i]), bows[40 + i])
    order = [0, 1, 2, 3, 3, 2, 1, 0, 2, 2, 0, 1, 3, 0, 1, 2, 3, 3, 3, 0, 1, 1, 2, 0, 0, 3, 2, 1, 0, 1, 2, 3]
    c0 = launches(mt)
    slots = mt.KfdbAddFramesBatch([dbs[d] for d in order], frames[:32], hms[:32])
    assert launches(mt) - c0 == 1
    for d in range(4):
        mine = [s for s, o in zip(slots, order) if o == d]
        assert mine == list(range(d, d + len(mine))), d
        assert dbs[d].size()[0] == d + len(mine) == len(dbs[d]._seq)
    ref = M.KeyFrameDatabase(mt)
    for j in range(32):
        ref.add(host_view(M, frames[j], fvs[j], hms[j]), bows[j])
    for d in range(4):
        same_db(ref, dbs[d], [j for j, o in enumerate(order) if o == d], [s for s, o in zip(slots, order) if o == d])
    queries = [F for nm, F, _, _ in wf if nm.startswith("tum")]
    mt.ComputeBoWBatch(voc, queries, LEVELSUP, want_host=False)
    before = [dbs[d].read_slot(s) for d, s in zip(order, slots)]
    search = lambda: mt.SearchByBoWDbBatch(dbs, [None] * 4, queries[:4]) + [dbs[d].SearchByBoWKFPairs(dbs[d].size()[0] - 1, None) for d in range(4)]
    s0 = search()
    for F in frames:
        F.resident.close()
    others = [resident(M, mt, random_keys(rng, 1000), rng.integers(0, 256, (1000, 32), dtype=np.uint8)) for _ in range(40)]
    mt.ComputeBoWBatch(voc, others, LEVELSUP, want_host=False)
    after = [dbs[d].read_slot(s) for d, s in zip(order, slots)]
    for x, y in zip(before, after):
        assert all(np.array_equal(x[k], y[k]) for k in FIELDS)
    for x, y in zip(s0, search()):
        same_blocks(x, y)
    assert max(int(x[0].max()) for x in s0) > 20


def test_refusals_name_the_job_and_change_nothing(M, voc, world):
    from orb_slam2_b200 import _lib
    from orb_slam2_b200._lib import BorbError
    mt, wf = world
    rng = np.random.default_rng(66)
    good = [F for _, F, _, _ in wf[:3]]
    db, db2 = M.KeyFrameDatabase(mt), M.KeyFrameDatabase(mt)
    mt.KfdbAddFramesBatch([db, db2], good[:2], None)
    sizes = lambda: (db.size(), db2.size(), len(db._seq), len(db2._seq))
    s0 = sizes()

    def refused(dbs, frames, job, slot_null=None):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            if slot_null is None:
                mt.KfdbAddFramesBatch(dbs, frames, None)
            else:
                jobs = (M._KfdbAddJobC * len(frames))()
                out = np.zeros(len(frames), np.int32)
                for j, (d, F) in enumerate(zip(dbs, frames)):
                    jobs[j].db, jobs[j].frame = d._h.value, F.resident._h.value
                    jobs[j].slot_out = None if j == slot_null else out.ctypes.data + 4 * j
                _lib.check(mt._lib.borb_kfdb_add_frames(mt._h, jobs, len(frames)), "borb_kfdb_add_frames")
        assert ei.value.status == 1 and str(ei.value).split(": ", 2)[2].startswith(f"job {job}:"), str(ei.value)
        assert launches(mt) == c0 and sizes() == s0

    refused([db, None, db2], good, 1)
    no_bow = resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
    refused([db, db2, db], [good[0], good[1], no_bow], 2)
    refused([db, db2, db], [good[0], M.FrameView(None, None, SCALE, (0, 0, 1, 1)), good[1]], 1)
    refused([db2, db, db], good, 2, slot_null=2)
    old = resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
    mt.ComputeBoWBatch(voc, [old], LEVELSUP, want_host=False)
    old.resident.close()
    recycled = resident(M, mt, random_keys(rng, 300), rng.integers(0, 256, (300, 32), dtype=np.uint8))
    refused([db, db], [good[0], recycled], 1)
    if _lib.device_count() > 1:                              # a database on another device than the matcher and the frames
        far = M.KeyFrameDatabase(mt, device=1)
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            mt.KfdbAddFramesBatch([db, far], good[:2], None)
        assert ei.value.status == 1 and "job 1:" in str(ei.value) and launches(mt) == c0 and far.size()[0] == 0
    assert mt.KfdbAddFramesBatch([], [], None) == [] and sizes() == s0


def test_concurrent_adds_and_searches(M, voc, world):
    """One thread adds batches of 5 keyframes while another queries the database and searches it (its own matcher each, as
    LoopClosing and Tracking): every query sees a whole number of batches and equals the final database's query cut to its slots,
    and every search equals the same search after the last add."""
    mt, wf = world
    rng = np.random.default_rng(67)
    frames, fvs, bows, hms = keyframes_300(M, mt, voc, wf, rng)
    frames, hms = frames[:60], hms[:60]
    db = M.KeyFrameDatabase(mt)
    mt.KfdbAddFramesBatch(db, frames[:5], hms[:5])
    mq = M.ORBmatcher(0.75, True)
    q = [F for nm, F, _, _ in wf if nm.startswith("tum")][:2]
    mq.ComputeBoWBatch(voc, q, LEVELSUP, want_host=False)
    seen, errors = [], []
    done = threading.Event()

    def adder():
        try:
            for i in range(5, 60, 5):
                mt.KfdbAddFramesBatch(db, frames[i:i + 5], hms[i:i + 5])
        except Exception as e:                                # noqa: BLE001 - reported by the main thread
            errors.append(e)
        finally:
            done.set()

    def searcher():
        try:
            while True:
                last = done.is_set()
                cw = mq.KfdbQueryBatch(db, q)
                sl = list(range(db.size()[0]))
                seen.append((cw, sl, mq.SearchByBoWDbBatch(db, [sl, sl[::2]], q)))
                if last:
                    break
        except Exception as e:                                # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=adder), threading.Thread(target=searcher)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert db.size()[0] == 60 and len(seen) >= 2
    final_q = mq.KfdbQueryBatch(db, q)
    for cw, sl, got in seen:
        for (c, s, f), (c2, s2, f2) in zip(cw, final_q):
            k = len(c)
            assert k % 5 == 0 and np.array_equal(c, c2[:k]) and np.array_equal(s, s2[:k]) and np.array_equal(f, f2[:k])
        want = mq.SearchByBoWDbBatch(db, [sl, sl[::2]], q)
        for x, y in zip(got, want):
            same_blocks(x, y)


@pytest.fixture(scope="module")
def add_adapter(tmp_path_factory):
    """tests/kfdb_add_adapter_wrap.cpp: kfdb_add_resident next to kfdb_add on stand-in KeyFrames, linked against libborb.so."""
    out = str(tmp_path_factory.mktemp("kfdb_add_adapter") / "libkfdbaddadapt.so")
    lib_dir = os.path.join(ROOT, "orb_slam2_b200")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "oracle", "cvmini"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "kfdb_add_adapter_wrap.cpp"), "-o", out, "-L", lib_dir,
                           "-l:libborb.so", "-Wl,-rpath," + lib_dir])
    lib = C.CDLL(out)
    lib.kfdb_add_adapter_run.restype = C.c_int
    lib.kfdb_add_adapter_run.argtypes = [C.c_int, C.c_void_p] + [C.c_void_p] * 2 + [C.c_void_p] + [C.c_void_p] * 3 + [C.c_void_p] * 3 + \
        [C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def test_adapter_add_resident_equals_kfdb_add(M, world, add_adapter):
    from orb_slam2_b200._lib import KP_DTYPE
    mt, wf = world
    rng = np.random.default_rng(68)
    sel = [x for x in wf if not x[0].startswith("random_8192")]
    views = [host_view(M, F, fv, None) for _, F, fv, _ in sel]
    hms = [None if i % 3 == 0 else (rng.random(F.resident.n) < 0.7).astype(np.uint8) for i, (_, F, _, _) in enumerate(sel)]
    keep = []

    def ptrs(arrs, dtype):
        a = [np.ascontiguousarray(x, dtype) if x is not None else None for x in arrs]
        keep.append(a)
        return (C.c_void_p * len(a))(*[x.ctypes.data if x is not None else None for x in a])
    bw = [np.fromiter(b.keys(), np.uint32, len(b)) for _, _, _, b in sel]
    bv = [np.fromiter(b.values(), np.float64, len(b)) for _, _, _, b in sel]
    n = len(sel)
    nf = np.array([len(v.mvKeysUn) for v in views], np.int32)
    nn = np.array([len(v.mFeatVec.node_id) for v in views], np.int32)
    nb = np.array([len(b) for b in bw], np.int32)
    err = C.create_string_buffer(512)
    rc = add_adapter.kfdb_add_adapter_run(n, nf.ctypes.data, ptrs([v.mvKeysUn for v in views], KP_DTYPE), ptrs([v.mDescriptors for v in views], np.uint8),
                                          nn.ctypes.data, ptrs([v.mFeatVec.node_id for v in views], np.uint32),
                                          ptrs([v.mFeatVec.start for v in views], np.int32), ptrs([v.mFeatVec.feat_idx for v in views], np.uint32),
                                          nb.ctypes.data, ptrs(bw, np.uint32), ptrs(bv, np.float64), ptrs(hms, np.uint8),
                                          (C.c_void_p * n)(*[F.resident._h.value for _, F, _, _ in sel]), err, 512)
    assert rc == 0, err.value.decode()
