"""KeyFrameDatabase::add of one new keyframe for each of N camera streams (LoopClosing::DetectLoop), N in 1, 8, 32: TUM-shaped 640x480
@1000 keyframes, resident through borb_frames_from_extractor with BoW from borb_frames_compute_bow (vocabulary k=10 L=6, random tree,
levelsup 4), each stream with its own database that already holds 300 keyframes.  Two arms:
   A (host path):     what a host does without resident adds: it keeps host copies of the keyframe's keys, descriptors, BowVector and
                      FeatureVector (the optional host outputs of the calls above) and calls borb_kfdb_add N times: host packing, a
                      cudaMalloc and a synchronous upload per keyframe;
   B (resident path): one borb_kfdb_add_frames for the N streams: one launch, one synchronisation, only the MapPoint masks uploaded.
Both arms are first run once on fresh databases through the Python API and must leave equal databases (borb_debug_kfdb_read, slot by
slot).  Timed: host clock around the C calls (prebuilt arguments, no Python packing inside the loop), median and 25th-75th percentile
of `--reps` runs after warm-up; every run appends N more slots (the databases grow from 300 keyframes).  A separate run with
torch.profiler gives the device time of kfdb_insert_kernel per call.  The card name and power limit are read in the same run.
usage: python tools/bench_kfdb_add.py [--reps 30] [--out DIR]  -> one JSON line on stdout (and DIR/bench_kfdb_add.json)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, sharding, synth                      # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit, warm_clocks          # noqa: E402
from tools.bench_track_ref import kernel_times                                 # noqa: E402

LEVELSUP = 4
TUM_K = (517.3, 516.5, 318.6, 255.3)
TUM_DIST = (0.2624, -0.9531, -0.0054, 0.0026, 1.1633)


def stats(ts):
    ts = np.asarray(ts) * 1e3
    return {"median_ms": round(float(np.median(ts)), 4), "p25_ms": round(float(np.percentile(ts, 25)), 4),
            "p75_ms": round(float(np.percentile(ts, 75)), 4)}


def main(reps, out_dir, ns=(1, 8, 32), warmup=3):
    n_max = max(ns)
    X = ORBextractor(1000)
    imgs = [synth.mono_frame(500 + i, 0, 0, 640, 480) for i in range(n_max)]
    outs = X.extract_batch(imgs)
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    mt = M.ORBmatcher(0.75, True)
    lib = mt._lib
    rng = np.random.default_rng(5)
    frames, host = M.frames_from_extractor(mt, X, list(range(n_max)), [len(k) for k, _ in outs], TUM_K, TUM_DIST)
    bows = mt.ComputeBoWBatch(voc, frames, LEVELSUP)
    hms = [(rng.random(F.resident.n) < 0.7).astype(np.uint8) for F in frames]
    # the host copies arm A keeps: keys_un and BoW from the calls' host outputs, descriptors from the extraction
    views = [M.KeyFrameView(mvKeysUn=host["keys_un"][i], mDescriptors=outs[i][1], mFeatVec=bows[i][1], has_mp=hms[i]) for i in range(n_max)]
    for i, F in enumerate(frames):
        r = F.resident.read(stereo=False)
        assert np.array_equal(r["keys_un"], views[i].mvKeysUn) and np.array_equal(r["desc"], views[i].mDescriptors)
    # 300-keyframe databases, one per stream, filled from 40 source keyframes
    src = X.extract_batch([synth.mono_frame(900 + i, 0, 0, 640, 480) for i in range(40)])
    src_views = []
    for k, d in src:
        bow, fv = voc.transform(d, LEVELSUP)
        src_views.append((M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.8).astype(np.uint8)), bow))

    def databases(n):
        dbs = [M.KeyFrameDatabase(mt) for _ in range(n)]
        for db in dbs:
            for i in range(300):
                db.add(*src_views[i % len(src_views)])
        return dbs

    # both arms on fresh databases: equal results
    dA, dB = databases(n_max), databases(n_max)
    for i, db in enumerate(dA):
        db.add(views[i], bows[i][0])
    mt.KfdbAddFramesBatch(dB, frames, hms)
    for a, b in zip(dA, dB):
        assert a.size() == b.size()
        ra, rb = a.read_slot(300), b.read_slot(300)
        assert all(np.array_equal(ra[k], rb[k]) for k in ("block", "host_meta"))
    del dA, dB

    # prebuilt C arguments of both arms
    cviews = [v._c() for v in views]
    bow_arr = [M.KeyFrameDatabase._bow_arrays(b) for b, _ in bows]
    slot = C.c_int32(-1)
    res = {"gpu": gpu_name_and_power_limit(), "streams": {}}
    for n in ns:
        dbs = databases(n)
        slots = np.zeros(n, np.int32)
        jobs = (M._KfdbAddJobC * n)()
        for j in range(n):
            jobs[j].db, jobs[j].frame = dbs[j]._h.value, frames[j].resident._h.value
            jobs[j].has_mp, jobs[j].slot_out = hms[j].ctypes.data, slots.ctypes.data + 4 * j

        def arm_a():
            for j in range(n):
                w, v = bow_arr[j]
                assert lib.borb_kfdb_add(dbs[j]._h, C.byref(cviews[j]), w.ctypes.data, v.ctypes.data, len(w), C.byref(slot)) == 0

        def arm_b():
            assert lib.borb_kfdb_add_frames(mt._h, jobs, n) == 0

        out = {}
        for name, fn in (("A_host_add", arm_a), ("B_add_frames", arm_b)):
            warm_clocks()
            for _ in range(warmup):
                fn()
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                fn()
                ts.append(time.perf_counter() - t0)
            out[name] = stats(ts)
        out["B_kernel_us"] = round(kernel_times(arm_b, ("kfdb_insert_kernel",))["kfdb_insert_kernel"], 2)
        out["A_over_B"] = round(out["A_host_add"]["median_ms"] / out["B_add_frames"]["median_ms"], 2)
        res["streams"][str(n)] = out
        del dbs
    line = {"bench": "kfdb_add", "config": "N streams x one TUM-shaped 640x480 @1000 keyframe into a 300-keyframe database each "
            "(vocabulary k=10 L=6, levelsup 4)", "reps": reps, **res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_kfdb_add.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    main(a.reps, a.out)
