"""Loop closure's first search, SearchByBoW(KeyFrame*, KeyFrame*) (LoopClosing::ComputeSim3, src/LoopClosing.cc:251-280), on the
resident keyframe database.  EuRoC-shaped 752x480 @1200 keyframes, vocabulary k=10 L=6 (random tree), levelsup 4.  Workloads:
   candidates: one loop-closing keyframe against k = 3, 10, 30 candidates of a 2000-keyframe database:
               k x borb_search_by_bow_kf on host views (one upload and one synchronisation per pair, today's drop-in)
               vs one borb_search_by_bow_kf_db_pairs;
   streams:    32 streams, each with its own 300-keyframe database and 15 candidates: 32 borb_search_by_bow_kf_db_pairs
               vs one borb_search_by_bow_kf_db_batch;
   kernels:    device time (torch.profiler, a run of its own) of the KF-KF search of one slot against all 2000 slots, and of the
               KF-Frame (relocalisation) search of the same keyframe as a frame against all 2000 slots.
Both arms of every workload must return equal results before anything is timed.  Host clock around the public Python calls (each
ends in a synchronise) after warm-up: median, 25th and 75th percentile of `--reps`.
usage: python tools/bench_loop_closure.py [--reps 30] [--out DIR]  -> one JSON line on stdout (and DIR/bench_loop_closure.json)."""
import argparse
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
KERNELS = ("bowkf_pack_kernel", "bowkf_match_kernel", "bowdb_pack_kernel", "bowdb_match_kernel", "bowdb_finalize_kernel")


def spread(f, reps):
    f()
    warm_clocks()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); f(); t.append(time.perf_counter() - t0)
    p25, p50, p75 = np.percentile(np.asarray(t) * 1e6, [25, 50, 75])
    return {"median_us": float(p50), "p25_us": float(p25), "p75_us": float(p75)}


def build_db(mt, voc, outs, n_kf, masks, rng):
    """n_kf keyframes from the source frames, each with one of the bit-flip masks applied (~4 % of the descriptor bits)."""
    db = M.KeyFrameDatabase(mt)
    views = []
    for j in range(n_kf):
        k, d = outs[j % len(outs)]
        d = d ^ masks[int(rng.integers(len(masks)))][:len(d)]
        bow, fv = voc.transform(d, LEVELSUP)
        v = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.8).astype(np.uint8))
        db.add(v, bow)
        views.append(v)
    return db, views


def dense(nm, off, pairs, n1):
    out = np.full((len(nm), n1), -1, np.int32)
    for k in range(len(nm)):
        pr = pairs[off[k]:off[k] + nm[k]]
        out[k, (pr & 0xFFFF).astype(np.int64)] = (pr >> 16).astype(np.int32)
    return out


def same(a, b):
    (nm, off, pairs), (nm2, off2, pairs2) = a, b
    return np.array_equal(nm, nm2) and all(np.array_equal(pairs[off[k]:off[k] + nm[k]], pairs2[off2[k]:off2[k] + nm2[k]]) for k in range(len(nm)))


def main(reps, out_dir):
    X = ORBextractor(1200)
    n_src = 40
    outs = X.extract_batch([synth.mono_frame(50 + i, 0, 0, 752, 480) for i in range(n_src)])
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(1)
    masks = [np.packbits(rng.random((1400, 32, 8)) < 0.04, axis=2, bitorder="little").reshape(1400, 32) for _ in range(16)]
    big, views = build_db(mt, voc, outs, 2000, masks, np.random.default_rng(2))
    q = 7
    res = {"candidates": {}, "streams": {}}
    for k in (3, 10, 30):
        cands = np.random.default_rng(k).choice(2000, k, replace=False).astype(np.int32)
        cands[0] = q + n_src                                              # a keyframe of the same scene

        def single():
            return [mt.SearchByBoW_KF(views[q], views[c]) for c in cands]

        def one_call():
            return big.SearchByBoWKFPairs(q, cands)

        a, b = single(), one_call()
        d = dense(*b, len(views[q].mvKeysUn))
        assert all(n == b[0][i] and np.array_equal(m, d[i]) for i, (n, m) in enumerate(a))
        res["candidates"][str(k)] = {"single_calls": spread(single, reps), "one_call": spread(one_call, reps), "matches": int(b[0].sum())}
    own = [build_db(mt, voc, outs, 300, masks, np.random.default_rng(100 + s))[0] for s in range(32)]
    qs = [int(np.random.default_rng(200 + s).integers(300)) for s in range(32)]
    sls = [np.random.default_rng(300 + s).choice(300, 15, replace=False).astype(np.int32) for s in range(32)]

    def singles():
        return [db.SearchByBoWKFPairs(qq, sl) for db, qq, sl in zip(own, qs, sls)]

    def batch():
        return mt.SearchByBoWKFDbBatch(own, qs, sls)

    a, b = singles(), batch()
    assert all(same(x, y) for x, y in zip(a, b))
    res["streams"]["32"] = {"single_calls": spread(singles, reps), "batch": spread(batch, reps), "matches": int(sum(int(x[0].sum()) for x in b))}
    try:
        kq, dq = outs[q % n_src]
        Fq = M.KeyFrameView(mvKeysUn=kq, mDescriptors=views[q].mDescriptors, mFeatVec=views[q].mFeatVec)
        res["kernels_all_2000_slots"] = {
            "kf_kf_us": kernel_times(lambda: big.SearchByBoWKFPairs(q, None), KERNELS),
            "kf_frame_us": kernel_times(lambda: big.SearchByBoWPairs(None, Fq), KERNELS)}
    except Exception as e:                                               # the profiler is optional for the host-clock table
        res["kernel_us_error"] = repr(e)
    line = {"config": "SearchByBoW(KeyFrame*, KeyFrame*) on the resident keyframe database, EuRoC-shaped 752x480 @1200, k=10 L=6 "
                      "vocabulary, levelsup 4: candidates = one keyframe vs k candidates of a 2000-keyframe database (k x "
                      "borb_search_by_bow_kf vs one borb_search_by_bow_kf_db_pairs); streams = 32 own 300-keyframe databases, 15 "
                      "candidates each (32 single calls vs one batch); host time per call sequence",
            "gpu": gpu_name_and_power_limit(), "workloads": res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_loop_closure.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    main(a.reps, a.out)
