"""The relocalisation step of a tracking tick (Tracking::Relocalization: Frame::ComputeBoW, the KeyFrameDatabase query and
SearchByBoW(KeyFrame*, Frame&) against the candidate keyframes) for N lost camera streams on resident frames, N in 1, 8, 32,
EuRoC-shaped 752x480 @1200, vocabulary k=10 L=6 (random tree), levelsup 4.  Two workloads:
   reloc:   every stream has its own 300-keyframe database and searches the 15 best-scoring slots of its query;
   config4: N queries against one shared 2000-keyframe database, every slot searched (BASELINE configs[4] per query).
Compared per tick:
   single:  N x (borb_compute_bow + borb_kfdb_query + borb_search_by_bow_db_pairs on host views): 3 synchronisations each;
   batched: one borb_frames_compute_bow + one borb_kfdb_query_batch + one borb_search_by_bow_db_batch.
Both arms must return equal results before anything is timed.  Host clock around the public Python calls (each ends in a
synchronise), median of `--reps` after warm-up, taken right after a burst of extraction work (tools/bench_configs.warm_clocks).
A second run with torch.profiler gives the device time of the score, packer, match and finalize kernels per batched tick.
usage: python tools/bench_reloc_batch.py [--reps 20] [--out DIR]  -> one JSON line on stdout (and DIR/bench_reloc_batch.json)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, sharding, synth                      # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit, med                  # noqa: E402
from tools.bench_track_ref import kernel_times                                 # noqa: E402

LEVELSUP = 4
KERNELS = ("kfdb_score_kernel", "bowdb_pack_kernel", "bowdb_match_kernel", "bowdb_finalize_kernel")


def build_db(mt, voc, outs, n_kf, masks, rng):
    """n_kf keyframes from the source frames, each with one of the bit-flip masks applied (~4 % of the descriptor bits)."""
    db = M.KeyFrameDatabase(mt)
    for j in range(n_kf):
        k, d = outs[j % len(outs)]
        d = d ^ masks[int(rng.integers(len(masks)))][:len(d)]
        bow, fv = voc.transform(d, LEVELSUP)
        db.add(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=(rng.random(len(k)) < 0.8).astype(np.uint8)), bow)
    return db


def same(a, b):
    (nm, off, pairs), (nm2, off2, pairs2) = a, b
    return np.array_equal(nm, nm2) and all(np.array_equal(pairs[off[k]:off[k] + nm[k]], pairs2[off2[k]:off2[k] + nm2[k]]) for k in range(len(nm)))


def main(reps, out_dir, ns=(1, 8, 32)):
    n_max = max(ns)
    X = ORBextractor(1200)
    n_src = 40
    outs = X.extract_batch([synth.mono_frame(50 + i, 0, 0, 752, 480) for i in range(n_src)])
    lost = X.extract_batch([synth.mono_frame(50 + (7 * i) % n_src, 0, 1, 752, 480) for i in range(n_max)])   # the scenes seen again
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    mt = M.ORBmatcher(0.75, True)
    rng = np.random.default_rng(1)
    masks = [np.packbits(rng.random((1400, 32, 8)) < 0.04, axis=2, bitorder="little").reshape(1400, 32) for _ in range(16)]
    F = [M.FrameView(k, d, sf, (0.0, 0.0, 752.0, 480.0)).make_resident(mt) for k, d in lost]
    own = [build_db(mt, voc, outs, 300, masks, np.random.default_rng(100 + s)) for s in range(n_max)]
    shared = build_db(mt, voc, outs, 2000, masks, np.random.default_rng(2))
    host_fv = [voc.ComputeBoW(d, LEVELSUP) for _, d in lost]
    cands = [np.argsort(-db.query(bow)[1], kind="stable")[:15].astype(np.int32) for db, (bow, _) in zip(own, host_fv)]
    res = {}
    for name, dbs_of, slots_of in (("reloc", lambda n: own[:n], lambda n: cands[:n]), ("config4", lambda n: [shared] * n, lambda n: [None] * n)):
        res[name] = {}
        for n in ns:
            dbs, slots = dbs_of(n), slots_of(n)

            def single():
                out = []
                for j in range(n):
                    k, d = lost[j]
                    bow, fv = voc.ComputeBoW(d, LEVELSUP)
                    q = dbs[j].query(bow)
                    out.append((q, dbs[j].SearchByBoWPairs(slots[j], M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv))))
                return out

            def batched():
                mt.ComputeBoWBatch(voc, F[:n], LEVELSUP, want_host=False)
                q = mt.KfdbQueryBatch(dbs, F[:n])
                return list(zip(q, mt.SearchByBoWDbBatch(dbs, slots, F[:n])))

            a, b = single(), batched()
            for (qa, sa), (qb, sb) in zip(a, b):
                assert all(np.array_equal(x, y) for x, y in zip(qa, qb)) and same(sa, sb)
            t_single, t_batch = med(single, reps), med(batched, reps)
            res[name][str(n)] = {"single_calls_us": t_single * 1e6, "batched_us": t_batch * 1e6,
                                 "keyframes_searched": int(sum(len(s[0]) for _, s in b)), "pairs": int(sum(len(s[2]) for _, s in b))}
    try:
        for name, dbs_of, slots_of in (("reloc", lambda n: own[:n], lambda n: cands[:n]), ("config4", lambda n: [shared] * n, lambda n: [None] * n)):
            for n in ns:
                dbs, slots = dbs_of(n), slots_of(n)
                res[name][str(n)]["kernel_us"] = kernel_times(lambda: (mt.KfdbQueryBatch(dbs, F[:n]), mt.SearchByBoWDbBatch(dbs, slots, F[:n])), KERNELS)
    except Exception as e:                                               # the profiler is optional for the host-clock table
        res["kernel_us_error"] = repr(e)
    line = {"config": "relocalisation step of N EuRoC-shaped 752x480 @1200 lost streams on resident frames: N x (borb_compute_bow + "
                      "borb_kfdb_query + borb_search_by_bow_db_pairs on host views) vs borb_frames_compute_bow + borb_kfdb_query_batch + "
                      "borb_search_by_bow_db_batch, per-tick host time; reloc = own 300-keyframe database and 15 candidates per stream, "
                      "config4 = one shared 2000-keyframe database, every slot",
            "gpu": gpu_name_and_power_limit(), "workloads": res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_reloc_batch.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    main(a.reps, a.out)
