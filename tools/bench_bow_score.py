"""LoopClosing::DetectLoop's minScore (src/LoopClosing.cc:121-140) for N camera streams, N in 1, 8, 32: the current keyframe scored
against its 40 covisible keyframes, 30 of which LoopClosing has added to the stream's database and 10 that LocalMapping has connected
but LoopClosing has not added yet.  EuRoC-shaped 752x480 @1200 keyframes, resident through borb_frames_from_extractor, BoW from
borb_frames_compute_bow (random k=10 L=6 tree, levelsup 4).  Three arms:
   a (bow_score):  one borb_bow_score_batch over every stream's 40 covisible keyframes (30 slots, 10 frames);
   b (scratch db): the workaround without it: the 10 unslotted keyframes of every stream go into a scratch database with one
                   borb_kfdb_add_frames, a second borb_kfdb_query_batch scores every stream's query against its scratch database, and
                   each scratch database is cleared (the 30 slotted scores come from the DetectLoopCandidates query either way);
   c (host):       the host scores its own copies of the BowVectors (kept from borb_frames_compute_bow's optional host outputs; that
                   download is not timed) with a C++ restatement of DBoW2's L1 merge, N x 40 calls.
The three arms must give the same float scores (bit for bit) before anything is timed.  Timed: host clock around calls that end in a
synchronisation (prebuilt C arguments), median and 25th-75th percentile of `--reps` runs after warm-up.  A separate torch.profiler
run gives the device time of kfdb_score_kernel in arm a.  The card name and power limit are read in the same run.
usage: python tools/bench_bow_score.py [--reps 20] [--out DIR]  -> one JSON line on stdout (and DIR/bench_bow_score.json)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle_lib as O                                             # noqa: E402
from orb_slam2_b200 import matcher as M, sharding, synth                      # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit, warm_clocks          # noqa: E402
from tools.bench_track_ref import kernel_times                                 # noqa: E402

LEVELSUP = 4
EUROC_K = (435.2, 435.2, 376.0, 240.0)
POOL, N_COVIS, N_SLOTTED = 80, 40, 30


def stats(ts):
    ts = np.asarray(ts) * 1e3
    return {"median_ms": round(float(np.median(ts)), 4), "p25_ms": round(float(np.percentile(ts, 25)), 4),
            "p75_ms": round(float(np.percentile(ts, 75)), 4)}


def main(reps, out_dir, ns=(1, 8, 32), warmup=3):
    O.build()
    X = ORBextractor(1200)
    outs = X.extract_batch([synth.mono_frame(700 + i, 0, 0, 752, 480) for i in range(POOL)])
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    mt = M.ORBmatcher(0.75, True)
    lib = mt._lib
    frames, _ = M.frames_from_extractor(mt, X, list(range(POOL)), [len(k) for k, _ in outs], EUROC_K)
    host = [M.KeyFrameDatabase._bow_arrays(b) for b, _ in mt.ComputeBoWBatch(voc, frames, LEVELSUP)]
    port = O._plib().orbport_bow_score_l1
    port.restype = C.c_double
    port.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    common, first = C.c_int32(0), C.c_uint32(0)
    res = {"gpu": gpu_name_and_power_limit(), "streams": {}}
    for n in ns:
        q = [j % POOL for j in range(n)]                                     # stream j: its query and its covisible keyframes
        cov = [[(j * 7 + 1 + k) % POOL for k in range(N_COVIS)] for j in range(n)]
        dbs = [M.KeyFrameDatabase(mt) for _ in range(n)]
        scratch = [M.KeyFrameDatabase(mt) for _ in range(n)]
        for j in range(n):
            assert mt.KfdbAddFramesBatch(dbs[j], [frames[c] for c in cov[j][:N_SLOTTED]], None) == list(range(N_SLOTTED))
        # arm a's jobs
        refs = [(M._BowRefC * N_COVIS)(*[M._BowRefC(None, dbs[j]._h.value, k) for k in range(N_SLOTTED)] +
                                       [M._BowRefC(frames[c].resident._h.value, None, 0) for c in cov[j][N_SLOTTED:]]) for j in range(n)]
        sa = np.zeros((n, N_COVIS), np.float32)
        jobs_a = (M._BowScoreJobC * n)()
        for j in range(n):
            jobs_a[j].query = M._BowRefC(frames[q[j]].resident._h.value, None, 0)
            jobs_a[j].targets, jobs_a[j].n_targets, jobs_a[j].score = C.addressof(refs[j]), N_COVIS, sa[j].ctypes.data
        # arm b's jobs: the scratch adds and the second query
        n_un = N_COVIS - N_SLOTTED
        slots_b = np.zeros(n * n_un, np.int32)
        add_b = (M._KfdbAddJobC * (n * n_un))()
        for j in range(n):
            for k, c in enumerate(cov[j][N_SLOTTED:]):
                J = add_b[j * n_un + k]
                J.db, J.frame, J.has_mp, J.slot_out = scratch[j]._h.value, frames[c].resident._h.value, None, slots_b.ctypes.data + 4 * (j * n_un + k)
        cw, sb, fw, ns_b = (np.zeros((n, n_un), np.int32), np.zeros((n, n_un), np.float32), np.zeros((n, n_un), np.uint32),
                            np.zeros(n, np.int32))
        query_b = (M._KfdbQueryJobC * n)()
        for j in range(n):
            J = query_b[j]
            J.db, J.frame = scratch[j]._h.value, frames[q[j]].resident._h.value
            J.common_words, J.score, J.first_word, J.cap, J.n_slots = cw[j].ctypes.data, sb[j].ctypes.data, fw[j].ctypes.data, n_un, ns_b.ctypes.data + 4 * j
        sc = np.zeros((n, N_COVIS), np.float32)

        def arm_a():
            assert lib.borb_bow_score_batch(mt._h, jobs_a, n) == 0

        def arm_b():
            assert lib.borb_kfdb_add_frames(mt._h, add_b, n * n_un) == 0
            assert lib.borb_kfdb_query_batch(mt._h, query_b, n) == 0
            for db in scratch:
                assert lib.borb_kfdb_clear(db._h) == 0

        def arm_c():
            for j in range(n):
                w1, v1 = host[q[j]]
                for k, c in enumerate(cov[j]):
                    w2, v2 = host[c]
                    sc[j, k] = port(w1.ctypes.data, v1.ctypes.data, len(w1), w2.ctypes.data, v2.ctypes.data, len(w2), C.addressof(common),
                                    C.addressof(first))

        # equal results: a against c everywhere, b against c on the unslotted keyframes (the slotted ones come from the main query)
        arm_a(); arm_b(); arm_c()
        slotted = np.stack([s for _, s, _ in mt.KfdbQueryBatch(dbs, [frames[x] for x in q])])
        assert np.array_equal(sa.view(np.uint32), sc.view(np.uint32))
        assert np.array_equal(sb.view(np.uint32), sc[:, N_SLOTTED:].view(np.uint32))
        assert np.array_equal(slotted.view(np.uint32), sc[:, :N_SLOTTED].view(np.uint32))
        out = {}
        for name, fn in (("a_bow_score", arm_a), ("b_scratch_db", arm_b), ("c_host", arm_c)):
            warm_clocks()
            for _ in range(warmup):
                fn()
            ts = []
            for _ in range(reps):
                t0 = time.perf_counter()
                fn()
                ts.append(time.perf_counter() - t0)
            out[name] = stats(ts)
        out["a_kernel_us"] = round(kernel_times(arm_a, ("kfdb_score_kernel",))["kfdb_score_kernel"], 2)
        out["b_over_a"] = round(out["b_scratch_db"]["median_ms"] / out["a_bow_score"]["median_ms"], 2)
        out["c_over_a"] = round(out["c_host"]["median_ms"] / out["a_bow_score"]["median_ms"], 2)
        res["streams"][str(n)] = out
        del dbs, scratch
    line = {"bench": "bow_score", "config": f"N streams x one EuRoC-shaped 752x480 @1200 keyframe against {N_COVIS} covisible keyframes "
            f"({N_SLOTTED} database slots, {N_COVIS - N_SLOTTED} frames not yet added; vocabulary k=10 L=6, levelsup 4)", "reps": reps, **res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_bow_score.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    main(a.reps, a.out)
