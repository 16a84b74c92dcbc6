"""MapPoint::ComputeDistinctiveDescriptors of LocalMapping::SearchInNeighbors (src/LocalMapping.cc:526) for N camera streams, N in 1, 8,
32: each stream refreshes ~1500 MapPoints of 2-30 observations over its 20 resident neighbour keyframes (TUM-shaped 640x480 @1000,
made resident by borb_frames_from_extractor).  Each observation takes a feature of its own (a feature holds one MapPoint); a point
with more than 20 observations sees some keyframe at two features.  Three arms, all streams in one call each:
   (a) today without host copies: borb_debug_frame_read of every observing keyframe, a host gather of the rows, then
       borb_distinctive_descriptors, and the chosen rows picked on the host;
   (b) today with host copies of the keyframes' descriptors: the host gather, borb_distinctive_descriptors, the chosen rows;
   (c) borb_distinctive_descriptors_frames: only the observation tables go up, best_idx and the chosen rows come down.
All arms must give the same best_idx and descriptors before anything is timed.  Timed with the host clock, the three arms alternating
rep by rep after warm-up, median and 25th-75th percentile: once around the public Python calls (ResidentFrame.read,
ORBmatcher.ComputeDistinctiveDescriptors / ComputeDistinctiveDescriptorsFrames, whose per-point list packing is part of what a Python
caller pays), and once around the C calls with prebuilt flat arguments (what a C++ host pays).  A separate run with torch.profiler
gives the device time of distinctive_kernel in arms (b) and (c).  The card name and power limit are read in the same run.
usage: python tools/bench_distinctive_frames.py [--reps 30] [--out DIR]  -> one JSON line on stdout (and DIR/bench_distinctive_frames.json)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, synth                                 # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit, warm_clocks          # noqa: E402
from tools.bench_track_ref import kernel_times                                 # noqa: E402

TUM_K = (517.3, 516.5, 318.6, 255.3)
TUM_DIST = (0.2624, -0.9531, -0.0054, 0.0026, 1.1633)
N_KF = 20


def stats(ts):
    ts = np.asarray(ts) * 1e3
    return {"median_ms": round(float(np.median(ts)), 4), "p25_ms": round(float(np.percentile(ts, 25)), 4),
            "p75_ms": round(float(np.percentile(ts, 75)), 4)}


def stream_points(rng, n_feat):
    """One stream's refresh: groups of (keyframe in 0..19, feature) pairs; each observation takes a free feature."""
    free = [list(rng.permutation(n)) for n in n_feat]
    groups = []
    for _ in range(int(rng.integers(1400, 1601))):
        N = int(min(2 + rng.geometric(1 / 7), 30))
        kfs = rng.choice(N_KF, N, replace=N > N_KF)
        groups.append((kfs.astype(np.int32), np.array([free[k].pop() for k in kfs], np.int32)))
    return groups


def main(reps, out_dir, ns=(1, 8, 32), warmup=3):
    n_max = max(ns)
    X = ORBextractor(1000)
    outs = X.extract_batch([synth.mono_frame(700 + i, 0, 0, 640, 480) for i in range(40)])
    mt = M.ORBmatcher()
    lib = mt._lib
    rng = np.random.default_rng(11)
    # N_KF resident keyframes per stream, from the 40 extracted images (distinct frames, shared image content)
    imgs = [(s * 7 + i) % 40 for s in range(n_max) for i in range(N_KF)]
    frames, _ = M.frames_from_extractor(mt, X, imgs, [len(outs[i][0]) for i in imgs], TUM_K, TUM_DIST, want_host=False)
    n_feat = [len(outs[i][0]) for i in imgs]
    points = [stream_points(rng, n_feat[s * N_KF:(s + 1) * N_KF]) for s in range(n_max)]
    res = {"gpu": gpu_name_and_power_limit(), "streams": {}}
    for n in ns:
        fr = frames[:n * N_KF]
        rfs = [F.resident for F in fr]
        groups = [(f + s * N_KF, k) for s in range(n) for f, k in points[s]]
        n_pts = len(groups)
        # flat arguments: observation tables, offsets, frame table, and each observation's row in the stacked host copy
        off = np.zeros(n_pts + 1, np.int32)
        off[1:] = np.cumsum([len(f) for f, _ in groups])
        obs_f = np.concatenate([f for f, _ in groups]).astype(np.int32)
        obs_k = np.concatenate([k for _, k in groups]).astype(np.int32)
        table = (C.c_void_p * len(rfs))(*[rf._h.value for rf in rfs])
        cap = max(rf.n for rf in rfs)
        stacked = np.zeros((len(rfs), cap, 32), np.uint8)
        for i, rf in enumerate(rfs):
            stacked[i, :rf.n] = rf.read(stereo=False)["desc"]
        n_obs = int(off[-1])
        best = np.full(n_pts, -1, np.int32)
        desc = np.zeros((n_pts, 32), np.uint8)
        best_b = np.full(n_pts, -1, np.int32)

        # --- public Python calls
        def py_a():
            host = [rf.read(stereo=False)["desc"] for rf in rfs]
            g = [np.stack([host[a][b] for a, b in zip(f, k)]) for f, k in groups]
            b = mt.ComputeDistinctiveDescriptors(g)
            return b, np.stack([x[i] for x, i in zip(g, b)])

        def py_b():
            g = [stacked[f, k] for f, k in groups]
            b = mt.ComputeDistinctiveDescriptors(g)
            return b, np.stack([x[i] for x, i in zip(g, b)])

        def py_c():
            return mt.ComputeDistinctiveDescriptorsFrames(fr, groups)

        # --- C calls on prebuilt flat arguments
        def c_a():
            for i, rf in enumerate(rfs):
                assert lib.borb_debug_frame_read(rf._h, None, stacked[i].ctypes.data, None, None, None, None) == 0
            return c_b()

        def c_b():
            rows = stacked[obs_f, obs_k]
            assert lib.borb_distinctive_descriptors(mt._h, rows.ctypes.data, off.ctypes.data, n_pts, best_b.ctypes.data) == 0
            return best_b, rows[off[:-1] + best_b]

        def c_c():
            assert lib.borb_distinctive_descriptors_frames(mt._h, table, len(rfs), obs_f.ctypes.data, obs_k.ctypes.data, off.ctypes.data,
                                                           n_pts, best.ctypes.data, desc.ctypes.data) == 0
            return best, desc

        arms = {"python": (("a_read_gather_single", py_a), ("b_gather_single", py_b), ("c_frames", py_c)),
                "c_abi": (("a_read_gather_single", c_a), ("b_gather_single", c_b), ("c_frames", c_c))}
        ref_b, ref_d = py_c()
        for group in arms.values():
            for _, fn in group:
                b, d = fn()
                assert np.array_equal(b, ref_b) and np.array_equal(d, ref_d)
        assert np.all(ref_b >= 0)
        out = {"points": n_pts, "observations": n_obs, "keyframes": len(rfs),
               "h2d_bytes": {"a_b": n_obs * 32 + 4 * (n_pts + 1) + 8, "c": n_obs * 8 + 4 * (n_pts + 1) + 8 * len(rfs)},
               "d2h_bytes": {"a_keyframe_reads": int(sum(rf.n for rf in rfs)) * 32, "a_b": n_pts * 4, "c": n_pts * 36}}
        for level, group in arms.items():
            warm_clocks()
            for _ in range(warmup):
                for _, fn in group:
                    fn()
            ts = {name: [] for name, _ in group}
            for _ in range(reps):
                for name, fn in group:
                    t0 = time.perf_counter()
                    fn()
                    ts[name].append(time.perf_counter() - t0)
            out[level] = {name: stats(t) for name, t in ts.items()}
        out["kernel_us"] = {"b": round(kernel_times(c_b, ("distinctive_kernel",))["distinctive_kernel"], 2),
                            "c": round(kernel_times(c_c, ("distinctive_kernel",))["distinctive_kernel"], 2)}
        res["streams"][str(n)] = out
    line = {"bench": "distinctive_frames", "config": f"N streams x ~1500 MapPoints of 2-30 observations over {N_KF} resident TUM-shaped "
            "640x480 @1000 keyframes each, all streams in one call per arm", "reps": reps, **res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_distinctive_frames.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    main(a.reps, a.out)
