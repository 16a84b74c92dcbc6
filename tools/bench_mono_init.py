"""Monocular initialisation's search, SearchForInitialization(mInitialFrame, mCurrentFrame, mvbPrevMatched, mvIniMatches, 100)
(Tracking::MonocularInitialization, src/Tracking.cc:600), for N = 1, 8 and 32 camera streams.  TUM-shaped 640x480 frames at 2000
features (the initialisation extractor's 2 x nFeatures), no lens distortion: per stream s the initial frame is the left image of
synth.stereo_pair(300, s, 0, 640, 480) and the current frame the right one (a horizontal motion of 2-80 px, inside the window of
100); vbPrevMatched = the initial keypoints.  Frames are resident, made by borb_frames_from_extractor in mode 0.
   single: N x borb_search_for_initialization on host copies of the same frames (what a tracker calls today);
   batch:  one borb_search_for_initialization_batch.
Both arms must return equal results before anything is timed.  Host clock around the public Python calls (each ends in a
synchronise) after warm-up: median, 25th and 75th percentile of `--reps`.  Device time per kernel comes from torch.profiler in a run
of its own; the device scratch of each arm is read off its layout.
usage: python tools/bench_mono_init.py [--reps 30] [--out DIR]  -> one JSON line on stdout (and DIR/bench_mono_init.json)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, synth                                 # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit                       # noqa: E402
from tools.bench_loop_closure import spread                                    # noqa: E402
from tools.bench_track_ref import kernel_times                                 # noqa: E402

K_TUM = (517.306408, 516.469215, 318.643040, 255.313989)
SINGLE_KERNELS = ("grid_sort_jobs_kernel", "init_prefix_kernel", "init_replay_kernel")
BATCH_KERNELS = ("init_prefix_kernel", "init_prefix_batch_kernel", "init_replay_kernel", "init_replay_batch_kernel")


def scratch_bytes(n1s, grid=False):
    """Device scratch of one call: per job the prefix table (n1 x 8 entries x 4 B) and the window counts (n1 x 4 B), and with
    `grid` (the single call, whose current frame is a host view) that frame's grid, cell_start (64 x 48 + 1 entries) and cell_idx
    (8192 entries + 16 B); each 256-byte aligned."""
    al = lambda b: (b + 255) // 256 * 256
    g = al(4 * (64 * 48 + 1)) + al(4 * 8192 + 16) if grid else 0
    return int(sum(al(32 * n) + al(4 * n) + g for n in n1s))


def main(reps, out_dir, ns=(1, 8, 32)):
    n_max = max(ns)
    X = ORBextractor(2000)
    pairs = [synth.stereo_pair(300, s, 0, 640, 480) for s in range(n_max)]
    outs = X.extract_batch([p[0] for p in pairs] + [p[1] for p in pairs])
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    mt = M.ORBmatcher(0.9, True)
    frames, host = M.frames_from_extractor(mt, X, list(range(2 * n_max)), [len(o[0]) for o in outs], K_TUM, mode=0)
    b = tuple(float(x) for x in host["bounds"])
    views = [M.FrameView(host["keys_un"][i], outs[i][1], sf, b) for i in range(2 * n_max)]
    prevs = [np.stack([k["x"], k["y"]], 1).astype(np.float32) for k in host["keys_un"][:n_max]]
    res = {}
    for n in ns:
        def single():
            return [mt.SearchForInitialization(views[s], views[n_max + s], prevs[s], 100) for s in range(n)]

        def batch():
            return mt.SearchForInitializationBatch(frames[:n], frames[n_max:n_max + n], prevs[:n], 100)

        a, c = single(), batch()
        assert all(x[0] == y[0] and np.array_equal(x[1], y[1]) and np.array_equal(x[2], y[2]) for x, y in zip(a, c))
        n1s = [len(host["keys_un"][s]) for s in range(n)]
        res[str(n)] = {"single_calls": spread(single, reps), "batch": spread(batch, reps), "matches": int(sum(x[0] for x in c)),
                       "batch_scratch_bytes": scratch_bytes(n1s),
                       "single_call_scratch_bytes": max(scratch_bytes([p], grid=True) for p in n1s)}
    try:
        res["kernels_us"] = {
            "single_1": kernel_times(lambda: mt.SearchForInitialization(views[0], views[n_max], prevs[0], 100), SINGLE_KERNELS),
            "batch_1": kernel_times(lambda: mt.SearchForInitializationBatch(frames[:1], frames[n_max:n_max + 1], prevs[:1], 100),
                                    BATCH_KERNELS),
            "batch_32": kernel_times(lambda: mt.SearchForInitializationBatch(frames[:n_max], frames[n_max:], prevs, 100), BATCH_KERNELS)}
    except Exception as e:                                               # the profiler is optional for the host-clock table
        res["kernel_us_error"] = repr(e)
    line = {"config": "SearchForInitialization, window 100, nnratio 0.9, orientation check on; TUM-shaped 640x480 @2000 features, "
                      "initial = left, current = right image of synth.stereo_pair(300, s, 0, 640, 480); N x "
                      "borb_search_for_initialization on host views vs one borb_search_for_initialization_batch on resident frames; "
                      "host time per call sequence",
            "features": [len(o[0]) for o in outs[:3]], "gpu": gpu_name_and_power_limit(), "workloads": res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_mono_init.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    main(a.reps, a.out)
