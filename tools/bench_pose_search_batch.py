"""The pose searches that follow relocalisation's PnP and loop closure's Sim3Solver, for N = 1, 8 and 32 camera streams at 2000
features, no lens distortion, frames made resident by borb_frames_from_extractor (mode 0):
   reloc: SearchByProjection(CurrentFrame, pKF, sFound, 10, 100) (src/Tracking.cc:1452), TUM-shaped 640x480; per stream s the
          current frame is the left image of synth.stereo_pair(300, s, 0, 640, 480) and the keyframe's MapPoints the right image's
          features placed in the world (tests/match_fixtures.world_points_case);
          N x borb_search_by_projection_kf on host views vs one borb_search_by_projection_kf_batch;
   sim3:  SearchBySim3(mpCurrentKF, pKF, vpMatches12, s, R, t, 7.5) (src/LoopClosing.cc:323), EuRoC-shaped 752x480 keyframes: the left
          and right image of synth.stereo_pair(400, s, 0, 752, 480), one MapPoint per feature (match_fixtures.sim3_case);
          N x borb_search_by_sim3 vs one borb_search_by_sim3_batch;
   sim3proj: SearchByProjection(mpCurrentKF, mScw, mvpLoopMapPoints, mvpCurrentMatchedPoints, 10) (src/LoopClosing.cc:375) on the
          same EuRoC-shaped keyframes; N x borb_search_by_projection_sim3 vs one borb_search_by_projection_sim3_batch.
Both arms must return equal results before anything is timed.  Host clock around the public Python calls (each ends in a
synchronise) after warm-up: median, 25th and 75th percentile of `--reps`.  Device time per kernel comes from torch.profiler in a run
of its own.
With --before-lib PATH (a libborb.so built from an earlier commit) one single SearchBySim3 on host views is also timed with that
library and with this one, alternating the two in the same process, after checking that they return the same result.
usage: python tools/bench_pose_search_batch.py [--reps 30] [--before-lib PATH] [--out DIR]
       -> one JSON line on stdout (and DIR/bench_pose_search_batch.json)."""
import argparse
import ctypes as C
import dataclasses
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import _lib, matcher as M, synth                          # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tests import match_fixtures as mf                                         # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit, warm_clocks          # noqa: E402
from tools.bench_loop_closure import spread                                    # noqa: E402
from tools.bench_track_ref import kernel_times                                 # noqa: E402

K_TUM = (517.306408, 516.469215, 318.643040, 255.313989)
K_EUROC = (458.654, 457.296, 367.215, 248.375)
PROJ_KERNELS = ("project_points_kernel", "project_points_batch_kernel", "proj_candidates_kernel", "proj_candidates_batch_kernel",
                "proj_resolve_kernel", "proj_resolve_batch_kernel")
SIM3_KERNELS = ("grid_sort_jobs_kernel", "project_points_batch_kernel", "fuse_batch_kernel", "sim3_agree_batch_kernel")


def same(a, b):
    return all(x[0] == y[0] and np.array_equal(x[1], y[1]) for x, y in zip(a, b)) and len(a) == len(b)


def streams(n_max, shape, seed, K):
    """n_max stereo pairs extracted at 2000 features: host views and resident frames of the left (0..n-1) and right (n..2n-1) images."""
    X = ORBextractor(2000)
    pairs = [synth.stereo_pair(seed, s, 0, *shape) for s in range(n_max)]
    outs = X.extract_batch([p[0] for p in pairs] + [p[1] for p in pairs])
    mt = M.ORBmatcher(0.9, True)
    frames, host = M.frames_from_extractor(mt, X, list(range(2 * n_max)), [len(o[0]) for o in outs], K, mode=0)
    b = tuple(float(x) for x in host["bounds"])
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    vs = [dict(w=shape[0], h=shape[1], kl=host["keys_un"][s], dl=outs[s][1], kr=host["keys_un"][n_max + s], dr=outs[n_max + s][1],
               disp=pairs[s][2], scale=sf) for s in range(n_max)]
    return mt, frames, vs, b, [len(o[0]) for o in outs]


class _BeforeMatcher(M.ORBmatcher):
    """An ORBmatcher on another build of libborb.so (same C ABI for the calls used here)."""

    def __init__(self, path, nnratio, checkOri):
        lib = C.CDLL(os.path.abspath(path))
        for name, (res, args) in _lib._SIGNATURES.items():
            if hasattr(lib, name):
                getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
        self._lib = lib
        self.mfNNratio, self.mbCheckOrientation = float(np.float32(nnratio)), bool(checkOri)
        h = C.c_void_p()
        assert lib.borb_matcher_create(0, C.byref(h)) == 0
        self._h = h


def alternate(fa, fb, reps):
    """Median / quartiles of fa and fb timed in alternation (a, b, a, b, ...) after one warm-up call each."""
    fa(); fb()
    warm_clocks()
    ta, tb = [], []
    for _ in range(reps):
        t0 = time.perf_counter(); fa(); ta.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); fb(); tb.append(time.perf_counter() - t0)
    q = lambda t: dict(zip(("p25_us", "median_us", "p75_us"), (float(x) for x in np.percentile(np.asarray(t) * 1e6, [25, 50, 75]))))
    return q(ta), q(tb)


def main(reps, out_dir, before_lib, ns=(1, 8, 32)):
    n_max = max(ns)
    res = {}
    # ---- relocalisation: TUM-shaped current frames
    mt, frames, vs, b, feats_tum = streams(n_max, (640, 480), 300, K_TUM)
    kf = []
    for s in range(n_max):
        Cur, P, Tcw, Ow, K = mf.world_points_case(vs[s], 500 + s)
        Cur = dataclasses.replace(Cur, bounds=b)
        kf.append((Cur, dataclasses.replace(Cur, resident=frames[s].resident), P, Tcw, Ow, K))
    for n in ns:
        def single():
            return [mt.SearchByProjectionKF(j[0], j[2], j[3], j[4], j[5], 10.0, 100) for j in kf[:n]]

        def batch():
            return mt.SearchByProjectionKFBatch([j[1] for j in kf[:n]], [j[2] for j in kf[:n]], [(j[3], j[4]) for j in kf[:n]], kf[0][5],
                                                10.0, 100)
        a, c = single(), batch()
        assert same(a, c)
        res[f"reloc_{n}"] = {"single_calls": spread(single, reps), "batch": spread(batch, reps), "matches": int(sum(x[0] for x in c))}
    # ---- loop closure: EuRoC-shaped keyframes
    mt2, frames2, vs2, b2, feats_euroc = streams(n_max, (752, 480), 400, K_EUROC)
    loop = []
    for s in range(n_max):
        KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = mf.sim3_case(vs2[s], 600 + s)
        KF1, KF2 = dataclasses.replace(KF1, bounds=b2), dataclasses.replace(KF2, bounds=b2)
        C1, Pq, Tq, Oq, _ = mf.world_points_case(vs2[s], 700 + s)      # mvpLoopMapPoints: the candidate's points seen from KF1
        loop.append(((KF1, KF2, P1, P2, T1w, T2w, S12, S21, K), frames2[s], frames2[n_max + s],
                     (dataclasses.replace(C1, bounds=b2), dataclasses.replace(C1, bounds=b2, resident=frames2[s].resident), Pq, Tq, Oq)))
    for n in ns:
        L = loop[:n]

        def single3():
            return [mt2.SearchBySim3(*j[0], 7.5) for j in L]

        def batch3():
            return mt2.SearchBySim3Batch([j[1] for j in L], [j[2] for j in L], [j[0][2] for j in L], [j[0][3] for j in L],
                                         [(j[0][4], j[0][5]) for j in L], [(j[0][6], j[0][7]) for j in L], L[0][0][8], 7.5)

        def singlep():
            return [mt2.SearchByProjectionSim3(j[3][0], j[3][2], j[3][3], j[3][4], L[0][0][8], 10) for j in L]

        def batchp():
            return mt2.SearchByProjectionSim3Batch([j[3][1] for j in L], [j[3][2] for j in L], [(j[3][3], j[3][4]) for j in L], L[0][0][8], 10)
        a, c = single3(), batch3()
        assert same(a, c)
        ap, cp = singlep(), batchp()
        assert same(ap, cp)
        res[f"sim3_{n}"] = {"single_calls": spread(single3, reps), "batch": spread(batch3, reps), "matches": int(sum(x[0] for x in c))}
        res[f"sim3proj_{n}"] = {"single_calls": spread(singlep, reps), "batch": spread(batchp, reps), "matches": int(sum(x[0] for x in cp))}
    if before_lib:
        old = _BeforeMatcher(before_lib, 0.75, True)
        one = loop[0][0]
        assert same([old.SearchBySim3(*one, 7.5)], [mt2.SearchBySim3(*one, 7.5)])
        tb, ta = alternate(lambda: old.SearchBySim3(*one, 7.5), lambda: mt2.SearchBySim3(*one, 7.5), reps)
        res["sim3_single_before_after"] = {"before": tb, "after": ta}
        old.close()
    try:
        res["kernels_us"] = {
            "reloc_single_1": kernel_times(lambda: mt.SearchByProjectionKF(kf[0][0], kf[0][2], kf[0][3], kf[0][4], kf[0][5], 10.0, 100),
                                           PROJ_KERNELS),
            "reloc_batch_32": kernel_times(lambda: mt.SearchByProjectionKFBatch([j[1] for j in kf], [j[2] for j in kf],
                                                                                [(j[3], j[4]) for j in kf], kf[0][5], 10.0, 100), PROJ_KERNELS),
            "sim3_single_1": kernel_times(lambda: mt2.SearchBySim3(*loop[0][0], 7.5), SIM3_KERNELS),
            "sim3_batch_32": kernel_times(lambda: mt2.SearchBySim3Batch([j[1] for j in loop], [j[2] for j in loop], [j[0][2] for j in loop],
                                                                        [j[0][3] for j in loop], [(j[0][4], j[0][5]) for j in loop],
                                                                        [(j[0][6], j[0][7]) for j in loop], loop[0][0][8], 7.5), SIM3_KERNELS),
            "sim3proj_batch_32": kernel_times(lambda: mt2.SearchByProjectionSim3Batch([j[3][1] for j in loop], [j[3][2] for j in loop],
                                                                                      [(j[3][3], j[3][4]) for j in loop], loop[0][0][8], 10),
                                              PROJ_KERNELS)}
    except Exception as e:                                               # the profiler is optional for the host-clock table
        res["kernel_us_error"] = repr(e)
    line = {"config": "reloc: SearchByProjection(F, pKF, sFound, 10, 100), ORBmatcher(0.9, true), TUM-shaped 640x480 @2000; "
                      "sim3: SearchBySim3(..., 7.5) and sim3proj: SearchByProjection(pKF, Scw, ..., 10), EuRoC-shaped 752x480 @2000; "
                      "N single calls on host views vs one *_batch call on resident frames; host time per call sequence",
            "features_tum": feats_tum[:3], "features_euroc": feats_euroc[:3], "gpu": gpu_name_and_power_limit(), "workloads": res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_pose_search_batch.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--before-lib", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    main(a.reps, a.out, a.before_lib)
