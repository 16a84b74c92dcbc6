"""The matcher part of one LocalMapping step (LocalMapping::CreateNewMapPoints' SearchForTriangulation against every neighbour and
SearchInNeighbors' Fuse calls) for N camera streams, N in 1, 8, 32, TUM-shaped 640x480 @1000, vocabulary k=10 L=6 (random tree),
levelsup 4, ~60 % of the features with MapPoints; the neighbours re-observe the keyframe (keypoints moved by ~0.5 px,
~3 % of the descriptor bits flipped).  Two workloads:
   stereo: 10 neighbours (the reference's nn for stereo / RGB-D), stereo coordinates on half the features;
   mono:   20 neighbours, no stereo coordinates.
Each stream fuses its keyframe's MapPoints into 25 target keyframes, then the targets' points into its keyframe.
Compared per tick:
   single:  N x (nn borb_search_for_triangulation on host views + 25 borb_fuse + 1 borb_fuse on resident keyframes);
   batched: one borb_search_for_triangulation_batch (resident keyframes with BoW: only has_mp and mvLevelSigma2 cross PCIe) +
            26 borb_fuse_batch calls of N jobs (one per target index, then the final Fuse of every stream).
Both arms must return equal results before anything is timed.  Host clock around the public Python calls (each ends in a
synchronise), median of `--reps` after warm-up, taken right after a burst of extraction work (tools/bench_configs.warm_clocks).
A second run with torch.profiler gives the device time of the triangulation, projection and fuse kernels per batched tick.
usage: python tools/bench_localmap_batch.py [--reps 20] [--out DIR]  -> one JSON line on stdout (and DIR/bench_localmap_batch.json)."""
import argparse
import dataclasses
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
TARGETS = 25
K = (517.3, 516.5, 318.6, 255.3)
BF = 40.0
KERNELS = ("triangulation_kernel", "project_points_batch_kernel", "fuse_batch_kernel")
F12 = np.array([[0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]], np.float32)          # a rectified pair: same row
EPIPOLE = (300.0, 240.0)


def world_points(k, d, sf, rng, n_pts):
    """Points seen by a keyframe at the identity pose: its keypoints back-projected at random depths, with the MapPoint fields
    Fuse reads.  The first n_pts keypoints (the ones that carry a MapPoint)."""
    k, d = k[:n_pts], d[:n_pts]
    z = rng.uniform(2.0, 20.0, len(k))
    P = np.stack([(k["x"] - K[2]) * z / K[0], (k["y"] - K[3]) * z / K[1], z], 1)
    dist = np.linalg.norm(P, axis=1)
    maxd = dist * sf[np.clip(k["octave"], 0, len(sf) - 1)]
    return M.WorldPointsView(world_pos=P.astype(np.float32), descriptors=d, max_distance=maxd.astype(np.float32),
                             min_distance=(maxd / sf[-1]).astype(np.float32), normal=(P / dist[:, None]).astype(np.float32),
                             valid=(rng.random(len(k)) < 0.95).astype(np.uint8))


def main(reps, out_dir, ns=(1, 8, 32)):
    n_max = max(ns)
    X = ORBextractor(1000)
    outs = X.extract_batch([synth.mono_frame(70 + i, 0, 0, 640, 480) for i in range(n_max)])
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    inv_sigma2 = (np.float32(1.0) / (sf * sf)).astype(np.float32)
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    mt = M.ORBmatcher(0.6, False)                                     # CreateNewMapPoints: ORBmatcher matcher(0.6,false)
    rng = np.random.default_rng(1)
    identity = np.eye(4, dtype=np.float32)[:3]
    res = {}
    for name, nn in (("stereo", 10), ("mono", 20)):
        # stream s: keyframe = source frame s; its neighbours re-observe it (keypoints moved by ~0.5 px, ~3 % of the descriptor
        # bits flipped), so that the searches find what a real neighbourhood gives them.  Host views and resident frames of each.
        host, resident = {}, {}

        def add(key, k, d):
            ur = np.where(rng.random(len(k)) < 0.5, k["x"] - rng.uniform(5, 60, len(k)), -1.0).astype(np.float32) if name == "stereo" else None
            hm = (rng.random(len(k)) < 0.6).astype(np.uint8)
            host[key] = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=voc.ComputeBoW(d, LEVELSUP)[1], has_mp=hm, mvuRight=ur,
                                       mvScaleFactors=sf, mvLevelSigma2=sf * sf)
            resident[key] = dataclasses.replace(M.FrameView(k, d, sf, (0.0, 0.0, 640.0, 480.0), mvuRight=ur, mvInvLevelSigma2=inv_sigma2)
                                                .make_resident(mt), has_mp=hm)

        for s in range(n_max):
            k, d = outs[s]
            add((s, -1), k, d)
            for t in range(nn):
                kt = k.copy()
                kt["x"] = np.clip(kt["x"] + rng.normal(0, 0.5, len(k)), 0, 639).astype(np.float32)
                flip = np.packbits(rng.random((len(d), 32, 8)) < 0.03, axis=2, bitorder="little").reshape(len(d), 32)
                add((s, t), kt, d ^ flip)
        mt.ComputeBoWBatch(voc, list(resident.values()), LEVELSUP, want_host=False)
        nbr = lambda s: [(s, t) for t in range(nn)]
        targets = lambda s: [(s, t % nn) for t in range(TARGETS)]
        pts = {s: world_points(outs[s][0], outs[s][1], sf, np.random.default_rng(200 + s), int(0.6 * len(outs[s][0]))) for s in range(n_max)}
        cand = {s: world_points(np.concatenate([host[t].mvKeysUn for t in nbr(s)[:3]]), np.concatenate([host[t].mDescriptors for t in nbr(s)[:3]]),
                                sf, np.random.default_rng(300 + s), 2400) for s in range(n_max)}
        pose = (identity, np.zeros(3, np.float32))
        res[name] = {}
        for n in ns:
            streams = list(range(n))

            def single():
                tri, fz = [], []
                for s in streams:
                    tri.append([mt.SearchForTriangulation(host[(s, -1)], host[t], F12, EPIPOLE) for t in nbr(s)])
                    fz.append([mt.Fuse(resident[t], pts[s], pose[0], pose[1], K, BF, 3.0) for t in targets(s)] +
                              [mt.Fuse(resident[(s, -1)], cand[s], pose[0], pose[1], K, BF, 3.0)])
                return tri, fz

            def batched():
                kf1s = [resident[(s, -1)] for s in streams for _ in range(nn)]
                kf2s = [resident[t] for s in streams for t in nbr(s)]
                flat = mt.SearchForTriangulationBatch(kf1s, kf2s, [F12] * len(kf1s), [EPIPOLE] * len(kf1s))
                tri = [flat[i * nn:(i + 1) * nn] for i in range(n)]
                by_target = [mt.FuseBatch([resident[targets(s)[t]] for s in streams], [pts[s] for s in streams], [pose] * n, K, BF, 3.0)
                             for t in range(TARGETS)]
                last = mt.FuseBatch([resident[(s, -1)] for s in streams], [cand[s] for s in streams], [pose] * n, K, BF, 3.0)
                return tri, [[by_target[t][i] for t in range(TARGETS)] + [last[i]] for i in range(n)]

            (ta, fa), (tb, fb) = single(), batched()
            assert all(np.array_equal(x, y) for a, b in zip(ta, tb) for x, y in zip(a, b))
            assert all(x[0] == y[0] and np.array_equal(x[1], y[1]) for a, b in zip(fa, fb) for x, y in zip(a, b))
            t_single, t_batch = med(single, reps), med(batched, reps)
            res[name][str(n)] = {"single_calls_us": t_single * 1e6, "batched_us": t_batch * 1e6, "triangulation_jobs": n * nn,
                                 "fuse_jobs": n * (TARGETS + 1), "pairs": int(sum(len(p) for a in tb for p in a)),
                                 "fused": int(sum(x[0] for a in fb for x in a))}
            try:
                res[name][str(n)]["kernel_us"] = kernel_times(batched, KERNELS)
            except Exception as e:                                       # the profiler is optional for the host-clock table
                res[name][str(n)]["kernel_us_error"] = repr(e)
    line = {"config": "LocalMapping matcher step of N TUM-shaped 640x480 @1000 streams: N x (nn borb_search_for_triangulation on host "
                      "views + 25 borb_fuse + 1 borb_fuse) vs one borb_search_for_triangulation_batch + 26 borb_fuse_batch, per-tick "
                      "host time; stereo: nn = 10, mono: nn = 20",
            "gpu": gpu_name_and_power_limit(), "workloads": res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_localmap_batch.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    main(a.reps, a.out)
