"""The reference-keyframe step of a tracking tick (Tracking::TrackReferenceKeyFrame: Frame::ComputeBoW + SearchByBoW(KeyFrame*,
Frame&)) for N TUM-shaped 640x480 @1000 camera streams on resident frames, N in 1, 8, 32.  Each stream's reference keyframe is a
second resident frame of the same scene (the right view of a synthetic stereo pair) with MapPoints on ~70 % of its features;
vocabulary k=10 L=6 (random tree), levelsup 4.  Compared per tick:
   single:  N x (borb_compute_bow + borb_search_by_bow on host views): descriptors and both views cross PCIe, 2 synchronisations each;
   batched: one borb_frames_compute_bow + one borb_search_by_bow_batch (keyframes through kf_frame: only has_mp crosses PCIe).
Host clock around the public Python calls (each ends in a synchronise), median of `--reps` after warm-up, taken right after a burst
of extraction work (tools/bench_configs.warm_clocks).  A second run with torch.profiler gives the device time of the two device-BoW
kernels (bow_transform_batch_kernel, bow_build_kernel) per batched call.
usage: python tools/bench_track_ref.py [--reps 20] [--out DIR]  -> one JSON line on stdout (and DIR/bench_track_ref.json)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, sharding, synth                      # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402
from tools.bench_configs import gpu_name_and_power_limit, med                  # noqa: E402

LEVELSUP = 4


def kernel_times(fn, names, iters=20):
    """Mean device time per call of the named kernels, from torch.profiler's CUDA activity (a run of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                out[n] += ev.device_time_total / iters                   # us per call
    return out


def main(reps, out_dir, ns=(1, 8, 32)):
    n_max = max(ns)
    X = ORBextractor(1000)
    pairs = [synth.stereo_pair(300 + i, 0, 0, 640, 480) for i in range(n_max)]
    cur = X.extract_batch([p[0] for p in pairs])
    ref = X.extract_batch([p[1] for p in pairs])
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    bounds = (0.0, 0.0, 640.0, 480.0)
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    mt = M.ORBmatcher(0.7, True)
    rng = np.random.default_rng(4)
    F = [M.FrameView(k, d, sf, bounds).make_resident(mt) for k, d in cur]
    has_mp = [(rng.random(len(k)) < 0.7).astype(np.uint8) for k, _ in ref]
    KF = [M.FrameView(k, d, sf, bounds, has_mp=hm).make_resident(mt) for (k, d), hm in zip(ref, has_mp)]
    mt.ComputeBoWBatch(voc, KF, LEVELSUP, want_host=False)              # the keyframes got their BoW when they were made
    KF_host = [M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=voc.ComputeBoW(d, LEVELSUP)[1], has_mp=hm) for (k, d), hm in zip(ref, has_mp)]
    res = {}
    for n in ns:
        def single():
            out = []
            for j in range(n):
                k, d = cur[j]
                _, fv = voc.ComputeBoW(d, LEVELSUP)
                out.append(mt.SearchByBoW(KF_host[j], M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv)))
            return out

        def batched():
            mt.ComputeBoWBatch(voc, F[:n], LEVELSUP, want_host=False)
            return mt.SearchByBoWBatch(KF[:n], F[:n])

        a, b = single(), batched()
        assert all(x[0] == y[0] and np.array_equal(x[1], y[1]) for x, y in zip(a, b))
        t_single, t_batch = med(single, reps), med(batched, reps)
        res[str(n)] = {"single_calls_us": t_single * 1e6, "batched_us": t_batch * 1e6, "matches": int(sum(x[0] for x in b)),
                       "features": int(sum(len(c[0]) for c in cur[:n]))}
    try:
        names = ("bow_transform_batch_kernel", "bow_build_kernel")
        for n in ns:
            res[str(n)]["kernel_us"] = kernel_times(lambda: mt.ComputeBoWBatch(voc, F[:n], LEVELSUP, want_host=False), names)
    except Exception as e:                                               # the profiler is optional for the host-clock table
        res["kernel_us_error"] = repr(e)
    line = {"config": "reference-keyframe step of N TUM-shaped 640x480 @1000 streams on resident frames: N x (borb_compute_bow + "
                      "borb_search_by_bow on host views) vs borb_frames_compute_bow + borb_search_by_bow_batch, per-tick host time",
            "gpu": gpu_name_and_power_limit(), "streams": res}
    print(json.dumps(line), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_track_ref.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    main(a.reps, a.out)
