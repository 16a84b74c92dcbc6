"""Secondary measurements for BASELINE.json configs[2] and configs[4] (parity-test configurations, not bench lines):
   config 2: RGB-D TUM-shaped 640x480 extract + SearchByProjection against 300 local MapPoints — us per call;
   config 4: EuRoC-shaped 752x480 @1200 features, loop-closure / relocalisation against a 2000-keyframe database:
             one KeyFrameDatabase query (shared words + L1 score for all keyframes) and SearchByBoW against all
             2000 resident keyframes;
   tracking tick of N streams: the motion-model search (SearchByProjection(CurrentFrame, LastFrame)) plus the local-map search
             (Tracking::SearchLocalPoints) of N TUM-shaped 640x480 @1000 streams with a few hundred to ~2000 local MapPoints each,
             as N single calls of each search and as one batched call of each, for N in 1, 8, 32.
All times are wall-clock around the public Python call (host buffers in, results out), median of `--reps`, taken right
after a burst of extraction work so that the SM clocks are where a running tracker keeps them.
usage: python tools/bench_configs.py [--kfs 2000] [--reps 20]  -> one JSON line per config on stdout."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, sharding, synth                      # noqa: E402
from orb_slam2_b200.extractor import ORBextractor                              # noqa: E402


_WARM = {}


def warm_clocks(seconds=0.4):
    """A lightly loaded GPU idles at low SM clocks, which would inflate every us-scale number below; in the tracker the
    extractor keeps the clocks up.  Run extraction work for a moment right before a timed block."""
    if "x" not in _WARM:
        _WARM["x"] = ORBextractor(2000)
        _WARM["imgs"] = [synth.mono_frame(9, 0, i, *synth.KITTI) for i in range(16)]
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        _WARM["x"].extract_batch(_WARM["imgs"])


def med(f, reps):
    f()
    warm_clocks()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); f(); t.append(time.perf_counter() - t0)
    return float(np.median(t))


def config2(reps):
    X = ORBextractor(1000)
    img0, img1 = synth.mono_frame(1, 0, 0, 640, 480), synth.mono_frame(1, 0, 1, 640, 480)
    k0, d0 = X(img0)
    k1, d1 = X(img0)          # the "current" frame sees the same scene; 300 of its features stand in for local MapPoints
    rng = np.random.default_rng(0)
    sel = rng.choice(len(k0), 300, replace=False)
    F = M.FrameView(k1, d1, X.GetScaleFactors(), (0.0, 0.0, 640.0, 480.0))
    mps = M.MapPointsView(k0["x"][sel] + rng.normal(0, 1.5, 300).astype(np.float32), k0["y"][sel] + rng.normal(0, 1.5, 300).astype(np.float32),
                          np.zeros(300, np.float32), k0["octave"][sel].astype(np.int32), np.full(300, 0.9, np.float32), d0[sel])
    mt = M.ORBmatcher(0.8, True)
    n, _ = mt.SearchByProjection(F, mps, 3.0)
    t_match = med(lambda: mt.SearchByProjection(F, mps, 3.0), reps)
    t_ext = med(lambda: X(img1), reps)
    # motion-model tracking: every feature of the last frame carries a MapPoint (SearchByProjection(CurrentFrame, LastFrame))
    K = (525.0, 525.0, 319.5, 239.5)
    z = rng.uniform(2.0, 20.0, len(k0)).astype(np.float32)
    Pw = np.stack([(k0["x"] - K[2]) * z / K[0], (k0["y"] - K[3]) * z / K[1], z], 1).astype(np.float32)
    Last = M.LastFrameView(mvKeysUn=k0, world_pos=Pw, descriptors=d0)
    Tcw = np.eye(4, dtype=np.float32)[:3]
    nl, _ = mt.SearchByProjectionLast(F, Last, Tcw, K, 40.0, 7.0)
    t_last = med(lambda: mt.SearchByProjectionLast(F, Last, Tcw, K, 40.0, 7.0), reps)
    return {"config": "configs[2]: TUM-shaped 640x480 @1000, extract + SearchByProjection vs 300 local MapPoints", "matches": int(n),
            "extract_ms": t_ext * 1e3, "search_by_projection_us": t_match * 1e6, "frames_per_s_serial": 1.0 / (t_ext + t_match),
            "search_by_projection_last_frame_us": t_last * 1e6, "last_frame_queries": int(len(k0)), "last_frame_matches": int(nl)}


def config4(n_kf, reps):
    voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
    X = ORBextractor(1200)
    rng = np.random.default_rng(1)
    n_src = 40
    outs = X.extract_batch([synth.mono_frame(50 + i, 0, 0, 752, 480) for i in range(n_src)])
    mt = M.ORBmatcher(0.75, True)
    db = M.KeyFrameDatabase(mt)
    t_add = 0.0
    n_feat = 0
    for j in range(n_kf):
        k, d = outs[j % n_src]
        if j >= n_src:                                         # derive further keyframes by flipping ~4 % of the descriptor bits
            flip = (rng.random((len(d), 32, 8)) < 0.04)
            d = d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)
        bow, fv = voc.transform(d, 4)
        kf = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=np.ones(len(k), np.uint8))
        t0 = time.perf_counter(); db.add(kf, bow); t_add += time.perf_counter() - t0
        n_feat += len(k)
    qk, qd = outs[3]
    flip = (rng.random((len(qd), 32, 8)) < 0.02)
    qd = qd ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(qd), 32)
    qbow, qfv = voc.transform(qd, 4)
    F = M.KeyFrameView(mvKeysUn=qk, mDescriptors=qd, mFeatVec=qfv)
    t_bowvec = med(lambda: voc.ComputeBoW(qd, 4), reps)
    cw, sc, fw = db.query(qbow)
    t_query = med(lambda: db.query(qbow), reps)
    slots = np.arange(n_kf, dtype=np.int32)
    nm, off, pairs = db.SearchByBoWPairs(None, F)
    cap = int(nm.sum()) + 1024
    t_bow = med(lambda: db.SearchByBoWPairs(None, F, pairs_cap=cap), reps)
    t_bow_counts = med(lambda: db.SearchByBoWPairs(None, F, want_pairs=False), reps)
    top = np.argsort(-sc)[:20].astype(np.int32)
    t_bow20 = med(lambda: db.SearchByBoW(top, F), reps)
    db_bytes = db.size()[1]
    return {"config": f"configs[4]: EuRoC-shaped 752x480 @1200, {n_kf}-keyframe resident database (vocabulary k=10 L=6, random tree)",
            "keyframes": n_kf, "features_per_keyframe": n_feat / n_kf, "db_device_MB": db_bytes / 1e6, "add_ms_per_keyframe": t_add / n_kf * 1e3,
            "compute_bow_us": t_bowvec * 1e6, "kfdb_query_us": t_query * 1e6, "best_common_words": int(cw.max()), "best_score": float(sc.max()),
            "search_by_bow_all_ms": t_bow * 1e3, "search_by_bow_all_counts_only_ms": t_bow_counts * 1e3, "search_by_bow_all_pairs": int(nm.sum()),
            "search_by_bow_all_matches_max": int(nm.max()),
            "search_by_bow_all_descriptor_GBps": n_feat * 32 / t_bow / 1e9,
            "search_by_bow_top20_us": t_bow20 * 1e6}


def gpu_name_and_power_limit():
    """Read-only query of the card the numbers were measured on."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def track_streams(reps, ns=(1, 8, 32)):
    X = ORBextractor(1000)
    n_max = max(ns)
    outs = X.extract_batch([synth.mono_frame(200 + i, 0, 0, 640, 480) for i in range(n_max)])
    sf = np.asarray(X.GetScaleFactors(), np.float32)
    K, bf = (525.0, 525.0, 319.5, 239.5), 40.0
    T = np.eye(4, dtype=np.float32)[:3]
    Ow = np.zeros(3, np.float32)
    mt = M.ORBmatcher(0.8, True)
    rng = np.random.default_rng(2)
    frames, lasts, points = [], [], []
    for i, (k, d) in enumerate(outs):
        n = len(k)
        z = rng.uniform(2.0, 20.0, n).astype(np.float32)
        Pw = np.stack([(k["x"] - K[2]) * z / K[0], (k["y"] - K[3]) * z / K[1], z], 1).astype(np.float32)
        frames.append(M.FrameView(k, d, sf, (0.0, 0.0, 640.0, 480.0)).make_resident(mt))
        lasts.append(M.LastFrameView(mvKeysUn=k, world_pos=Pw, descriptors=d))
        # local map: the frame's own points (in view) and, for the larger maps, points beside the view that isInFrustum rejects
        n_lp = 300 + (i * 389) % 1700
        n_in = min(n_lp, n)
        extra = n_lp - n_in
        side = np.stack([rng.uniform(30, 60, extra), rng.uniform(-5, 5, extra), rng.uniform(2, 20, extra)], 1).astype(np.float32)
        Pl = np.concatenate([Pw[:n_in], side]).astype(np.float32)
        dist = np.linalg.norm(Pl.astype(np.float64), axis=1)
        octv = np.concatenate([k["octave"][:n_in], np.zeros(extra, np.int32)])
        maxd = (dist * sf[octv] * 0.95).astype(np.float32)
        desc = np.concatenate([d[:n_in], d[:extra] if extra <= n else np.resize(d, (extra, 32))]).astype(np.uint8)
        points.append(M.WorldPointsView(world_pos=Pl, descriptors=desc, max_distance=maxd, min_distance=(maxd / sf[-1]).astype(np.float32),
                                        normal=(Pl / dist[:, None]).astype(np.float32)))
    res = {}
    for n in ns:
        F, L, P = frames[:n], lasts[:n], points[:n]

        def single():
            m = 0
            for j in range(n):
                m += mt.SearchByProjectionLast(F[j], L[j], T, K, bf, 15.0)[0]
                m += mt.SearchLocalPoints(F[j], P[j], T, Ow, K, bf, 1.0)["nmatches"]
            return m

        def batched():
            m = sum(r[0] for r in mt.SearchByProjectionLastBatch(F, L, [T] * n, K, bf, 15.0))
            return m + sum(r["nmatches"] for r in mt.SearchLocalPointsBatch(F, P, [(T, Ow)] * n, K, bf, 1.0))

        assert single() == batched()
        t_single, t_batch = med(single, reps), med(batched, reps)
        res[str(n)] = {"single_calls_us": t_single * 1e6, "batched_us": t_batch * 1e6, "matches": int(batched()),
                       "local_points": int(sum(len(p.world_pos) for p in P))}
    return {"config": "tracking tick of N TUM-shaped 640x480 @1000 streams: SearchByProjection(CurrentFrame, LastFrame) + "
                      "SearchLocalPoints (300-1999 local MapPoints per stream), per-tick host time of N single calls of each search vs "
                      "one batched call of each", "gpu": gpu_name_and_power_limit(), "streams": res}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--kfs", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    print(json.dumps(config2(a.reps)), flush=True)
    print(json.dumps(config4(a.kfs, a.reps)), flush=True)
    print(json.dumps(track_streams(a.reps)), flush=True)
