#!/usr/bin/env python
"""bench.py — throughput of the CUDA ORB front-end (H100, sm_90a) on the BASELINE.json configurations; see DESIGN.md §Measurement.

  python bench.py [--config 1|2|4] [--gpus N] [--steps K] [--warmup W] [--impl b200|reference]
  N>1:  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 ... bench.py --gpus N ...

  --config 1 (default)  configs[1]: stereo KITTI-00-shaped 1242x375 @2000: extract L + extract R + ComputeStereoMatches
  --config 2            configs[2]: RGB-D TUM-shaped 640x480 @1000: extract + Frame constructor tail (UndistortKeyPoints,
                        ComputeStereoFromRGBD, AssignFeaturesToGrid) + SearchByProjection vs 300 local MapPoints
  --config 4            configs[4]: EuRoC-shaped 752x480 @1200 query frames against a 2000-keyframe resident database:
                        ComputeBoW + KeyFrameDatabase scoring + SearchByBoW against every keyframe
One "step" = `passes_per_step` passes of the hot path over one batch of synthetic input per GPU; passes_per_step is calibrated
after warm-up so that one step takes >= 55 ms, so the timed region grows with --steps (the default 20 steps take >= 1.1 s).
  value     frames/s, whole job, inputs already resident in HBM (device buffers in, counts out)
  e2e       same metric through the C-ABI call with HOST (pinned) buffers: H2D of the inputs and D2H of the results
            inside the timed region
  roofline  dominant kernel: algorithmic bytes per launch / its mean launch time (CUDA events on the library's stream)
  cpu_baseline  the reference's own sources compiled verbatim (oracle/_ref) timed on this box's host cores on a bounded
            sample of the same workload (rank 0, N=1 only); value = all cores, one_core_value = a single core
--impl reference: that CPU implementation alone, all host threads, same metric/config (no GPU work).
The GPU arm asserts equality with the oracle on a sample of its own outputs before timing (outside the timed region).
--dump-outputs DIR: after the timed steps, the arrays the timed call returned in its last pass (config 1: keypoints, descriptors,
            counts, mvuRight, mvDepth read back from HBM; config 2: SearchByProjection matches; config 4: scores and SearchByBoW
            pairs) go to DIR/<name>.npy as float32 / float64.  Inputs depend on the arguments only, and the calibrated pass count
            is rounded so that the last pass always sees the same input, so two builds can be compared output for output.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SEED = 2024
SHAPES = {1: (1242, 375, 2000, 1441432), 2: (640, 480, 1000, 950532), 4: (752, 480, 1200, 1117367)}   # w, h, nFeatures, sum of level pixels (SURVEY §8)
BF, FX = 386.1448, 718.856                                # Camera.bf, Camera.fx (KITTI00-02.yaml)
TUM1_K = (517.306408, 516.469215, 318.643040, 255.313989)  # Examples/RGB-D/TUM1.yaml
TUM1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)
TUM1_BF, TUM1_DEPTH_FACTOR = 40.0, 1.0 / 5000.0
EUROC_BF, EUROC_FX = 47.90639384423901, 435.2046959714599   # Examples/Stereo/EuRoC.yaml
N_MAPPOINTS = 300
METRICS = {
    1: "stereo frames/sec (ORB extract L+R + ComputeStereoMatches, KITTI-shaped 1242x375 @2000 kpts)",
    2: "RGB-D frames/sec (ORB extract + UndistortKeyPoints + ComputeStereoFromRGBD + SearchByProjection vs 300 local MapPoints, TUM-shaped 640x480 @1000 kpts)",
    4: "loop-closure query frames/sec (ComputeBoW + KeyFrameDatabase scoring + SearchByBoW vs 2000-keyframe DB, EuRoC-shaped 752x480 @1200 kpts)",
}
WORKLOADS = {
    1: "configs[1]: stereo KITTI-00-shaped 1242x375, 2000 feats, extract + ComputeStereoMatches",
    2: "configs[2]: RGB-D TUM-shaped 640x480, extract + SearchByProjection vs 300 local MapPoints",
    4: "configs[4]: EuRoC-shaped 752x480 stereo + SearchByBoW loop-closure Hamming vs 2000-keyframe descriptor DB",
}


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def host_cores() -> int:
    try:
        return len(os.sched_getaffinity(0))
    except AttributeError:
        return os.cpu_count() or 1


def hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (NVIDIA H100 SXM data sheet, HBM3; not measured)"


# ----------------------------------------------------------------------------------------------
# synthetic inputs (deterministic from seed, stream, frame — SURVEY §8d)
# ----------------------------------------------------------------------------------------------
def make_pairs(stream_id: int, n: int, w: int, h: int):
    from orb_slam2_b200 import synth
    L, R = [], []
    for i in range(n):
        l, r, _ = synth.stereo_pair(SEED, stream_id, i, w, h)
        L.append(l); R.append(r)
    return L, R


def make_rgbd(stream_id: int, n: int, w: int, h: int):
    """Gray frames + registered CV_16U depth maps (5000 units per metre, ~15 % sensor holes)."""
    from orb_slam2_b200 import synth
    imgs, depths = [], []
    yy, xx = np.mgrid[0:h, 0:w]
    for i in range(n):
        imgs.append(synth.mono_frame(SEED, stream_id, i, w, h))
        rng = np.random.default_rng([SEED, stream_id, i, 77])
        raw = (5000.0 * (1.6 + 0.9 * np.sin(xx / 90.0 + i) * np.cos(yy / 70.0 - stream_id))).astype(np.uint16)
        raw[rng.random((h, w)) < 0.15] = 0
        depths.append(raw)
    return imgs, depths


def make_mappoints(keys, desc, scale_factors, rng, u_right=None):
    """300 'local MapPoints' for a frame: a random subset of its own features as seen a moment earlier — projection jittered by
    ~1.5 px, predicted level = the feature's octave (what Frame::isInFrustum leaves in mTrackProj* / mnTrackScaleLevel)."""
    n = min(N_MAPPOINTS, len(keys))
    sel = rng.choice(len(keys), n, replace=False)
    px = (keys["x"][sel] + rng.normal(0, 1.5, n)).astype(np.float32)
    py = (keys["y"][sel] + rng.normal(0, 1.5, n)).astype(np.float32)
    # mTrackProjXR = u - mbf/z of the MapPoint: consistent with the feature's own mvuRight where the depth sensor saw it
    pxr = (px - 20.0).astype(np.float32)
    if u_right is not None:
        ur = np.asarray(u_right, np.float32)[sel]
        pxr = np.where(ur >= 0, ur + (px - keys["x"][sel]), pxr).astype(np.float32)
    return dict(px=px, py=py, pxr=pxr, lvl=keys["octave"][sel].astype(np.int32), vc=np.full(n, 0.9, np.float32), desc=np.ascontiguousarray(desc[sel]))


DUMP_LIMIT = 64 << 20


def dump_outputs(out_dir: str, arrays: dict) -> None:
    """Writes each array as out_dir/<name>.npy: float arrays keep float32 / float64, integers become float32 when every value is
    exact in it (|v| < 2^24) and float64 otherwise."""
    os.makedirs(out_dir, exist_ok=True)
    conv = {}
    for name, a in arrays.items():
        a = np.ascontiguousarray(a)
        if a.dtype.kind == "f":
            a = a.astype(np.float64 if a.dtype == np.float64 else np.float32)
        else:
            a = a.astype(np.float32 if a.size == 0 or np.abs(a.astype(np.int64)).max() < (1 << 24) else np.float64)
        conv[name] = a
    total = sum(a.nbytes for a in conv.values())
    assert total <= DUMP_LIMIT, f"--dump-outputs: {total} bytes exceed the {DUMP_LIMIT}-byte limit"
    for name, a in conv.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)
    log(f"dumped {len(conv)} arrays ({total / 1e6:.1f} MB) to {out_dir}")


def keypoint_columns(kps: np.ndarray) -> np.ndarray:
    """borb_keypoint rows -> (n, 6) float32: x, y, size, angle, response, octave."""
    return np.stack([kps[f].astype(np.float32) for f in ("x", "y", "size", "angle", "response", "octave")], axis=1).reshape(-1, 6)


# ----------------------------------------------------------------------------------------------
# CPU reference arms: the reference's own sources compiled verbatim (oracle/_ref); restatements only where noted
# ----------------------------------------------------------------------------------------------
class CpuPool:
    """One independent camera stream per host thread (ctypes releases the GIL inside the oracle calls)."""

    def __init__(self, workers):
        self.workers = workers
        self.threads = len(workers)

    def run(self, items_per_thread: int):
        """Every worker processes items_per_thread items; returns (items/s over all workers, seconds)."""
        def body(t):
            for i in range(items_per_thread):
                self.workers[t](t * items_per_thread + i)
        ths = [threading.Thread(target=body, args=(t,)) for t in range(self.threads)]
        t0 = time.perf_counter()
        for th in ths: th.start()
        for th in ths: th.join()
        dt = time.perf_counter() - t0
        return self.threads * items_per_thread / dt, dt


def cpu_workers(cfg: int, threads: int, data):
    """Returns (kind, description, [worker(i) -> None] * threads, items_scale) where one call of a worker processes
    `items_scale` frames' worth of the config's workload."""
    from oracle import oracle_lib as O
    O.build()
    kind = "reference" if O.have_ref() else "port"
    Ext = O.RefExtractor if kind == "reference" else O.PortExtractor
    w, h, nfeat, _ = SHAPES[cfg]
    if cfg == 1:
        L, R = data
        stereo = O.ref_stereo if (kind == "reference" and O.have_frameref()) else (lambda *a: O.port_stereo(*a)[:2])

        def make():
            EL, ER = Ext(nfeat), Ext(nfeat)

            def run(i):
                j = i % len(L)
                kl, dl = EL(L[j]); kr, dr = ER(R[j])
                stereo(kl, dl, kr, dr, [EL.level(q) for q in range(8)], [ER.level(q) for q in range(8)], EL.scale, EL.inv_scale, BF, FX)
            return run
        desc = ("extract L+R with the reference's ORBextractor.cc + Frame::ComputeStereoMatches of the reference's Frame.cc, both compiled verbatim (oracle/_ref)"
                if kind == "reference" else "restated extractor + stereo (oracle port)")
        return kind, desc, [make() for _ in range(threads)], 1.0
    if cfg == 2:
        imgs, depths_f, mps = data
        from orb_slam2_b200.matcher import FrameView, MapPointsView
        K4 = np.array(TUM1_K, np.float32); D = np.array(TUM1_DIST, np.float32)
        frame_fn = O.ref_rgbd_frame if (kind == "reference" and O.have_frameref()) else O.port_rgbd_frame
        match_fn = O.ref_search_by_projection if (kind == "reference" and O.have_matchref()) else O.port_search_by_projection

        def make():
            E = Ext(nfeat)

            def run(i):
                j = i % len(imgs)
                k, d = E(imgs[j])
                fr = frame_fn(k, K4, D, TUM1_BF, depths_f[j])
                F = FrameView(fr["keys_un"], d, E.scale, tuple(float(x) for x in fr["bounds"]), mvuRight=fr["u_right"])
                m = mps[j]
                match_fn(F, MapPointsView(m["px"], m["py"], m["pxr"], m["lvl"], m["vc"], m["desc"]), 3.0, 0.8)
            return run
        desc = ("ORBextractor.cc + Frame.cc (UndistortKeyPoints / ComputeStereoFromRGBD) + ORBmatcher.cc SearchByProjection, all compiled verbatim (oracle/_ref)"
                if kind == "reference" else "restated extractor / frame / matcher (oracle port)")
        return kind, desc, [make() for _ in range(threads)], 1.0
    # cfg == 4: one item = one query frame against a SAMPLE of the database (the sweep is linear in the keyframes)
    voc, kfs, kf_bows, queries, sample, n_kf = data
    per = [np.arange(t, len(kfs), max(1, len(kfs) // sample))[:sample] for t in range(threads)]
    sweeps = [O.RefBowSweep([kfs[i] for i in idx]) if (kind == "reference" and O.have_matchref()) else None for idx in per]
    scorers = [O.PortScoreSweep([kf_bows[i] for i in idx]) for idx in per]
    from orb_slam2_b200.matcher import FeatureVector, KeyFrameView

    def make(t):
        def run(i):
            k, d = queries[i % len(queries)]
            bw, bv, (fn, fs, fi) = O.port_compute_bow(voc, d, 4)
            scorers[t](bw, bv)
            F = KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=FeatureVector(fn, fs, fi))
            if sweeps[t] is not None:
                fh = sweeps[t].frame(F)
                sweeps[t].sweep(fh, 0.75, True)
                sweeps[t].free_frame(fh)
            else:
                for j in per[t]:
                    O.port_search_by_bow(kfs[j], F, 0.75, True)
        return run
    desc = (f"per query: TemplatedVocabulary::transform + L1 scoring (restated, oracle port) + the reference's ORBmatcher::SearchByBoW compiled verbatim "
            f"(oracle/_ref) against a {sample}-keyframe sample of the {n_kf}-keyframe database per thread, rate scaled by {sample}/{n_kf}")
    return kind, desc, [make(t) for t in range(threads)], sample / float(n_kf)


def build_cpu_data(cfg: int, rank: int = 0, n_kf: int = 2000, sample: int = 64):
    """Inputs of the CPU arm built WITHOUT a GPU (the reference arm must run on a box's host cores alone)."""
    from oracle import oracle_lib as O
    w, h, nfeat, _ = SHAPES[cfg]
    if cfg == 1:
        return make_pairs(rank, 16, w, h)
    if cfg == 2:
        imgs, raws = make_rgbd(rank, 8, w, h)
        depths_f = [O.port_depth_to_float(r, TUM1_DEPTH_FACTOR) for r in raws]
        E = O.PortExtractor(nfeat)
        mps = []
        for i, im in enumerate(imgs):
            k, d = E(im)
            fr = O.port_rgbd_frame(k, np.array(TUM1_K, np.float32), np.array(TUM1_DIST, np.float32), TUM1_BF, depths_f[i])
            mps.append(make_mappoints(fr["keys_un"], d, E.scale, np.random.default_rng([SEED, rank, i, 5]), fr["u_right"]))   # projections live in the undistorted image
        return imgs, depths_f, mps
    # cfg 4: a database sample is enough for the CPU arm (cost is linear in the keyframes): `sample` keyframes per thread
    voc = O.PortVocabulary.random(10, 6, 7)
    E = O.PortExtractor(nfeat)
    from orb_slam2_b200 import synth
    from orb_slam2_b200.matcher import FeatureVector, KeyFrameView
    rng = np.random.default_rng(1)
    src = [E(synth.mono_frame(50 + i, 0, 0, w, h)) for i in range(8)]
    kfs, bows = [], []
    for j in range(max(sample * 2, 16)):
        k, d = src[j % len(src)]
        if j >= len(src):
            flip = (rng.random((len(d), 32, 8)) < 0.04)
            d = d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)
        bw, bv, (fn, fs, fi) = O.port_compute_bow(voc, d, 4)
        kfs.append(KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=FeatureVector(fn, fs, fi), has_mp=np.ones(len(k), np.uint8)))
        bows.append((bw, bv))
    queries = [src[3], src[5]]
    # the database the GPU arm sweeps has n_kf keyframes; the CPU arm times `sample` of them per thread and scales
    return voc, kfs, bows, queries, min(sample, len(kfs)), n_kf


def run_cpu_baseline(cfg: int, threads: int, data, items_per_thread: int):
    """(all-core rate, one-core rate, kind, description, seconds) in frames/s of the config's workload."""
    kind, desc, workers, scale = cpu_workers(cfg, threads, data)
    pool = CpuPool(workers)
    pool.run(1)                                          # warm-up: arena page faults, caches
    rate, dt = pool.run(items_per_thread)
    one = CpuPool(workers[:1])
    rate1, dt1 = one.run(max(1, items_per_thread // 2))
    return rate * scale, rate1 * scale, kind, desc, dt + dt1


def run_reference(args, rank: int):
    if rank != 0:
        return
    cfg = args.config
    threads = host_cores()
    data = build_cpu_data(cfg, 0, args.keyframes)
    kind, desc, workers, scale = cpu_workers(cfg, threads, data)
    pool = CpuPool(workers)
    per = max(1, args.ref_items_per_thread)
    for _ in range(max(1, min(args.warmup, 2))):
        pool.run(1)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        pool.run(per)
    total = time.perf_counter() - t0
    val = threads * per * args.steps / total * scale
    sample_txt = f"{threads} threads x {per} items per step, {args.steps} steps; {desc}"
    line = {"impl": "reference", "metric": METRICS[cfg], "value": val, "unit": "frames/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": total / args.steps * 1e3, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "u8", "data": "synthetic", "config": {"workload": WORKLOADS[cfg]},
            "cpu_baseline": {"value": val, "unit": "frames/s", "cores": threads, "kind": kind, "sample": sample_txt},
            "e2e": {"value": val, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


# ----------------------------------------------------------------------------------------------
# clocks sampler
# ----------------------------------------------------------------------------------------------
class Clocks:
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap,power.draw")

    def __init__(self, gpu: int):
        self.gpu, self.p, self.lines = gpu, None, []

    def start(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                                       "-i", str(self.gpu)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.p = None

    def _read(self):
        for ln in self.p.stdout:
            self.lines.append(ln.strip())

    def stop(self):
        if not self.p:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.p.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 6:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for nm, v in zip(names, f[2:6]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


class Env:
    """torch / torch.distributed plumbing shared by the three GPU arms."""

    def __init__(self, rank, world, local_rank):
        import torch
        import torch.distributed as dist
        self.torch, self.dist = torch, dist
        self.rank, self.world, self.local_rank = rank, world, local_rank
        if not torch.cuda.is_available():
            raise SystemExit("bench.py: no CUDA device visible - the GPU arm has no CPU fallback")
        torch.cuda.set_device(local_rank)
        self.dev = torch.device("cuda", local_rank)
        if world > 1:
            os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")     # stdout carries exactly one JSON line
            dist.init_process_group("nccl", device_id=self.dev)
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        self.clocks = Clocks(local_rank if vis is None else int(vis.split(",")[local_rank]))

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def max_over_ranks(self, v: float) -> float:
        t = self.torch.tensor([v], dtype=self.torch.float64, device=self.dev)
        if self.world > 1:
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item())

    def passes_per_step(self, t_pass_s: float, multiple: int) -> int:
        """Inner repeat so that one step takes >= ~55 ms (same value on every rank), rounded up to a multiple of `multiple`
        (the input buffers x handles cycle) so that the last pass of every step sees the same input and handle."""
        t = self.max_over_ranks(t_pass_s)
        n = int(min(100000, max(1, math.ceil(0.055 / max(t, 1e-7)))))
        return -(-n // multiple) * multiple

    def finish(self):
        if self.world > 1:
            self.dist.barrier()
            self.dist.destroy_process_group()


def timed(env: Env, fn_pass, drain, K: int, inner: int):
    """K steps x inner passes between barriers + device synchronisation; CUDA events on the current stream bracket the region
    (both sides synchronised, so they and the host clock see the same interval).  Returns (event ms, wall ms)."""
    torch = env.torch
    env.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t0 = time.perf_counter()
    k = 0
    for _ in range(K):
        for _ in range(inner):
            fn_pass(k)
            k += 1
    drain()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    e1.record()
    torch.cuda.synchronize()
    return float(e0.elapsed_time(e1)), wall


# ----------------------------------------------------------------------------------------------
# configs[1]: stereo KITTI
# ----------------------------------------------------------------------------------------------
def run_config1(args, env: Env):
    torch, dist = env.torch, env.dist
    rank, world, local_rank, dev = env.rank, env.world, env.local_rank, env.dev
    from orb_slam2_b200 import _lib, sharding
    from orb_slam2_b200.extractor import ORBextractor
    from orb_slam2_b200.matcher import ORBVocabulary
    lib = _lib.load()
    W_IMG, H_IMG, NFEAT, LEVEL_PIXELS = SHAPES[1]
    B, K, Wm = args.pairs, args.steps, max(args.warmup, 3)
    NBUF, NH = 4, args.handles

    # ---- NCCL plumbing that the path really has (SURVEY §8e): the packed vocabulary (k=10, L=6 tree of ORBvoc's shape,
    # ~48 MB) is built on rank 0 only, broadcast ONCE over NCCL into every GPU's HBM and adopted there; counters are
    # all-gathered at the end.  No collective touches the per-frame data path.
    voc_ms, voc_bytes, voc = None, None, None
    if world > 1:
        if rank == 0:
            voc = ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6, device=local_rank)
            ptr, nbytes = voc.blob()
            src_blob = torch.as_tensor(sharding.DeviceBlobView(ptr, nbytes), device=dev)
        else:
            src_blob = None
        torch.cuda.synchronize()
        dist.barrier()
        t0 = time.perf_counter()
        blob = sharding.broadcast_blob(src_blob, src=0, device=dev)
        torch.cuda.synchronize()
        voc_ms = (time.perf_counter() - t0) * 1e3
        voc_bytes = int(blob.numel())
        if rank != 0:
            voc = ORBVocabulary.from_blob(blob.data_ptr(), voc_bytes, device=local_rank)

    # ---- synthetic inputs: B distinct pairs of this rank's camera stream; NBUF rotating batches (row-rolled copies keep the
    # stereo geometry) so consecutive steps never re-read the same pixels from L2
    t0 = time.perf_counter()
    Ls, Rs = make_pairs(rank, B, W_IMG, H_IMG)
    host = np.empty((NBUF, 2 * B, H_IMG, W_IMG), np.uint8)
    for j in range(NBUF):
        for p in range(B):
            host[j, 2 * p] = np.roll(Ls[p], 37 * j, axis=0)
            host[j, 2 * p + 1] = np.roll(Rs[p], 37 * j, axis=0)
    log(f"[rank {rank}] generated {B} pairs x {NBUF} buffers in {time.perf_counter() - t0:.1f}s")
    d_in = torch.from_numpy(host).to(dev)
    pitch, img_stride = W_IMG, W_IMG * H_IMG

    exts = [ORBextractor(NFEAT, 1.2, 8, 20, 7, device=local_rank) for _ in range(NH)]
    cap = exts[0].capacity(W_IMG, H_IMG)
    for x in exts:
        x.reserve(W_IMG, H_IMG, 2 * B)
    b = float(np.float32(BF) / np.float32(FX))
    n_lr = [(torch.zeros(B, dtype=torch.int32).pin_memory(), torch.zeros(B, dtype=torch.int32).pin_memory()) for _ in range(NH)]

    # ---- parity before timing: the first pairs of buffer 0 against the oracle (outside every timed region)
    parity = None
    if rank == 0 and not args.no_parity:
        from oracle import oracle_lib as O
        got = exts[0].stereo_frames([host[0, 0]], [host[0, 1]], BF, FX)[0]
        E1, E2 = O.PortExtractor(NFEAT), O.PortExtractor(NFEAT)
        kl, dl = E1(host[0, 0]); kr, dr = E2(host[0, 1])
        ur, dp, _ = O.port_stereo(kl, dl, kr, dr, [E1.level(i) for i in range(8)], [E2.level(i) for i in range(8)], E1.scale, E1.inv_scale, BF, FX)
        assert np.array_equal(got["mvKeys"], kl) and np.array_equal(got["mDescriptors"], dl) and np.array_equal(got["mvKeysRight"], kr)
        assert np.array_equal(got["mDescriptorsRight"], dr) and np.array_equal(got["mvuRight"], ur) and np.array_equal(got["mvDepth"], dp)
        parity = f"pair 0 of buffer 0: {len(kl)}+{len(kr)} keypoints, descriptors, mvuRight, mvDepth bit-identical to the oracle"

    def step_resident(k):
        x, (nl, nr) = exts[k % NH], n_lr[k % NH]
        _lib.check(lib.borb_stereo_frames_device_enqueue(x._h, d_in[k % NBUF].data_ptr(), B, W_IMG, H_IMG, pitch, img_stride, BF, b,
                                                         nl.data_ptr(), nr.data_ptr(), None, None, cap), "stereo_frames_device_enqueue")

    def drain():
        for x in exts:
            _lib.check(lib.borb_sync(x._h), "borb_sync")

    env.clocks.start()          # sampled across warm-up and BOTH timed regions (continuous load)
    for k in range(Wm * NH):
        step_resident(k)
    drain()
    assert int(n_lr[0][0].min()) >= NFEAT, "warm-up produced too few keypoints"
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for k in range(NH * 4):
        step_resident(k)
    drain(); torch.cuda.synchronize()
    inner = env.passes_per_step((time.perf_counter() - t0) / (NH * 4), math.lcm(NBUF, NH))

    # ---- timed region 1: HBM-resident throughput
    launches0 = sum(x.launch_count() for x in exts)
    ms, _ = timed(env, step_resident, drain, K, inner)
    launches = sum(x.launch_count() for x in exts) - launches0
    if args.dump_outputs and rank == 0:
        # the last pass ran on handle NH-1 over buffer NBUF-1 (inner is a multiple of both); its results are still in HBM
        from orb_slam2_b200._lib import KP_DTYPE
        n = min(B, 64)                                        # 64 pairs x ~0.7 MB stay under the dump limit
        kl, kr = np.zeros((n, cap), KP_DTYPE), np.zeros((n, cap), KP_DTYPE)
        dl, dr = np.zeros((n, cap, 32), np.uint8), np.zeros((n, cap, 32), np.uint8)
        nl, nr = np.zeros(n, np.int32), np.zeros(n, np.int32)
        ur, dp = np.zeros((n, cap), np.float32), np.zeros((n, cap), np.float32)
        _lib.check(lib.borb_stereo_frames_results(exts[(K * inner - 1) % NH]._h, n, kl.ctypes.data, dl.ctypes.data, nl.ctypes.data,
                                                  kr.ctypes.data, dr.ctypes.data, nr.ctypes.data, ur.ctypes.data, dp.ctypes.data, cap),
                   "stereo_frames_results")
        dump_outputs(args.dump_outputs, {
            "n_left": nl, "n_right": nr,
            "keypoints_left": np.concatenate([keypoint_columns(kl[p, :nl[p]]) for p in range(n)]),
            "keypoints_right": np.concatenate([keypoint_columns(kr[p, :nr[p]]) for p in range(n)]),
            "descriptors_left": np.concatenate([dl[p, :nl[p]] for p in range(n)]),
            "descriptors_right": np.concatenate([dr[p, :nr[p]] for p in range(n)]),
            "u_right": np.concatenate([ur[p, :nl[p]] for p in range(n)]), "depth": np.concatenate([dp[p, :nl[p]] for p in range(n)])})
    # per-kernel device times: a short single-handle pass right after the timed region (with several batches in flight the
    # events of one stream would also count the other streams' kernels), CUDA events on the launching stream
    exts[0].set_timing(True)
    for k in range(0, NH * 16, NH):
        step_resident(k)
    drain()
    tot = (C.c_double * 8)(); nst = C.c_uint64()
    _lib.check(lib.borb_stage_times_total(exts[0]._h, tot, C.byref(nst)), "borb_stage_times_total")
    exts[0].set_timing(False)
    stage_ms = {n: float(tot[i] / max(nst.value, 1)) for i, n in enumerate(("upload", "pyramid", "fast_nms", "quadtree", "blur", "orient_brief", "stereo", "download"))}
    ms_max = env.max_over_ranks(ms)
    value = world * B * K * inner / (ms_max * 1e-3)

    # ---- timed region 2: end to end through the C ABI with HOST buffers
    h_in = torch.from_numpy(host).pin_memory()
    outs = []
    for _ in range(NH):
        outs.append(dict(kl=torch.empty((B, cap, 28), dtype=torch.uint8).pin_memory(), kr=torch.empty((B, cap, 28), dtype=torch.uint8).pin_memory(),
                         dl=torch.empty((B, cap, 32), dtype=torch.uint8).pin_memory(), dr=torch.empty((B, cap, 32), dtype=torch.uint8).pin_memory(),
                         nl=torch.zeros(B, dtype=torch.int32).pin_memory(), nr=torch.zeros(B, dtype=torch.int32).pin_memory(),
                         ur=torch.empty((B, cap), dtype=torch.float32).pin_memory(), dp=torch.empty((B, cap), dtype=torch.float32).pin_memory()))
    ptr_tabs = []
    for j in range(NBUF):
        base = h_in[j].data_ptr()
        ptr_tabs.append(((C.c_void_p * B)(*[base + (2 * p) * img_stride for p in range(B)]), (C.c_void_p * B)(*[base + (2 * p + 1) * img_stride for p in range(B)])))

    def step_e2e(k):
        x, o = exts[k % NH], outs[k % NH]
        _lib.check(lib.borb_sync(x._h), "borb_sync")               # previous use of this handle / its host buffers
        pl, pr = ptr_tabs[k % NBUF]
        _lib.check(lib.borb_stereo_frames_enqueue(x._h, pl, pr, B, W_IMG, H_IMG, W_IMG, BF, b, o["kl"].data_ptr(), o["dl"].data_ptr(),
                                                  o["nl"].data_ptr(), o["kr"].data_ptr(), o["dr"].data_ptr(), o["nr"].data_ptr(),
                                                  o["ur"].data_ptr(), o["dp"].data_ptr(), cap), "stereo_frames_enqueue")

    for k in range(Wm * NH):
        step_e2e(k)
    drain()
    _, e2e_wall = timed(env, step_e2e, drain, K, inner)
    e2e_value = world * B * K * inner / (env.max_over_ranks(e2e_wall) * 1e-3)
    clk = env.clocks.stop()
    assert int(outs[0]["nl"].min()) >= NFEAT
    h2d = 2 * B * W_IMG * H_IMG
    d2h = B * (2 * cap * (28 + 32) + 2 * 4 + 2 * cap * 4)

    gathered = None
    if world > 1:
        kps0 = outs[0]["dl"][0, :NFEAT].numpy()
        words, _, _ = voc.transform_raw(kps0, 4)
        gathered = sharding.gather_counters([B * K * inner, int(n_lr[0][0].sum()), int(n_lr[0][1].sum()), int((outs[0]["ur"] >= 0).sum()),
                                             int(words.astype(np.int64).sum() % (1 << 31))], device=dev).tolist()
    if rank != 0:
        return
    peak, peak_src = hbm_peak()
    fast_bytes = LEVEL_PIXELS * 2 * B
    fast_ms = stage_ms["fast_nms"]
    achieved = fast_bytes / (fast_ms * 1e-3) / 1e9 if fast_ms > 0 else 0.0
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        threads = host_cores()
        r_all, r_one, kind, desc, dt = run_cpu_baseline(1, threads, (Ls[:16], Rs[:16]), args.cpu_items_per_thread)
        cpu = {"value": r_all, "unit": "frames/s", "cores": threads, "kind": kind, "one_core_value": r_one,
               "sample": f"{threads} host threads x {args.cpu_items_per_thread} of the same synthetic stereo pairs ({dt:.1f}s wall); {desc}"}
    line = {"metric": METRICS[1], "value": value, "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": Wm,
            "ms_per_step": ms_max / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
            "config": {"workload": WORKLOADS[1], "pairs_per_pass_per_gpu": B, "passes_per_step": inner, "batches_in_flight": NH,
                       "parallelism": f"{world} independent camera streams, one per GPU (no data-path collective)",
                       "cache": f"inputs larger than L2: {NBUF} rotating batches x {2 * B * W_IMG * H_IMG / 1e6:.0f} MB input + {2 * B * 2 * 1.75:.0f} MB pyramids per pass vs 50 MB L2",
                       "parity_checked": parity},
            "clocks": clk, "gpu_launches": int(launches),
            "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": h2d * inner, "d2h_bytes_per_step": d2h * inner},
            "roofline": {"kernel": "fast_kernel", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": None, "peak_source": peak_src, "algorithmic_bytes_per_launch": fast_bytes,
                         "mean_launch_ms": fast_ms},
            "stage_ms_per_pass": stage_ms, "cpu_baseline": cpu}
    if voc_ms is not None:
        line["nccl"] = {"vocabulary_broadcast_ms": voc_ms, "vocabulary_bytes": voc_bytes,
                        "counter_fields": list(sharding.COUNTER_FIELDS[:4]) + ["vocabulary_word_checksum"], "counters_all_gather": gathered}
    print(json.dumps(line), flush=True)


# ----------------------------------------------------------------------------------------------
# configs[2]: RGB-D TUM — extract + Frame constructor tail + SearchByProjection vs 300 local MapPoints
# ----------------------------------------------------------------------------------------------
def run_config2(args, env: Env):
    torch = env.torch
    rank, world, local_rank, dev = env.rank, env.world, env.local_rank, env.dev
    from orb_slam2_b200 import _lib, matcher as M
    from orb_slam2_b200.extractor import ORBextractor
    lib = _lib.load()
    W, H, NFEAT, LEVEL_PIXELS = SHAPES[2]
    B, K, Wm = args.frames, args.steps, max(args.warmup, 3)
    NBUF, NH = 4, args.handles

    imgs, raws = make_rgbd(rank, B, W, H)
    himg = np.empty((NBUF, B, H, W), np.uint8); hdep = np.empty((NBUF, B, H, W), np.uint16)
    for j in range(NBUF):
        for i in range(B):
            himg[j, i] = np.roll(imgs[i], 41 * j, axis=0); hdep[j, i] = np.roll(raws[i], 41 * j, axis=0)
    h_img, h_dep = torch.from_numpy(himg).pin_memory(), torch.from_numpy(hdep.view(np.int16)).pin_memory()
    d_img, d_dep = h_img.to(dev), h_dep.to(dev)
    exts = [ORBextractor(NFEAT, 1.2, 8, 20, 7, device=local_rank) for _ in range(NH)]
    mats = [M.ORBmatcher(0.8, True, device=local_rank) for _ in range(NH)]
    cap = exts[0].capacity(W, H)
    for x in exts:
        x.reserve(W, H, B)
    sf = exts[0].GetScaleFactors()
    cam = M._CameraC(*TUM1_K, *TUM1_DIST, TUM1_BF)
    factor = float(np.float32(TUM1_DEPTH_FACTOR))

    # ---- MapPoints of every (buffer, frame): from a first extraction; pinned, prebuilt C views
    mp_views, mp_keep, first = [], [], {}
    for j in range(NBUF):
        outs = exts[0].extract_batch([himg[j, i] for i in range(B)])
        _, hst = M.frames_from_extractor(mats[0], exts[0], np.arange(B), [len(k) for k, _ in outs], TUM1_K, TUM1_DIST, bf=TUM1_BF, mode=2,
                                         depth=[hdep[j, i] for i in range(B)], depth_factor=TUM1_DEPTH_FACTOR)
        row = []
        for i, (k, d) in enumerate(outs):
            m = make_mappoints(hst["keys_un"][i], d, sf, np.random.default_rng([SEED, rank, j, i]), hst["u_right"][i])     # projections live in the undistorted image
            arrs = [np.ascontiguousarray(m[f]) for f in ("px", "py", "pxr", "lvl", "vc", "desc")]
            mp_keep.append(arrs)
            row.append(M._MapPointViewC(len(arrs[0]), *[a.ctypes.data for a in arrs], None, None))
            if j == 0 and i < 3:
                first[i] = (k, d, m)
        mp_views.append(row)
    mp_arrays = [(M._MapPointViewC * B)(*mp_views[j]) for j in range(NBUF)]          # contiguous view arrays for the batched call
    images = np.arange(B, dtype=np.int32)

    # ---- parity before timing (rank 0): extraction, frame tail and matches of the first frames against the oracle
    parity = None
    if rank == 0 and not args.no_parity:
        from oracle import oracle_lib as O
        exts[0].extract_batch([himg[0, i] for i in range(B)])
        nk = np.array([len(first[i][0]) for i in range(3)], np.int32)
        frames, host = M.frames_from_extractor(mats[0], exts[0], [0, 1, 2], nk, TUM1_K, TUM1_DIST, bf=TUM1_BF, mode=2,
                                               depth=[hdep[0, i] for i in range(3)], depth_factor=TUM1_DEPTH_FACTOR)
        E = O.PortExtractor(NFEAT)
        tot_m = 0
        for i in range(3):
            k, d, m = first[i]
            ko, do = E(himg[0, i])
            assert np.array_equal(k, ko) and np.array_equal(d, do), "extraction differs from the oracle"
            want = O.port_rgbd_frame(ko, np.array(TUM1_K, np.float32), np.array(TUM1_DIST, np.float32), TUM1_BF, O.port_depth_to_float(hdep[0, i], TUM1_DEPTH_FACTOR))
            assert np.array_equal(host["keys_un"][i], want["keys_un"]) and np.array_equal(host["u_right"][i], want["u_right"]) and np.array_equal(host["depth"][i], want["depth"])
            F = M.FrameView(want["keys_un"], do, sf, tuple(float(x) for x in want["bounds"]), mvuRight=want["u_right"])
            mv = M.MapPointsView(m["px"], m["py"], m["pxr"], m["lvl"], m["vc"], m["desc"])
            n_o, m_o = O.port_search_by_projection(F, mv, 3.0, 0.8)
            n_g, m_g = mats[0].SearchByProjection(frames[i], mv, 3.0)
            assert n_g == n_o and np.array_equal(m_g, m_o), "SearchByProjection differs from the oracle"
            (n_b, m_b), = mats[0].SearchByProjectionBatch([frames[i]], [mv], 3.0)
            assert n_b == n_o and np.array_equal(m_b, m_o), "batched SearchByProjection differs from the oracle"
            tot_m += n_g
        parity = f"frames 0-2 of buffer 0: keypoints, descriptors, mvKeysUn, mvuRight, mvDepth and {tot_m} SearchByProjection matches bit-identical to the oracle"
        del frames

    # ---- per-handle call state
    class H_:
        pass
    hs = []
    for k in range(NH):
        s = H_()
        s.x, s.m = exts[k], mats[k]
        s.n_out = np.zeros(B, np.int32)
        s.frames = (C.c_void_p * B)()
        s.b4 = np.zeros(4, np.float32)
        s.match = np.zeros(N_MAPPOINTS + 8, np.int32)
        s.nm = C.c_int32(0)
        s.fv = M._FrameViewC(0, None, None, None, None, 0.0, 0.0, 0.0, 0.0, 8, None, None)
        s.kps = torch.empty((B, cap, 28), dtype=torch.uint8).pin_memory(); s.desc = torch.empty((B, cap, 32), dtype=torch.uint8).pin_memory()
        s.ku = torch.empty((B, cap, 28), dtype=torch.uint8).pin_memory(); s.ur = torch.empty((B, cap), dtype=torch.float32).pin_memory()
        s.dp = torch.empty((B, cap), dtype=torch.float32).pin_memory()
        s.matches = 0
        s.fvs = (M._FrameViewC * B)(*[M._FrameViewC(0, None, None, None, None, 0.0, 0.0, 0.0, 0.0, 8, None, None) for _ in range(B)])
        s.match_all = np.zeros((B, N_MAPPOINTS + 8), np.int32)
        s.match_ptrs = (C.c_void_p * B)(*[s.match_all[i].ctypes.data for i in range(B)])
        s.nms = np.zeros(B, np.int32)
        hs.append(s)
    dep_dev = [(C.c_void_p * B)(*[d_dep[j, i].data_ptr() for i in range(B)]) for j in range(NBUF)]
    dep_host = [(C.c_void_p * B)(*[h_dep[j, i].data_ptr() for i in range(B)]) for j in range(NBUF)]
    img_host = [(C.c_void_p * B)(*[h_img[j, i].data_ptr() for i in range(B)]) for j in range(NBUF)]
    p_images, p_i32 = images.ctypes.data, C.POINTER(C.c_int32)

    def match_all(s, j):
        # the B frames of the pass belong to B independent camera streams: ONE batched call (one launch pair, one synchronisation)
        if args.per_frame_calls:
            tot = 0
            for i in range(B):
                s.fv.resident = s.frames[i]
                _lib.check(lib.borb_search_by_projection(s.m._h, C.byref(s.fv), C.byref(mp_views[j][i]), 3.0, 0.8, s.match.ctypes.data, C.byref(s.nm)), "search_by_projection")
                tot += s.nm.value
        else:
            for i in range(B):
                s.fvs[i].resident = s.frames[i]
            _lib.check(lib.borb_search_by_projection_batch(s.m._h, s.fvs, mp_arrays[j], B, 3.0, 0.8, s.match_ptrs, s.nms.ctypes.data), "search_by_projection_batch")
            tot = int(s.nms.sum())
        for i in range(B):
            lib.borb_frame_destroy(s.frames[i])
        s.matches = tot

    def pass_resident(s, k):
        j = k % NBUF
        _lib.check(lib.borb_extract_batch_device(s.x._h, d_img[j].data_ptr(), B, W, H, W, W * H, None, None, cap, s.n_out.ctypes.data), "extract_batch_device")
        _lib.check(lib.borb_frames_from_extractor(s.m._h, s.x._h, p_images, B, s.n_out.ctypes.data, C.byref(cam), 2, dep_dev[j], 1 | 4, factor, 0,
                                                  None, None, None, 0, s.b4.ctypes.data, s.frames), "frames_from_extractor")
        match_all(s, j)

    def pass_e2e(s, k):
        j = k % NBUF
        _lib.check(lib.borb_extract_batch(s.x._h, img_host[j], B, W, H, W, s.kps.data_ptr(), s.desc.data_ptr(), cap, s.n_out.ctypes.data), "extract_batch")
        _lib.check(lib.borb_frames_from_extractor(s.m._h, s.x._h, p_images, B, s.n_out.ctypes.data, C.byref(cam), 2, dep_host[j], 1, factor, 2 * W,
                                                  s.ku.data_ptr(), s.ur.data_ptr(), s.dp.data_ptr(), cap, s.b4.ctypes.data, s.frames), "frames_from_extractor")
        match_all(s, j)

    # NH host threads = NH camera-stream groups, each with its own extractor + matcher handle (ctypes releases the GIL)
    def run_passes(fn, n_total):
        """n_total passes dealt round-robin to the NH handle threads."""
        errs = []

        def body(t):
            try:
                for k in range(t, n_total, NH):
                    fn(hs[t], k)
            except BaseException as ex:       # a worker thread must not die silently
                errs.append(ex)
        ths = [threading.Thread(target=body, args=(t,)) for t in range(NH)]
        for th in ths: th.start()
        for th in ths: th.join()
        if errs:
            raise errs[0]

    env.clocks.start()
    run_passes(pass_resident, Wm * NH)
    assert hs[0].matches > B * 100, f"warm-up produced too few matches ({hs[0].matches} for {B} frames)"
    torch.cuda.synchronize(); t0 = time.perf_counter()
    run_passes(pass_resident, NH * 2)
    torch.cuda.synchronize()
    inner = env.passes_per_step((time.perf_counter() - t0) / (NH * 2), math.lcm(NBUF, NH))
    launches0 = sum(x.launch_count() for x in exts)
    ml0 = sum(_mlaunch(lib, m) for m in mats)
    ms, _ = timed(env, lambda k: None, lambda: run_passes(pass_resident, K * inner), 0, 0)
    launches = sum(x.launch_count() for x in exts) - launches0 + sum(_mlaunch(lib, m) for m in mats) - ml0
    if args.dump_outputs and rank == 0:
        last = hs[(K * inner - 1) % NH]                       # the last pass: handle NH-1, buffer NBUF-1 (inner is a multiple of both)
        dump_outputs(args.dump_outputs, {"n_keypoints": last.n_out, "n_matches": last.nms, "matches": last.match_all[:, :N_MAPPOINTS]})
    ms_max = env.max_over_ranks(ms)
    value = world * B * K * inner / (ms_max * 1e-3)
    # FAST stage time (single handle, CUDA events on the library's stream)
    exts[0].set_timing(True)
    for k in range(16):
        _lib.check(lib.borb_extract_batch_device(exts[0]._h, d_img[k % NBUF].data_ptr(), B, W, H, W, W * H, None, None, cap, hs[0].n_out.ctypes.data), "extract")
    tot = (C.c_double * 8)(); nst = C.c_uint64()
    _lib.check(lib.borb_stage_times_total(exts[0]._h, tot, C.byref(nst)), "stage_times_total")
    exts[0].set_timing(False)
    stage_ms = {n: float(tot[i] / max(nst.value, 1)) for i, n in enumerate(("upload", "pyramid", "fast_nms", "quadtree", "blur", "orient_brief", "stereo", "download"))}

    run_passes(pass_e2e, Wm * NH)
    _, e2e_wall = timed(env, lambda k: None, lambda: run_passes(pass_e2e, K * inner), 0, 0)
    e2e_value = world * B * K * inner / (env.max_over_ranks(e2e_wall) * 1e-3)

    # ---- single-stream call latency of the matcher on a resident frame (the number a Tracking thread sees per frame)
    s = hs[0]
    _lib.check(lib.borb_extract_batch_device(s.x._h, d_img[0].data_ptr(), B, W, H, W, W * H, None, None, cap, s.n_out.ctypes.data), "extract")
    _lib.check(lib.borb_frames_from_extractor(s.m._h, s.x._h, p_images, B, s.n_out.ctypes.data, C.byref(cam), 2, dep_dev[0], 1 | 4, factor, 0,
                                              None, None, None, 0, s.b4.ctypes.data, s.frames), "frames_from_extractor")
    lat = []
    for r in range(400):
        i = r % B
        s.fv.resident = s.frames[i]
        t0 = time.perf_counter()
        lib.borb_search_by_projection(s.m._h, C.byref(s.fv), C.byref(mp_views[0][i]), 3.0, 0.8, s.match.ctypes.data, C.byref(s.nm))
        lat.append(time.perf_counter() - t0)
    for i in range(B):
        lib.borb_frame_destroy(s.frames[i])
    lat = np.array(lat[100:]) * 1e6
    clk = env.clocks.stop()
    if rank != 0:
        return
    peak, peak_src = hbm_peak()
    fast_bytes = LEVEL_PIXELS * B
    fast_ms = stage_ms["fast_nms"]
    achieved = fast_bytes / (fast_ms * 1e-3) / 1e9 if fast_ms > 0 else 0.0
    mp_bytes = N_MAPPOINTS * (4 * 5 + 32)
    h2d = B * (W * H + 2 * W * H + mp_bytes)
    d2h = B * (cap * (28 + 32) + cap * (28 + 8) + N_MAPPOINTS * 4 + 8)
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        threads = host_cores()
        data = build_cpu_data(2, rank)
        r_all, r_one, kind, desc, dt = run_cpu_baseline(2, threads, data, args.cpu_items_per_thread)
        # the verbatim matcher call alone, one core (what the judge's "on par with one CPU core" referred to)
        from oracle import oracle_lib as O
        cpu_match_us = None
        if O.have_matchref():
            k, d, m = first[0]
            want = O.port_rgbd_frame(k, np.array(TUM1_K, np.float32), np.array(TUM1_DIST, np.float32), TUM1_BF, O.port_depth_to_float(hdep[0, 0], TUM1_DEPTH_FACTOR))
            F = M.FrameView(want["keys_un"], d, sf, tuple(float(x) for x in want["bounds"]), mvuRight=want["u_right"])
            mv = M.MapPointsView(m["px"], m["py"], m["pxr"], m["lvl"], m["vc"], m["desc"])
            tt = []
            for _ in range(30):
                t0 = time.perf_counter(); O.ref_search_by_projection(F, mv, 3.0, 0.8); tt.append(time.perf_counter() - t0)
            cpu_match_us = float(np.median(tt) * 1e6)
        cpu = {"value": r_all, "unit": "frames/s", "cores": threads, "kind": kind, "one_core_value": r_one,
               "search_by_projection_us_per_call_one_core": cpu_match_us,
               "sample": f"{threads} host threads x {args.cpu_items_per_thread} of the same synthetic RGB-D frames ({dt:.1f}s wall); {desc}"}
    line = {"metric": METRICS[2], "value": value, "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": Wm, "ms_per_step": ms_max / K,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
            "config": {"workload": WORKLOADS[2], "frames_per_pass_per_gpu": B, "passes_per_step": inner, "batches_in_flight": NH,
                       "map_points_per_frame": N_MAPPOINTS, "camera": "TUM1.yaml (k1 = 0.2624: UndistortKeyPoints active), DepthMapFactor 5000, CV_16U depth",
                       "parallelism": f"{world} GPUs x {NH} host threads, each {B} independent RGB-D streams per pass (no data-path collective)",
                       "cache": f"inputs larger than L2: {NBUF} rotating batches; {NH} handles x {B} x 1.9 MB of pyramids + blurred copies in flight vs 50 MB L2",
                       "parity_checked": parity},
            "clocks": clk, "gpu_launches": int(launches),
            "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": h2d * inner, "d2h_bytes_per_step": d2h * inner},
            "roofline": {"kernel": "fast_kernel", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                         "peak_source": peak_src, "algorithmic_bytes_per_launch": fast_bytes, "mean_launch_ms": fast_ms},
            "matcher_calls": "one borb_search_by_projection call per frame" if args.per_frame_calls else "one borb_search_by_projection_batch call per pass (the frames of a pass are independent camera streams)",
            "matcher_latency": {"call": "borb_search_by_projection on a device-resident frame, 300 MapPoints from host buffers, matches back to the host",
                                "us_p50": float(np.median(lat)), "us_p10": float(np.percentile(lat, 10)), "us_p99": float(np.percentile(lat, 99)), "calls": int(len(lat))},
            "stage_ms_per_pass": stage_ms, "cpu_baseline": cpu}
    print(json.dumps(line), flush=True)


def _mlaunch(lib, m):
    n = C.c_uint64(0)
    lib.borb_matcher_launch_count(m._h, C.byref(n))
    return n.value


# ----------------------------------------------------------------------------------------------
# configs[4]: loop-closure / relocalisation query against a 2000-keyframe resident database
# ----------------------------------------------------------------------------------------------
def run_config4(args, env: Env):
    torch, dist = env.torch, env.dist
    rank, world, local_rank, dev = env.rank, env.world, env.local_rank, env.dev
    from orb_slam2_b200 import _lib, matcher as M, sharding, synth
    from orb_slam2_b200.extractor import ORBextractor
    lib = _lib.load()
    W, H, NFEAT, _ = SHAPES[4]
    n_kf, K, Wm = args.keyframes, args.steps, max(args.warmup, 3)
    Q = args.queries

    # ---- vocabulary: built on rank 0, broadcast over NCCL, adopted from the blob elsewhere (SURVEY §8e)
    voc_ms, voc_bytes = None, None
    if world > 1:
        if rank == 0:
            voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6, device=local_rank)
            ptr, nbytes = voc.blob()
            src_blob = torch.as_tensor(sharding.DeviceBlobView(ptr, nbytes), device=dev)
        else:
            src_blob = None
        torch.cuda.synchronize(); dist.barrier(); t0 = time.perf_counter()
        blob = sharding.broadcast_blob(src_blob, src=0, device=dev)
        torch.cuda.synchronize()
        voc_ms, voc_bytes = (time.perf_counter() - t0) * 1e3, int(blob.numel())
        if rank != 0:
            voc = M.ORBVocabulary.from_blob(blob.data_ptr(), voc_bytes, device=local_rank)
    else:
        voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6, device=local_rank)

    X = ORBextractor(NFEAT, 1.2, 8, 20, 7, device=local_rank)
    mt = M.ORBmatcher(0.75, True, device=local_rank)
    db = M.KeyFrameDatabase(mt, device=local_rank)
    rng = np.random.default_rng(1)
    n_src = 40
    t0 = time.perf_counter()
    outs = X.extract_batch([synth.mono_frame(50 + i, rank, 0, W, H) for i in range(n_src)])
    kfs, bows, db_bytes, n_feat = [], [], 0, 0
    for j in range(n_kf):
        k, d = outs[j % n_src]
        if j >= n_src:                                         # further keyframes: ~4 % of the descriptor bits flipped
            flip = (rng.random((len(d), 32, 8)) < 0.04)
            d = d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)
        bow, fv = voc.ComputeBoW(d, 4)
        kf = M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=np.ones(len(k), np.uint8))
        db.add(kf, bow)
        m = len(fv.feat_idx)
        db_bytes += m * (32 + 2 + 4 + 1) + len(fv.node_id) * 8 + 4
        n_feat += len(k)
        if j < 64 or j % 97 == 0:
            kfs.append((j, kf, bow))
    log(f"[rank {rank}] database of {n_kf} keyframes ({db.size()[1] / 1e6:.0f} MB in HBM) built in {time.perf_counter() - t0:.1f}s")
    # query frames: EuRoC-shaped stereo pairs of scenes that are in the database
    Lq, Rq = [], []
    for q in range(Q):
        l, r, _ = synth.stereo_pair(SEED, rank, q, W, H)
        Lq.append(synth.mono_frame(50 + (3 + 5 * q) % n_src, rank, 0, W, H) if q % 2 == 0 else l); Rq.append(r)
    cap = X.capacity(W, H)
    X.reserve(W, H, 2 * Q)
    hq = torch.from_numpy(np.stack([np.stack([Lq[q], Rq[q]]) for q in range(Q)])).pin_memory()       # (Q, 2, H, W)
    pl = (C.c_void_p * Q)(*[hq[q, 0].data_ptr() for q in range(Q)]); pr = (C.c_void_p * Q)(*[hq[q, 1].data_ptr() for q in range(Q)])
    o = dict(kl=torch.empty((Q, cap, 28), dtype=torch.uint8).pin_memory(), kr=torch.empty((Q, cap, 28), dtype=torch.uint8).pin_memory(),
             dl=torch.empty((Q, cap, 32), dtype=torch.uint8).pin_memory(), dr=torch.empty((Q, cap, 32), dtype=torch.uint8).pin_memory(),
             nl=torch.zeros(Q, dtype=torch.int32).pin_memory(), nr=torch.zeros(Q, dtype=torch.int32).pin_memory(),
             ur=torch.empty((Q, cap), dtype=torch.float32).pin_memory(), dp=torch.empty((Q, cap), dtype=torch.float32).pin_memory())
    b = float(np.float32(EUROC_BF) / np.float32(EUROC_FX))

    def extract_queries():
        _lib.check(lib.borb_stereo_frames(X._h, pl, pr, Q, W, H, W, EUROC_BF, b, o["kl"].data_ptr(), o["dl"].data_ptr(), o["nl"].data_ptr(),
                                          o["kr"].data_ptr(), o["dr"].data_ptr(), o["nr"].data_ptr(), o["ur"].data_ptr(), o["dp"].data_ptr(), cap), "stereo_frames")
    extract_queries()
    nq = o["nl"].numpy().copy()
    from orb_slam2_b200._lib import KP_DTYPE
    qk = [np.ascontiguousarray(o["kl"][q, :nq[q]].numpy()).view(KP_DTYPE).reshape(-1).copy() for q in range(Q)]
    qd = [np.ascontiguousarray(o["dl"][q, :nq[q]].numpy()).copy() for q in range(Q)]
    # NH query streams in flight per GPU (independent relocalising / loop-closing agents on one map): each host thread owns a matcher
    # handle, a vocabulary handle (sharing the device blob), an extractor and its call buffers; the database is shared.
    NH = max(1, args.handles)
    nmax = int(nq.max())
    vp = lambda a: a.ctypes.data
    pairs_cap = n_kf * 64 + 65536
    vptr, vbytes = voc.blob()

    class QStream:
        def __init__(self, t):
            self.mt = mt if t == 0 else M.ORBmatcher(0.75, True, device=local_rank)
            self.voc = voc if t == 0 else M.ORBVocabulary.from_blob(vptr, vbytes, device=local_rank)
            self.X = X if t == 0 else ORBextractor(NFEAT, 1.2, 8, 20, 7, device=local_rank)
            if t:
                self.X.reserve(W, H, 2 * Q)
            self.o = o if t == 0 else dict(kl=torch.empty((Q, cap, 28), dtype=torch.uint8).pin_memory(), kr=torch.empty((Q, cap, 28), dtype=torch.uint8).pin_memory(),
                                           dl=torch.empty((Q, cap, 32), dtype=torch.uint8).pin_memory(), dr=torch.empty((Q, cap, 32), dtype=torch.uint8).pin_memory(),
                                           nl=torch.zeros(Q, dtype=torch.int32).pin_memory(), nr=torch.zeros(Q, dtype=torch.int32).pin_memory(),
                                           ur=torch.empty((Q, cap), dtype=torch.float32).pin_memory(), dp=torch.empty((Q, cap), dtype=torch.float32).pin_memory())
            self.bw = np.zeros(nmax, np.uint32); self.bv = np.zeros(nmax, np.float64); self.fnode = np.zeros(nmax, np.uint32)
            self.fstart = np.zeros(nmax + 1, np.int32); self.fidx = np.zeros(nmax, np.uint32)
            self.nb, self.nn = C.c_int32(0), C.c_int32(0)
            self.cw = np.zeros(n_kf, np.int32); self.sc = np.zeros(n_kf, np.float32); self.fw = np.zeros(n_kf, np.uint32); self.ns = C.c_int32(0)
            self.nm = np.zeros(n_kf, np.int32); self.off = np.zeros(n_kf, np.int32)
            self.pairs = np.zeros(pairs_cap, np.uint32); self.npairs = C.c_int32(0)
            self.kfv = M._KeyFrameViewC()
            self.n_pairs = 0

        def extract(self):
            oo = self.o
            _lib.check(lib.borb_stereo_frames(self.X._h, pl, pr, Q, W, H, W, EUROC_BF, b, oo["kl"].data_ptr(), oo["dl"].data_ptr(), oo["nl"].data_ptr(),
                                              oo["kr"].data_ptr(), oo["dr"].data_ptr(), oo["nr"].data_ptr(), oo["ur"].data_ptr(), oo["dp"].data_ptr(), cap), "stereo_frames")

        def query(self, keys, desc, n):
            """ComputeBoW -> KeyFrameDatabase scoring -> SearchByBoW against every keyframe (compact pairs)."""
            _lib.check(lib.borb_compute_bow(self.voc._h, desc, n, 4, vp(self.bw), vp(self.bv), C.byref(self.nb), vp(self.fnode), vp(self.fstart), vp(self.fidx),
                                            C.byref(self.nn)), "compute_bow")
            _lib.check(lib.borb_kfdb_query(self.mt._h, db._h, vp(self.bw), vp(self.bv), self.nb.value, vp(self.cw), vp(self.sc), vp(self.fw), n_kf, C.byref(self.ns)), "kfdb_query")
            kfv = self.kfv
            kfv.n = n; kfv.keys_un = keys; kfv.desc = desc; kfv.has_mp = None; kfv.u_right = None
            kfv.fv = M._FeatVecC(self.nn.value, vp(self.fnode), vp(self.fstart), vp(self.fidx)); kfv.n_levels = 0; kfv.scale_factors = None; kfv.level_sigma2 = None
            _lib.check(lib.borb_search_by_bow_db_pairs(self.mt._h, db._h, None, n_kf, C.byref(kfv), 0.75, 1, vp(self.nm), vp(self.off), vp(self.pairs), pairs_cap,
                                                       C.byref(self.npairs)), "search_by_bow_db_pairs")
            self.n_pairs = self.npairs.value

    qs = [QStream(t) for t in range(NH)]
    s0 = qs[0]
    bw, bv, fnode, fstart, fidx, nb, nn = s0.bw, s0.bv, s0.fnode, s0.fstart, s0.fidx, s0.nb, s0.nn
    cw, sc, fw, nm, off, pairs = s0.cw, s0.sc, s0.fw, s0.nm, s0.off, s0.pairs
    state = dict(pairs=0)

    def query(keys, desc, n):
        s0.query(keys, desc, n)
        state["pairs"] = s0.n_pairs

    def pass_resident(st, k):
        q = k % Q
        st.query(qk[q].ctypes.data, qd[q].ctypes.data, int(nq[q]))

    def pass_e2e(st, k):
        # one pass = Q query frames: stereo extraction of the Q pairs from host images, then the three calls per query
        st.extract()
        for q in range(Q):
            st.query(st.o["kl"][q].data_ptr(), st.o["dl"][q].data_ptr(), int(st.o["nl"][q]))

    def run_passes(fn, n_total):
        """n_total passes dealt round-robin to the NH stream threads (ctypes releases the GIL during the calls)."""
        errs = []

        def body(t):
            try:
                for k in range(t, n_total, NH):
                    fn(qs[t], k)
            except BaseException as ex:
                errs.append(ex)
        ths = [threading.Thread(target=body, args=(t,)) for t in range(NH)]
        for th in ths: th.start()
        for th in ths: th.join()
        if errs:
            raise errs[0]

    # ---- parity before timing (rank 0): scores and SearchByBoW results of query 0 against the oracle on a keyframe sample
    parity = None
    if rank == 0 and not args.no_parity:
        from oracle import oracle_lib as O
        query(qk[0].ctypes.data, qd[0].ctypes.data, int(nq[0]))
        qbow = dict(zip(bw[:nb.value].tolist(), bv[:nb.value].tolist()))
        F = M.KeyFrameView(mvKeysUn=qk[0], mDescriptors=qd[0], mFeatVec=M.FeatureVector(fnode[:nn.value].copy(), fstart[:nn.value + 1].copy(), fidx[:fstart[nn.value]].copy()))
        chk = 0
        for j, kf, bow in kfs:
            so, co, fo = O.port_bow_score(qbow, bow)
            assert cw[j] == co and sc[j] == np.float32(so), "KeyFrameDatabase score differs from the oracle"
            n_o, m_o = O.port_search_by_bow(kf, F, 0.75, True)
            pr_ = pairs[off[j]:off[j] + nm[j]]
            dense = np.full(len(qk[0]), -1, np.int32); dense[(pr_ & 0xFFFF).astype(np.int64)] = (pr_ >> 16).astype(np.int32)
            assert nm[j] == n_o and np.array_equal(dense, m_o), "SearchByBoW differs from the oracle"
            chk += int(n_o)
        parity = f"query 0: L1 scores and SearchByBoW matches against {len(kfs)} of the {n_kf} keyframes ({chk} matches) bit-identical to the oracle"

    env.clocks.start()
    run_passes(pass_resident, Wm * 2 * NH)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    run_passes(pass_resident, 8 * NH)
    torch.cuda.synchronize()
    inner = env.passes_per_step((time.perf_counter() - t0) / (8 * NH), math.lcm(Q, NH))
    ml0 = sum(_mlaunch(lib, x.mt) for x in qs)
    ms, _ = timed(env, lambda k: None, lambda: run_passes(pass_resident, K * inner), 0, 0)
    launches = sum(_mlaunch(lib, x.mt) for x in qs) - ml0 + K * inner       # + the vocabulary descent kernel of every ComputeBoW
    if args.dump_outputs and rank == 0:
        st = qs[(K * inner - 1) % NH]                         # the last pass: stream NH-1, query (K * inner - 1) % Q
        dump_outputs(args.dump_outputs, {"bow_word": st.bw[:st.nb.value], "bow_value": st.bv[:st.nb.value], "common_words": st.cw,
                                         "scores": st.sc, "first_word": st.fw, "n_matches": st.nm, "pair_offset": st.off,
                                         "pairs": st.pairs[:st.npairs.value]})
    ms_max = env.max_over_ranks(ms)
    value = world * K * inner / (ms_max * 1e-3)
    # device time of the database search kernels (CUDA events on the matcher's stream), one stream alone
    lib.borb_matcher_set_timing(mt._h, 1)
    kms, lat = [], []
    for k in range(16):
        t1 = time.perf_counter()
        pass_resident(s0, k)
        lat.append((time.perf_counter() - t1) * 1e6)
        f = C.c_float(0); lib.borb_matcher_last_kernel_ms(mt._h, C.byref(f)); kms.append(f.value)
    lib.borb_matcher_set_timing(mt._h, 0)
    kernel_ms = float(np.mean(kms))
    query_us = float(np.median(lat))
    state["pairs"] = s0.n_pairs
    run_passes(pass_e2e, Wm * NH)
    inner_e = max(1, inner // Q)
    _, e2e_wall = timed(env, lambda k: None, lambda: run_passes(pass_e2e, K * inner_e), 0, 0)
    e2e_value = world * Q * K * inner_e / (env.max_over_ranks(e2e_wall) * 1e-3)
    clk = env.clocks.stop()
    if rank != 0:
        return
    peak, peak_src = hbm_peak()
    achieved = db_bytes / (kernel_ms * 1e-3) / 1e9 if kernel_ms > 0 else 0.0
    h2d = Q * (2 * W * H) + Q * (int(nq.mean()) * (32 + 2 + 4 + 4 + 12) + 4096)
    d2h = Q * (2 * cap * 60 + 8 * cap + n_kf * 20 + int(state["pairs"]) * 4 + int(nq.mean()) * 16)
    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        threads = host_cores()
        data = build_cpu_data(4, rank, n_kf)
        r_all, r_one, kind, desc, dt = run_cpu_baseline(4, threads, data, max(1, args.cpu_items_per_thread // 2))
        cpu = {"value": r_all, "unit": "frames/s", "cores": threads, "kind": kind, "one_core_value": r_one,
               "sample": f"{threads} host threads x {max(1, args.cpu_items_per_thread // 2)} queries ({dt:.1f}s wall); {desc}"}
    line = {"metric": METRICS[4], "value": value, "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": Wm, "ms_per_step": ms_max / K,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
            "config": {"workload": WORKLOADS[4], "keyframes": n_kf, "features_per_keyframe": n_feat / n_kf, "database_MB_in_HBM": db.size()[1] / 1e6,
                       "vocabulary": "k=10 L=6 seeded random tree of ORBvoc's shape (1,111,111 nodes)", "query_frames": Q, "passes_per_step": inner,
                       "pairs_per_query": int(state["pairs"]), "query_streams_in_flight": NH,
                       "parallelism": f"{world} GPUs x {NH} host threads, each an independent query stream on the GPU's database (no data-path collective; NCCL: vocabulary broadcast only)",
                       "cache": f"the database sweep reads {db_bytes / 1e6:.0f} MB per query vs 50 MB L2: successive queries do find part of it in L2 (the reference's relocalisation re-reads the same keyframes too)",
                       "e2e_pass": f"{Q} query frames: stereo extraction from host images + ComputeBoW + scoring + SearchByBoW each", "parity_checked": parity},
            "clocks": clk, "gpu_launches": int(launches),
            "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": h2d * inner_e, "d2h_bytes_per_step": d2h * inner_e},
            "roofline": {"kernel": "bowdb_match_kernel (+ bowdb_finalize_kernel)", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                         "frac": achieved / peak, "traffic": None, "peak_source": peak_src,
                         "algorithmic_bytes_per_launch": db_bytes, "mean_launch_ms": kernel_ms},
            "query_latency": {"call": "ComputeBoW + KeyFrameDatabase scoring + SearchByBoW vs all keyframes, one stream alone, host buffers in and out",
                              "us_p50": query_us},
            "cpu_baseline": cpu}
    if voc_ms is not None:
        line["nccl"] = {"vocabulary_broadcast_ms": voc_ms, "vocabulary_bytes": voc_bytes}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=1, choices=[1, 2, 4], help="index into BASELINE.json configs (1 = the headline metric)")
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=32, help="config 1: stereo pairs per pass per GPU")
    ap.add_argument("--frames", type=int, default=32, help="config 2: RGB-D frames per pass per handle")
    ap.add_argument("--keyframes", type=int, default=2000, help="config 4: keyframes in the resident database")
    ap.add_argument("--queries", type=int, default=8, help="config 4: distinct query frames")
    ap.add_argument("--handles", type=int, default=None, help="batches / query streams in flight per GPU (one CUDA stream / host thread each); default: config 1 -> 6, configs 2 and 4 -> 8")
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--cpu-items-per-thread", type=int, default=8)
    ap.add_argument("--ref-items-per-thread", type=int, default=4)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--per-frame-calls", action="store_true", help="config 2: one borb_search_by_projection call per frame instead of the batched call")
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the arrays the timed call returned in its last pass to DIR/<name>.npy")
    args = ap.parse_args()
    if args.dump_outputs and args.per_frame_calls:
        ap.error("--dump-outputs reads the batched matcher call's results; it cannot be combined with --per-frame-calls")
    if args.handles is None:
        args.handles = {1: 6, 2: 8, 4: 8}.get(args.config, 4)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, rank)
        return
    env = Env(rank, world, local_rank)
    {1: run_config1, 2: run_config2, 4: run_config4}[args.config](args, env)
    env.finish()


if __name__ == "__main__":
    main()
