"""Catalogue of the poisoned-memory check (tests/test_gpu_poison.py): one case builder per entry point that launches a kernel or fills
a buffer the library reuses or recycles, and the table that maps every BORB_API name of include/borb.h to the cases that drive it
(COVERED) or to the reason it needs none (NOT_COVERED).

A case is a function of the shared handles (Ctx) that runs its calls and returns every output it got - nested tuples, lists, dicts,
dataclasses and arrays, flattened by outputs() - cut to the extent the API defines (n keypoints of cap, n_left stereo entries, ...).
Within a family, CASES runs a larger case before the smaller ones, so that the grow-only buffers are bigger than the later calls
need.  The inputs come from the existing fixture modules; the GPU import happens only when a case runs.  Test tooling."""
import ctypes as C
import dataclasses

import numpy as np

from tests import frame_input_cases as fic
from tests import match_fixtures as mf
from orb_slam2_b200 import synth

BF, FX = mf.BF, mf.FX
B = np.float32(BF) / np.float32(FX)
LEVELSUP = 2
K_CAM = (525.0, 525.0, 319.5, 239.5)


# ---------------------------------------------------------------------------------------------------------- flattening
def outputs(obj, prefix="out"):
    """{path: (dtype, shape, bytes)} of every array or scalar inside obj."""
    out = {}

    def walk(o, p):
        if o is None:
            out[p] = ("none", (), b"")
        elif isinstance(o, np.ndarray):
            a = np.ascontiguousarray(o)
            out[p] = (str(a.dtype), a.shape, a.tobytes())
        elif isinstance(o, dict):
            for k in sorted(o, key=str):
                walk(o[k], f"{p}.{k}")
        elif isinstance(o, (list, tuple)):
            for i, x in enumerate(o):
                walk(x, f"{p}[{i}]")
        elif dataclasses.is_dataclass(o):
            for f in dataclasses.fields(o):
                if not f.name.startswith("_") and f.name != "resident":
                    walk(getattr(o, f.name), f"{p}.{f.name}")
        elif isinstance(o, (bool, int, float, np.generic, str)):
            a = np.asarray(o)
            out[p] = (str(a.dtype), a.shape, a.tobytes())
        else:
            raise TypeError(f"{p}: cannot flatten {type(o)}")
    walk(obj, prefix)
    return out


def take(view, sel):
    """The per-point view (MapPointsView / WorldPointsView / LastFrameView) restricted to the points sel."""
    return dataclasses.replace(view, **{f.name: getattr(view, f.name)[sel] for f in dataclasses.fields(view)
                                        if isinstance(getattr(view, f.name), np.ndarray)})


# ---------------------------------------------------------------------------------------------------------- shared handles
class Ctx:
    """One matcher, one vocabulary and two extractors for the whole catalogue (handles, and so their grow-only buffers, live across
    every pass), plus the fixture inputs."""

    def __init__(self, oracle):
        from orb_slam2_b200 import matcher as M, sharding, _lib
        from orb_slam2_b200.extractor import ORBextractor
        self.M, self.lib = M, _lib
        self.mt = M.ORBmatcher(0.75, True)
        self.voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
        self.XA, self.XB = ORBextractor(1000), ORBextractor(1200)
        self.XR = ORBextractor(1000)                                # rectified input: its maps stay installed
        w, h = 640, 480
        self.XR.set_rectify_maps(0, *fic.radial_rectify_maps((w, h), (w, h)), src_size=(w, h))
        self.big = mf.two_views(oracle, 5, (752, 480), 1500)
        self.small = mf.two_views(oracle, 6, (320, 240), 300)
        self.pairs = [synth.stereo_pair(40 + i, 0, 0, w, h)[:2] for i in range(3)]
        self.mono = [synth.mono_frame(50 + i, 0, 0, w, h) for i in range(4)]

    def close(self):
        for x in (self.mt, self.voc, self.XA, self.XB, self.XR):
            x.close()


def _debug(X, images, levels=8):
    """The extractor intermediates of the last batch: pyramid, blurred levels, candidates (sorted: fast_kernel appends them in no
    fixed order) and selected points."""
    def cand(l, i):
        c = X.debug_candidates(l, i)
        return c[np.lexsort(c.T[::-1])] if len(c) else c
    return {f"img{i}": dict(pyr=[X.pyramid(l, i) for l in range(levels)], blur=[X.debug_blurred(l, i) for l in range(levels)],
                            cand=[cand(l, i) for l in range(levels)], sel=[X.debug_selected(l, i) for l in range(levels)])
            for i in images}


# ---------------------------------------------------------------------------------------------------------- extractor
def ex_batch(c):
    """borb_extract_batch of 4 images, then the debug readers (the largest extraction: it runs first)."""
    out = c.XA.extract_batch(c.mono)
    return dict(res=out, dbg=_debug(c.XA, (0, 3)))


def ex_single(c):
    """borb_extract of one image after a 4-image batch."""
    return c.XA(c.mono[1])


def _enqueue(c, X, imgs, device=False):
    lib = c.lib
    so = lib.load()
    n, (h, w) = len(imgs), imgs[0].shape
    cap = X.capacity(w, h)
    kps = np.zeros((n, cap), lib.KP_DTYPE); desc = np.zeros((n, cap, 32), np.uint8); cnt = np.zeros(n, np.int32)
    if device:
        import torch
        d = torch.from_numpy(np.stack(imgs)).cuda()
        torch.cuda.synchronize()
        lib.check(so.borb_extract_batch_device(X._h, d.data_ptr(), n, w, h, w, w * h, lib.ptr(kps), lib.ptr(desc), cap, lib.ptr(cnt)),
                  "borb_extract_batch_device")
    else:
        imgs = [np.ascontiguousarray(i) for i in imgs]
        ptrs = (C.c_void_p * n)(*[i.ctypes.data for i in imgs])
        lib.check(so.borb_extract_batch_enqueue(X._h, ptrs, n, w, h, w, lib.ptr(kps), lib.ptr(desc), cap, lib.ptr(cnt)),
                  "borb_extract_batch_enqueue")
        lib.check(so.borb_sync(X._h), "borb_sync")
    X._last_n = n
    return [(kps[i, :cnt[i]].copy(), desc[i, :cnt[i]].copy()) for i in range(n)]


def ex_enqueue(c):
    """borb_extract_batch_enqueue + borb_sync of two scattered host images."""
    return _enqueue(c, c.XA, c.mono[2:4])


def ex_device(c):
    """borb_extract_batch_device of three device images, with the intermediates of the last one."""
    out = _enqueue(c, c.XA, c.mono[:3], device=True)
    return dict(res=out, dbg=_debug(c.XA, (2,)))


def ex_color(c):
    """RGB and BGRA host images (the converting upload)."""
    rgb = np.repeat(c.mono[0][:, :, None], 3, 2).copy(); rgb[:, :, 1] //= 2
    bgra = np.concatenate([rgb[:, :, ::-1], np.full(rgb.shape[:2] + (1,), 255, np.uint8)], 2)
    a = c.XA.extract_batch([rgb, rgb[::-1].copy()])
    c.XA.set_input_format(4, False)
    b = c.XA.extract_batch([bgra])
    c.XA.set_input_format(1)
    return dict(rgb=a, bgra=b)


def ex_rectified(c):
    """Raw frames rectified while they are uploaded (maps installed on XR), 3 images then 1."""
    a = c.XR.extract_batch(c.mono[:3])
    b = c.XR.extract_batch(c.mono[3:])
    return dict(a=a, b=b, dbg=_debug(c.XR, (0,)))


# ---------------------------------------------------------------------------------------------------------- stereo
def st_frames(c):
    """borb_stereo_frames of 3 pairs, then borb_stereo_match on the same extraction (default layout and index arrays)."""
    res = c.XA.stereo_frames([p[0] for p in c.pairs], [p[1] for p in c.pairs], BF, FX)
    nl = [len(r["mvKeys"]) for r in res]
    ur, dp = c.XA.stereo_match(3, BF, FX)
    ur2, dp2 = c.XA.stereo_match(2, BF, FX, left_idx=[2, 0], right_idx=[3, 1])
    return dict(res=res, match=[(ur[p, :nl[p]], dp[p, :nl[p]]) for p in range(3)],
                match_idx=[(ur2[0, :nl[1]], dp2[0, :nl[1]]), (ur2[1, :nl[0]], dp2[1, :nl[0]])])


def _stereo_c(c, X, pairs, device):
    lib = c.lib
    so = lib.load()
    n = len(pairs)
    h, w = pairs[0][0].shape
    cap = X.capacity(w, h)
    nl = np.zeros(n, np.int32); nr = np.zeros(n, np.int32)
    ur = np.zeros((n, cap), np.float32); dp = np.zeros((n, cap), np.float32)
    if device:
        import torch
        d = torch.from_numpy(np.stack([im for p in pairs for im in p])).cuda()
        torch.cuda.synchronize()
        lib.check(so.borb_stereo_frames_device(X._h, d.data_ptr(), n, w, h, w, w * h, BF, float(B), lib.ptr(nl), lib.ptr(nr),
                                               lib.ptr(ur), lib.ptr(dp), cap), "borb_stereo_frames_device")
    else:
        L = [np.ascontiguousarray(p[0]) for p in pairs]; R = [np.ascontiguousarray(p[1]) for p in pairs]
        pl = (C.c_void_p * n)(*[i.ctypes.data for i in L]); pr = (C.c_void_p * n)(*[i.ctypes.data for i in R])
        lib.check(so.borb_stereo_frames_enqueue(X._h, pl, pr, n, w, h, w, BF, float(B), None, None, lib.ptr(nl), None, None,
                                                lib.ptr(nr), lib.ptr(ur), lib.ptr(dp), cap), "borb_stereo_frames_enqueue")
        lib.check(so.borb_sync(X._h), "borb_sync")
    X._last_n = 2 * n
    kl = np.zeros((n, cap), lib.KP_DTYPE); dl = np.zeros((n, cap, 32), np.uint8); kr = np.zeros((n, cap), lib.KP_DTYPE)
    dr = np.zeros((n, cap, 32), np.uint8); nl2 = np.zeros(n, np.int32); nr2 = np.zeros(n, np.int32)
    ur2 = np.zeros((n, cap), np.float32); dp2 = np.zeros((n, cap), np.float32)
    lib.check(so.borb_stereo_frames_results(X._h, n, lib.ptr(kl), lib.ptr(dl), lib.ptr(nl2), lib.ptr(kr), lib.ptr(dr), lib.ptr(nr2),
                                            lib.ptr(ur2), lib.ptr(dp2), cap), "borb_stereo_frames_results")
    return [dict(nl=nl[p], nr=nr[p], ur=ur[p, :nl[p]], dp=dp[p, :nl[p]], kl=kl[p, :nl2[p]], dl=dl[p, :nl2[p]], kr=kr[p, :nr2[p]],
                 dr=dr[p, :nr2[p]], ur2=ur2[p, :nl2[p]], dp2=dp2[p, :nl2[p]]) for p in range(n)]


def st_device(c):
    """borb_stereo_frames_device of 2 pairs, read back with borb_stereo_frames_results."""
    return _stereo_c(c, c.XA, c.pairs[:2], True)


def st_enqueue(c):
    """borb_stereo_frames_enqueue + borb_sync of 1 pair, read back with borb_stereo_frames_results."""
    return _stereo_c(c, c.XA, c.pairs[2:], False)


def st_match2(c):
    """borb_stereo_match2: left image on XA, right image on XB (more features)."""
    lib = c.lib
    L, R = c.pairs[0]
    (kl, dl), = c.XA.extract_batch([L])
    (kr, dr), = c.XB.extract_batch([R])
    cap = c.XA.capacity(*L.shape[::-1])
    ur = np.zeros(cap, np.float32); dp = np.zeros(cap, np.float32)
    lib.check(lib.load().borb_stereo_match2(c.XA._h, c.XB._h, BF, float(B), lib.ptr(ur), lib.ptr(dp), cap), "borb_stereo_match2")
    return dict(kl=kl, kr=kr, ur=ur[:len(kl)], dp=dp[:len(kl)])


# ---------------------------------------------------------------------------------------------------------- frames from the extractor
def _read(frames, stereo):
    out = [F.resident.read(stereo=stereo) for F in frames]
    for F in frames:
        F.resident.close()
    return out


def fx_mono(c):
    """borb_frames_from_extractor, monocular, of a 4-image batch (distorted camera)."""
    res = c.XA.extract_batch(c.mono)
    K, dist = fic.DIST_CASES["tum1_5"]
    frames, host = c.M.frames_from_extractor(c.mt, c.XA, [3, 0, 2], [len(res[i][0]) for i in (3, 0, 2)], K, dist)
    return dict(host=host, dev=_read(frames, False))


def fx_stereo(c):
    """borb_frames_from_extractor, stereo, after borb_stereo_frames of 3 pairs."""
    res = c.XA.stereo_frames([p[0] for p in c.pairs], [p[1] for p in c.pairs], BF, FX)
    frames, host = c.M.frames_from_extractor(c.mt, c.XA, [0, 4], [len(res[0]["mvKeys"]), len(res[2]["mvKeys"])], K_CAM, bf=BF, mode=1)
    return dict(host=host, dev=_read(frames, True))


def fx_rgbd(c):
    """borb_frames_from_extractor, RGB-D, host float and raw depth maps."""
    res = c.XA.extract_batch(c.mono[:2])
    K, dist = fic.DIST_CASES["tum1_5"]
    nk = [len(r[0]) for r in res]
    a, ha = c.M.frames_from_extractor(c.mt, c.XA, [0, 1], nk, K, dist, bf=40.0, mode=2, depth=[fic.edge_depth_float(21 + i) for i in range(2)])
    b, hb = c.M.frames_from_extractor(c.mt, c.XA, [1], nk[1:], K, dist, bf=40.0, mode=2, depth=[fic.edge_depth_raw(23)],
                                      depth_factor=1.0 / 5000.0)
    return dict(ha=ha, hb=hb, a=_read(a, True), b=_read(b, True))


# ---------------------------------------------------------------------------------------------------------- matcher
def _res(c, F):
    return F.make_resident(c.mt)


def mt_frame_create(c):
    """borb_frame_create in pool order: an 8192-feature frame is released, then a 1000-feature stereo frame and a monocular frame take
    recycled blocks.  A frame made from a view has mvuRight but no mvDepth: its depth read is refused (BORB_ERR_INVALID_ARG)."""
    rng = np.random.default_rng(3)
    from orb_slam2_b200._lib import KP_DTYPE, BorbError
    k = np.zeros(8192, KP_DTYPE)
    k["x"] = rng.uniform(0, 752, 8192); k["y"] = rng.uniform(0, 480, 8192); k["octave"] = rng.integers(0, 8, 8192); k["class_id"] = -1
    d = rng.integers(0, 256, (8192, 32), dtype=np.uint8)
    v = c.big
    big = _res(c, c.M.FrameView(k, d, v["scale"], (0.0, 0.0, 752.0, 480.0)))
    r_big = big.resident.read(stereo=False)
    big.resident.close()
    st = _res(c, c.M.FrameView(v["kl"][:1000], v["dl"][:1000], v["scale"], (0.0, 0.0, 752.0, 480.0), mvuRight=v["ur"][:1000]))
    mono = _res(c, c.M.FrameView(v["kr"][:700], v["dr"][:700], v["scale"], (0.0, 0.0, 752.0, 480.0)))
    lib = c.lib
    ur = np.zeros(1000, np.float32); dp = np.zeros(1000, np.float32)
    lib.check(lib.load().borb_debug_frame_read(st.resident._h, None, None, lib.ptr(ur), None, None, None), "borb_debug_frame_read")
    depth_status = lib.load().borb_debug_frame_read(st.resident._h, None, None, None, lib.ptr(dp), None, None)
    out = dict(big=r_big, stereo=st.resident.read(stereo=False), ur=ur, depth_status=np.int32(depth_status),
               mono=mono.resident.read(stereo=False))
    st.resident.close(); mono.resident.close()
    return out


def mt_projection(c):
    """borb_search_by_projection on a host view and on a resident frame, then borb_search_by_projection_batch with a large, a small
    and an empty job."""
    F, mps = mf.projection_case(c.big, 11, n_mp=1200)
    Fs, mpss = mf.projection_case(c.small, 12, n_mp=200)
    a = c.mt.SearchByProjection(F, mps, 3.0)
    R, Rs = _res(c, F), _res(c, Fs)
    b = c.mt.SearchByProjection(R, mps, 3.0)
    bb = c.mt.SearchByProjectionBatch([R, Rs, Rs], [mps, mpss, take(mpss, slice(0, 0))], 3.0)
    s = c.mt.SearchByProjection(Fs, mpss, 5.0)
    R.resident.close(); Rs.resident.close()
    return dict(a=a, b=b, batch=bb, s=s)


def mt_last(c):
    """borb_search_by_projection_last (host view, resident) and its batch with an empty LastFrame job."""
    Cur, Last, Tcw, K = mf.last_frame_case(c.big, 13)
    Cs, Ls, Ts, Ks = mf.last_frame_case(c.small, 14)
    a = c.mt.SearchByProjectionLast(Cur, Last, Tcw, K, 40.0, 15.0)
    R, Rs = _res(c, Cur), _res(c, Cs)
    bb = c.mt.SearchByProjectionLastBatch([R, Rs, Rs], [Last, Ls, take(Ls, slice(0, 0))], [Tcw, Ts, Ts], K, 40.0, 7.0)
    s = c.mt.SearchByProjectionLast(Rs, Ls, Ts, Ks, 40.0, 7.0)
    R.resident.close(); Rs.resident.close()
    return dict(a=a, batch=bb, s=s)


def mt_kf_sim3proj(c):
    """borb_search_by_projection_kf / _sim3 (host views) and their batches on resident frames, with an empty points job."""
    F, P, Tcw, Ow, K = mf.world_points_case(c.big, 15)
    Fs, Ps, Ts, Os, _ = mf.world_points_case(c.small, 16)
    a = c.mt.SearchByProjectionKF(F, P, Tcw, Ow, K, 10.0, 100)
    b = c.mt.SearchByProjectionSim3(F, P, Tcw, Ow, K, 10)
    R, Rs = _res(c, F), _res(c, Fs)
    e = take(Ps, slice(0, 0))
    kb = c.mt.SearchByProjectionKFBatch([R, Rs, Rs], [P, Ps, e], [(Tcw, Ow), (Ts, Os), (Ts, Os)], K, 3.0, 64)
    sb = c.mt.SearchByProjectionSim3Batch([R, Rs, Rs], [P, Ps, e], [(Tcw, Ow), (Ts, Os), (Ts, Os)], K, 10)
    s = c.mt.SearchByProjectionKF(Fs, Ps, Ts, Os, K, 3.0, 64)
    R.resident.close(); Rs.resident.close()
    return dict(a=a, b=b, kb=kb, sb=sb, s=s)


def mt_local_points(c):
    """borb_search_local_points (host view) and its batch, with an empty points job."""
    F, P, Tcw, Ow, K = mf.world_points_case(c.big, 17)
    Fs, Ps, Ts, Os, _ = mf.world_points_case(c.small, 18)
    F = dataclasses.replace(F, mvuRight=c.big["ur"])
    a = c.mt.SearchLocalPoints(F, P, Tcw, Ow, K, 40.0, 3.0)
    R, Rs = _res(c, F), _res(c, Fs)
    bb = c.mt.SearchLocalPointsBatch([R, Rs, Rs], [P, Ps, take(Ps, slice(0, 0))], [(Tcw, Ow), (Ts, Os), (Ts, Os)], K, 40.0, 1.0)
    s = c.mt.SearchLocalPoints(Fs, Ps, Ts, Os, K, 40.0, 5.0)
    R.resident.close(); Rs.resident.close()
    return dict(a=a, batch=bb, s=s)


def mt_fuse(c):
    """borb_fuse, both overloads, and borb_fuse_batch with both mixed and an empty job."""
    KF, P, Tcw, Ow, K, bf = mf.fuse_case(c.big, 19)
    KFs, Ps, Ts, Os, _, _ = mf.fuse_case(c.small, 20)
    a = c.mt.Fuse(KF, P, Tcw, Ow, K, bf, 3.0, Scw=False)
    b = c.mt.Fuse(KF, P, Tcw, Ow, K, bf, 3.0, Scw=True)
    R, Rs = _res(c, KF), _res(c, KFs)
    e = take(Ps, slice(0, 0))
    f0 = c.mt.FuseBatch([R, Rs, Rs], [P, Ps, e], [(Tcw, Ow), (Ts, Os), (Ts, Os)], K, bf, 3.0, Scw=False)
    f1 = c.mt.FuseBatch([Rs, R], [Ps, P], [(Ts, Os), (Tcw, Ow)], K, bf, 5.0, Scw=True)
    s = c.mt.Fuse(KFs, Ps, Ts, Os, K, bf, 3.0, Scw=False)
    R.resident.close(); Rs.resident.close()
    return dict(a=a, b=b, f0=f0, f1=f1, s=s)


def mt_sim3(c):
    """borb_search_by_sim3 (host views) and borb_search_by_sim3_batch (a keyframe with itself as well)."""
    KF1, KF2, P1, P2, T1, T2, S12, S21, K = mf.sim3_case(c.big, 21)
    k1, k2, p1, p2, t1, t2, s12, s21, _ = mf.sim3_case(c.small, 22)
    a = c.mt.SearchBySim3(KF1, KF2, P1, P2, T1, T2, S12, S21, K, 7.5)
    R1, R2, r1, r2 = _res(c, KF1), _res(c, KF2), _res(c, k1), _res(c, k2)
    bb = c.mt.SearchBySim3Batch([R1, r1, r1], [R2, r2, r1], [P1, p1, p1], [P2, p2, p1], [(T1, T2), (t1, t2), (t1, t1)],
                                [(S12, S21), (s12, s21), (s12, s21)], K, 7.5)
    s = c.mt.SearchBySim3(k1, k2, p1, p2, t1, t2, s12, s21, K, 7.5)
    for R in (R1, R2, r1, r2):
        R.resident.close()
    return dict(a=a, batch=bb, s=s)


def mt_init(c):
    """borb_search_for_initialization (host views) and its batch on resident frames, a 0-feature current frame included."""
    v, vs = c.big, c.small
    bnd = (0.0, 0.0, float(v["w"]), float(v["h"]))
    F1 = c.M.FrameView(v["kl"], v["dl"], v["scale"], bnd)
    F2 = c.M.FrameView(v["kr"], v["dr"], v["scale"], bnd)
    f1 = c.M.FrameView(vs["kl"], vs["dl"], vs["scale"], (0.0, 0.0, 320.0, 240.0))
    f2 = c.M.FrameView(vs["kr"], vs["dr"], vs["scale"], (0.0, 0.0, 320.0, 240.0))
    empty = c.M.FrameView(vs["kr"][:0], vs["dr"][:0], vs["scale"], (0.0, 0.0, 320.0, 240.0))
    prev = np.stack([v["kl"]["x"], v["kl"]["y"]], 1).astype(np.float32)
    prevs = np.stack([vs["kl"]["x"], vs["kl"]["y"]], 1).astype(np.float32)
    a = c.mt.SearchForInitialization(F1, F2, prev, 100)
    R1, R2, r1, r2, re = _res(c, F1), _res(c, F2), _res(c, f1), _res(c, f2), _res(c, empty)
    bb = c.mt.SearchForInitializationBatch([R1, r1, r1], [R2, r2, re], [prev, prevs, prevs], 100)
    s = c.mt.SearchForInitialization(f1, f2, prevs, 50)
    for R in (R1, R2, r1, r2, re):
        R.resident.close()
    return dict(a=a, batch=bb, s=s)


def mt_distinctive(c):
    """borb_distinctive_descriptors and borb_distinctive_descriptors_frames, with points of 0, 1 and many observations."""
    rng = np.random.default_rng(23)
    v = c.big
    groups = [v["dl"][rng.integers(0, len(v["dl"]), n)] for n in (0, 1, 2, 7, 40)] * 30
    a = c.mt.ComputeDistinctiveDescriptors(groups)
    bnd = (0.0, 0.0, float(v["w"]), float(v["h"]))
    frames = [_res(c, c.M.FrameView(v["kl"], v["dl"], v["scale"], bnd)), _res(c, c.M.FrameView(v["kr"], v["dr"], v["scale"], bnd))]
    g = []
    for n in (0, 1, 3, 9, 25) * 20:
        fi = rng.integers(0, 2, n)
        g.append((fi, np.array([rng.integers(0, frames[f].resident.n) for f in fi], np.int32)))
    b = c.mt.ComputeDistinctiveDescriptorsFrames(frames, g)
    s = c.mt.ComputeDistinctiveDescriptors(groups[:5])
    for F in frames:
        F.resident.close()
    return dict(a=a, b=b, s=s)


def _kfs(c, v, seed):
    return mf.keyframe_views(v, c.voc, seed, LEVELSUP)


def mt_bow(c):
    """borb_search_by_bow (2 keyframes against a frame), borb_search_by_bow_kf, and borb_search_by_bow_batch on resident frames."""
    k1, k2 = _kfs(c, c.big, 24)
    s1, s2 = _kfs(c, c.small, 25)
    a = c.mt.SearchByBoW([k1, k2], k2)
    b = c.mt.SearchByBoW_KF(k1, k2)
    v, vs = c.big, c.small
    F = _res(c, c.M.FrameView(v["kr"], v["dr"], v["scale"], (0.0, 0.0, float(v["w"]), float(v["h"]))))
    Fs = _res(c, c.M.FrameView(vs["kr"], vs["dr"], vs["scale"], (0.0, 0.0, 320.0, 240.0)))
    c.mt.ComputeBoWBatch(c.voc, [F, Fs], LEVELSUP, want_host=False)
    bb = c.mt.SearchByBoWBatch([k1, s1, s1], [F, Fs, F])
    s = c.mt.SearchByBoW_KF(s1, s2)
    F.resident.close(); Fs.resident.close()
    return dict(a=a, b=b, batch=bb, s=s)


def mt_triangulation(c):
    """borb_search_for_triangulation and its batch (host views and resident keyframes with BoW)."""
    k1, k2 = _kfs(c, c.big, 26)
    s1, s2 = _kfs(c, c.small, 27)
    F12 = mf.rectified_F12(28)
    a = c.mt.SearchForTriangulation(k1, k2, F12, (300.0, 240.0), False)
    v = c.big
    bnd = (0.0, 0.0, float(v["w"]), float(v["h"]))
    R1 = _res(c, c.M.FrameView(v["kl"], v["dl"], v["scale"], bnd, mvuRight=v["ur"]))
    c.mt.ComputeBoWBatch(c.voc, [R1], LEVELSUP, want_host=False)
    R1 = dataclasses.replace(R1, has_mp=k1.has_mp)
    bb = c.mt.SearchForTriangulationBatch([R1, s1, s1], [k2, s2, s2], [F12] * 3, [(300.0, 240.0), (160.0, 120.0), (160.0, 120.0)],
                                          [False, False, True])
    s = c.mt.SearchForTriangulation(s1, s2, F12, (160.0, 120.0), True)
    R1.resident.close()
    return dict(a=a, batch=bb, s=s)


# ---------------------------------------------------------------------------------------------------------- vocabulary
def voc_bow(c):
    """borb_bow_transform and borb_compute_bow on 1500 and 300 descriptors, and borb_frames_compute_bow of three resident frames
    (one without features)."""
    v, vs = c.big, c.small
    a = [c.voc.transform_raw(d, 4) for d in (v["dl"], vs["dl"])]
    b = [c.voc.ComputeBoW(d, LEVELSUP) for d in (v["dl"], vs["dl"])]
    fr = [_res(c, c.M.FrameView(x["kl"][:n], x["dl"][:n], x["scale"], (0.0, 0.0, 752.0, 480.0))) for x, n in ((v, None), (vs, None), (vs, 0))]
    bb = c.mt.ComputeBoWBatch(c.voc, fr, LEVELSUP)
    for F in fr:
        F.resident.close()
    return dict(a=a, b=b, batch=bb)


# ---------------------------------------------------------------------------------------------------------- keyframe database
def kfdb(c):
    """The keyframe database: borb_kfdb_add of host views, borb_kfdb_add_frames of resident frames, borb_kfdb_set_has_mp (single and
    batch), borb_kfdb_erase, every block read back; borb_kfdb_query and its batch; borb_search_by_bow_db, _pairs, _batch;
    borb_search_by_bow_kf_db_pairs and _batch."""
    M = c.M
    rng = np.random.default_rng(29)
    db = M.KeyFrameDatabase(c.mt)
    views = _kfs(c, c.big, 30) + _kfs(c, c.small, 31) + _kfs(c, c.small, 32)
    slots = []
    for kv in views:
        bow, fv = c.voc.ComputeBoW(kv.mDescriptors, LEVELSUP)
        slots.append(db.add(dataclasses.replace(kv, mFeatVec=fv), bow))
    v, vs = c.big, c.small
    fr = [_res(c, M.FrameView(x["kl"], x["dl"], x["scale"], (0.0, 0.0, float(x["w"]), float(x["h"])))) for x in (v, vs, v)]
    c.mt.ComputeBoWBatch(c.voc, fr, LEVELSUP, want_host=False)
    slots += c.mt.KfdbAddFramesBatch(db, fr, [None, (rng.random(vs["kl"].shape[0]) < 0.5).astype(np.uint8), np.ones(len(v["kl"]), np.uint8)])
    db.set_has_mp(slots[0], (rng.random(len(views[0].mvKeysUn)) < 0.3).astype(np.uint8))
    db.set_has_mp_batch([slots[2], slots[3], slots[2]], [(rng.random(len(views[i].mvKeysUn)) < p).astype(np.uint8) for i, p in ((2, 0.2), (3, 0.9), (2, 0.6))])
    db.erase(slots[4])
    live = [s for s in slots if s != slots[4]]
    blocks = {s: db.read_slot(s) for s in live}
    qbow, qfv = c.voc.ComputeBoW(vs["dr"], LEVELSUP)
    q = db.query(qbow)
    qb = c.mt.KfdbQueryBatch(db, [fr[0], fr[1]])
    Fq = M.KeyFrameView(mvKeysUn=vs["kr"], mDescriptors=vs["dr"], mFeatVec=qfv)
    s_db = db.SearchByBoW(live[:3], Fq)
    s_pairs = db.SearchByBoWPairs(None, Fq)
    s_batch = c.mt.SearchByBoWDbBatch(db, [None, live[1:4], []], [fr[0], fr[1], fr[1]])
    kk = db.SearchByBoWKFPairs(live[0], None)
    kkb = c.mt.SearchByBoWKFDbBatch(db, [live[1], live[5]], [live, live[:2]])
    small = db.SearchByBoWPairs([live[2]], Fq)
    for F in fr:
        F.resident.close()
    return dict(slots=slots, blocks=blocks, q=q, qb=qb, s_db=s_db, s_pairs=_blocks(s_pairs), s_batch=[_blocks(r) for r in s_batch],
                kk=_blocks(kk), kkb=[_blocks(r) for r in kkb], small=_blocks(small))


def _blocks(res):
    """(n_matches, [each keyframe's pair block]) of a compact search result: the blocks are packed in no particular order, so
    pair_offset and the placement are not results."""
    nm, off, pairs = res
    return nm, [pairs[off[k]:off[k] + nm[k]] for k in range(len(nm))]


# families in run order: within a family every case follows a larger one
CASES = {
    "ex_batch": ex_batch, "ex_device": ex_device, "ex_enqueue": ex_enqueue, "ex_single": ex_single, "ex_color": ex_color,
    "ex_rectified": ex_rectified,
    "st_frames": st_frames, "st_device": st_device, "st_enqueue": st_enqueue, "st_match2": st_match2,
    "fx_mono": fx_mono, "fx_stereo": fx_stereo, "fx_rgbd": fx_rgbd,
    "mt_frame_create": mt_frame_create, "mt_projection": mt_projection, "mt_last": mt_last, "mt_kf_sim3proj": mt_kf_sim3proj,
    "mt_local_points": mt_local_points, "mt_fuse": mt_fuse, "mt_sim3": mt_sim3, "mt_init": mt_init, "mt_distinctive": mt_distinctive,
    "mt_bow": mt_bow, "mt_triangulation": mt_triangulation,
    "voc_bow": voc_bow,
    "kfdb": kfdb,
}

_EX = ("ex_batch", "ex_device", "ex_enqueue", "ex_single", "ex_color", "ex_rectified", "st_frames", "st_device", "st_enqueue",
       "st_match2", "fx_mono", "fx_stereo", "fx_rgbd")
# BORB_API name -> the cases that drive it
COVERED = {
    "borb_extractor_create": _EX, "borb_extractor_capacity": ("ex_enqueue", "st_device", "st_match2"),
    "borb_extract": ("ex_single",), "borb_extract_batch": ("ex_batch", "ex_color", "ex_rectified", "fx_mono", "fx_rgbd"),
    "borb_extract_batch_enqueue": ("ex_enqueue",), "borb_sync": ("ex_enqueue", "st_enqueue"),
    "borb_extract_batch_device": ("ex_device",), "borb_extractor_set_input_format": ("ex_color",),
    "borb_extractor_set_rectify_maps": ("ex_rectified",), "borb_extractor_pyramid": ("ex_batch", "ex_device", "ex_rectified"),
    "borb_debug_blurred": ("ex_batch", "ex_device", "ex_rectified"), "borb_debug_candidates": ("ex_batch", "ex_device", "ex_rectified"),
    "borb_debug_selected": ("ex_batch", "ex_device", "ex_rectified"),
    "borb_stereo_match": ("st_frames",), "borb_stereo_match2": ("st_match2",), "borb_stereo_frames": ("st_frames", "fx_stereo"),
    "borb_stereo_frames_enqueue": ("st_enqueue",), "borb_stereo_frames_device": ("st_device",),
    "borb_stereo_frames_device_enqueue": ("st_device",), "borb_stereo_frames_results": ("st_device", "st_enqueue"),
    "borb_matcher_create": tuple(n for n in CASES if not n.startswith(("ex_", "st_"))),
    "borb_frame_create": ("mt_frame_create", "mt_projection", "mt_last", "mt_kf_sim3proj", "mt_local_points", "mt_fuse", "mt_sim3",
                          "mt_init", "mt_distinctive", "mt_bow", "mt_triangulation", "voc_bow", "kfdb"),
    "borb_frame_destroy": ("mt_frame_create", "mt_projection", "fx_mono", "kfdb"),
    "borb_frames_from_extractor": ("fx_mono", "fx_stereo", "fx_rgbd"), "borb_debug_frame_read": ("mt_frame_create", "fx_mono", "fx_stereo", "fx_rgbd"),
    "borb_search_by_projection": ("mt_projection",), "borb_search_by_projection_batch": ("mt_projection",),
    "borb_search_by_projection_last": ("mt_last",), "borb_search_by_projection_last_batch": ("mt_last",),
    "borb_search_by_projection_kf": ("mt_kf_sim3proj",), "borb_search_by_projection_kf_batch": ("mt_kf_sim3proj",),
    "borb_search_by_projection_sim3": ("mt_kf_sim3proj",), "borb_search_by_projection_sim3_batch": ("mt_kf_sim3proj",),
    "borb_search_local_points": ("mt_local_points",), "borb_search_local_points_batch": ("mt_local_points",),
    "borb_fuse": ("mt_fuse",), "borb_fuse_batch": ("mt_fuse",), "borb_search_by_sim3": ("mt_sim3",), "borb_search_by_sim3_batch": ("mt_sim3",),
    "borb_search_for_initialization": ("mt_init",), "borb_search_for_initialization_batch": ("mt_init",),
    "borb_distinctive_descriptors": ("mt_distinctive",), "borb_distinctive_descriptors_frames": ("mt_distinctive",),
    "borb_search_by_bow": ("mt_bow",), "borb_search_by_bow_kf": ("mt_bow",), "borb_search_by_bow_batch": ("mt_bow",),
    "borb_search_for_triangulation": ("mt_triangulation",), "borb_search_for_triangulation_batch": ("mt_triangulation",),
    "borb_voc_create": ("voc_bow",), "borb_bow_transform": ("voc_bow",), "borb_compute_bow": ("voc_bow", "mt_bow", "kfdb"),
    "borb_frames_compute_bow": ("voc_bow", "mt_bow", "mt_triangulation", "kfdb"),
    "borb_kfdb_create": ("kfdb",), "borb_kfdb_add": ("kfdb",), "borb_kfdb_add_frames": ("kfdb",), "borb_kfdb_set_has_mp": ("kfdb",),
    "borb_kfdb_set_has_mp_batch": ("kfdb",), "borb_kfdb_erase": ("kfdb",), "borb_kfdb_size": ("kfdb",), "borb_kfdb_query": ("kfdb",),
    "borb_kfdb_query_batch": ("kfdb",), "borb_search_by_bow_db": ("kfdb",), "borb_search_by_bow_db_pairs": ("kfdb",),
    "borb_search_by_bow_db_batch": ("kfdb",), "borb_search_by_bow_kf_db_pairs": ("kfdb",), "borb_search_by_bow_kf_db_batch": ("kfdb",),
    "borb_debug_kfdb_read": ("kfdb",),
}

# BORB_API name -> why no poison case drives it
NOT_COVERED = {
    "borb_last_error": "status text, no device memory",
    "borb_status_str": "status text, no device memory",
    "borb_version": "a constant",
    "borb_device_count": "queries the driver only",
    "borb_host_alloc": "returns caller-owned pinned memory, which the library neither reuses nor reads",
    "borb_host_free": "releases caller-owned pinned memory",
    "borb_extractor_destroy": "lifecycle: releases the handle",
    "borb_matcher_destroy": "lifecycle: releases the handle",
    "borb_voc_destroy": "lifecycle: releases the handle",
    "borb_kfdb_destroy": "lifecycle: releases the handle",
    "borb_kfdb_clear": "lifecycle: frees every block; the next add allocates and fills a new one, which kfdb covers",
    "borb_extractor_tables": "host copies of the constructor tables, no device memory",
    "borb_extractor_reserve": "pure configuration: allocates the workspace that the extraction cases then fill and rewrite",
    "borb_frame_info": "host fields of the frame, no device memory",
    "borb_voc_load_text": "parses a file into the same blob borb_voc_create builds; the blob is immutable after creation",
    "borb_voc_blob": "returns the address of the immutable blob",
    "borb_voc_from_blob": "adopts a caller blob, immutable afterwards; its buffers are those borb_voc_create gives, which voc_bow covers",
    "borb_nccl_unique_id": "NCCL entry point: needs two GPUs and libnccl",
    "borb_nccl_comm_create": "NCCL entry point: needs two GPUs and libnccl",
    "borb_nccl_comm_destroy": "NCCL entry point: needs two GPUs and libnccl",
    "borb_voc_broadcast": "NCCL entry point: needs two GPUs and libnccl",
    "borb_matcher_set_timing": "timing switch: CUDA events only",
    "borb_matcher_last_kernel_ms": "timing readout",
    "borb_matcher_launch_count": "launch counter",
    "borb_launch_count": "launch counter",
    "borb_stage_times": "timing readout",
    "borb_stage_times_total": "timing readout",
    "borb_set_timing": "timing switch: CUDA events only",
    "borb_extractor_stream": "returns the handle's stream",
    "borb_debug_set_fast_mode": "ablation switch of fast_kernel; only mode 0 produces keypoints",
    "borb_debug_brief_slots": "host table, no device memory",
    "borb_debug_eval_math": "allocates fresh buffers per call and writes every output element (tests/test_gpu_device_math.py)",
    "borb_debug_set_poison": "the switch itself (tests/test_poison_catalogue.py checks its arguments)",
}
