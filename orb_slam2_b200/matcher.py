"""Host-side mirror of ORB_SLAM2::ORBmatcher (reference include/ORBmatcher.h:37-102) and ORBVocabulary over libborb.

The reference methods walk pointer graphs (Frame, KeyFrame, MapPoint); here their inputs are plain snapshots
(`FrameView`, `MapPointsView`, `KeyFrameView`) — exactly what the C++ adapter builds on the calling thread before it
calls the C ABI — and results are indices instead of MapPoint pointers.  Same method names, argument meaning and
thresholds as the reference; all compute happens in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import KP_DTYPE, check

TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 50, 30        # src/ORBmatcher.cc:37-39
BORB_ERR_CAPACITY = 5


class _FrameViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys_un", C.c_void_p), ("desc", C.c_void_p), ("u_right", C.c_void_p), ("occupied", C.c_void_p),
                ("min_x", C.c_float), ("min_y", C.c_float), ("max_x", C.c_float), ("max_y", C.c_float), ("n_levels", C.c_int32),
                ("scale_factors", C.c_void_p), ("resident", C.c_void_p)]


class _MapPointViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("proj_x", C.c_void_p), ("proj_y", C.c_void_p), ("proj_xr", C.c_void_p), ("level", C.c_void_p),
                ("view_cos", C.c_void_p), ("desc", C.c_void_p), ("valid", C.c_void_p), ("has_obs", C.c_void_p)]


class _LastFrameViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys_un", C.c_void_p), ("world_pos", C.c_void_p), ("desc", C.c_void_p), ("valid", C.c_void_p),
                ("has_obs", C.c_void_p)]


class _WorldPointsViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("world_pos", C.c_void_p), ("desc", C.c_void_p), ("max_distance", C.c_void_p),
                ("min_distance", C.c_void_p), ("normal", C.c_void_p), ("angle", C.c_void_p), ("valid", C.c_void_p)]


class _FeatVecC(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("node_id", C.c_void_p), ("start", C.c_void_p), ("feat_idx", C.c_void_p)]


class _KeyFrameViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys_un", C.c_void_p), ("desc", C.c_void_p), ("has_mp", C.c_void_p), ("u_right", C.c_void_p),
                ("fv", _FeatVecC), ("n_levels", C.c_int32), ("scale_factors", C.c_void_p), ("level_sigma2", C.c_void_p)]


class _BowJobC(C.Structure):                       # borb_bow_job
    _fields_ = [("frame", C.c_void_p), ("kf", _KeyFrameViewC), ("kf_frame", C.c_void_p), ("match", C.c_void_p)]


class _TriangulationJobC(C.Structure):             # borb_triangulation_job
    _fields_ = [("kf1", _KeyFrameViewC), ("kf1_frame", C.c_void_p), ("kf2", _KeyFrameViewC), ("kf2_frame", C.c_void_p), ("F12", C.c_float * 9),
                ("ex", C.c_float), ("ey", C.c_float), ("only_stereo", C.c_int32), ("pairs", C.c_void_p), ("cap", C.c_int32), ("n_pairs", C.c_void_p)]


class _FuseJobC(C.Structure):                      # borb_fuse_job
    _fields_ = [("kf", _FrameViewC), ("inv_level_sigma2", C.c_void_p), ("pts", _WorldPointsViewC), ("Tcw", C.c_float * 12), ("Ow", C.c_float * 3)] + \
               [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "bf", "log_scale_factor", "th")] + \
               [("scw_variant", C.c_int32), ("best_idx", C.c_void_p)]


class _KfdbQueryJobC(C.Structure):                  # borb_kfdb_query_job
    _fields_ = [("db", C.c_void_p), ("frame", C.c_void_p), ("common_words", C.c_void_p), ("score", C.c_void_p), ("first_word", C.c_void_p),
                ("cap", C.c_int32), ("n_slots", C.c_void_p)]


class _KfdbAddJobC(C.Structure):                    # borb_kfdb_add_job
    _fields_ = [("db", C.c_void_p), ("frame", C.c_void_p), ("has_mp", C.c_void_p), ("slot_out", C.c_void_p)]


class _BowRefC(C.Structure):                        # borb_bow_ref
    _fields_ = [("frame", C.c_void_p), ("db", C.c_void_p), ("slot", C.c_int32)]


class _BowScoreJobC(C.Structure):                   # borb_bow_score_job
    _fields_ = [("query", _BowRefC), ("targets", C.c_void_p), ("n_targets", C.c_int32), ("score", C.c_void_p)]


class _BowDbJobC(C.Structure):                      # borb_bow_db_job
    _fields_ = [("db", C.c_void_p), ("frame", C.c_void_p), ("slots", C.c_void_p), ("n_kf", C.c_int32), ("n_matches", C.c_void_p),
                ("pair_offset", C.c_void_p), ("pairs", C.c_void_p), ("pairs_cap", C.c_int32), ("n_pairs_total", C.c_void_p)]


class _BowKfDbJobC(C.Structure):                    # borb_bow_kf_db_job
    _fields_ = [("db", C.c_void_p), ("query_slot", C.c_int32), ("slots", C.c_void_p), ("n_kf", C.c_int32), ("n_matches", C.c_void_p),
                ("pair_offset", C.c_void_p), ("pairs", C.c_void_p), ("pairs_cap", C.c_int32), ("n_pairs_total", C.c_void_p)]


class _LocalPointsJobC(C.Structure):               # borb_local_points_job
    _fields_ = [("frame", _FrameViewC), ("pts", _WorldPointsViewC), ("has_obs", C.c_void_p), ("Tcw", C.c_float * 12), ("Ow", C.c_float * 3)] + \
               [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "mbf", "log_scale_factor", "th")] + \
               [(n, C.c_void_p) for n in ("in_view", "proj_x", "proj_y", "proj_xr", "level", "view_cos", "match_feat")]


class _LastFrameJobC(C.Structure):                 # borb_last_frame_job
    _fields_ = [("cur", _FrameViewC), ("last", _LastFrameViewC), ("Tcw", C.c_float * 12)] + \
               [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "bf", "th")] + \
               [("forward", C.c_int32), ("backward", C.c_int32), ("state_cur", C.c_void_p)]


class _InitJobC(C.Structure):                      # borb_init_job
    _fields_ = [("initial", C.c_void_p), ("current", C.c_void_p), ("prev_matched", C.c_void_p), ("window_size", C.c_int32),
                ("matches12", C.c_void_p)]


class _KfProjectionJobC(C.Structure):             # borb_kf_projection_job
    _fields_ = [("cur", _FrameViewC), ("pts", _WorldPointsViewC), ("Tcw", C.c_float * 12), ("Ow", C.c_float * 3)] + \
               [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "log_scale_factor", "th")] + \
               [("orb_dist", C.c_int32), ("state_cur", C.c_void_p)]


class _Sim3ProjectionJobC(C.Structure):           # borb_sim3_projection_job
    _fields_ = [("kf", _FrameViewC), ("pts", _WorldPointsViewC), ("Tcw", C.c_float * 12), ("Ow", C.c_float * 3)] + \
               [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "log_scale_factor")] + \
               [("th", C.c_int32), ("state_kf", C.c_void_p)]


class _Sim3JobC(C.Structure):                      # borb_sim3_job
    _fields_ = [("kf1", _FrameViewC), ("kf2", _FrameViewC), ("pts1", _WorldPointsViewC), ("pts2", _WorldPointsViewC)] + \
               [(n, C.c_float * 12) for n in ("T1w", "T2w", "S12", "S21")] + \
               [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "log_scale_factor1", "log_scale_factor2", "th")] + \
               [("match12", C.c_void_p)]


def _p(a):
    return a.ctypes.data if a is not None else None


def _per_job(x, n, ndim=0):
    """A per-job sequence, or one value (of `ndim` dimensions) for every job."""
    return list(x) if np.ndim(x) > ndim else [x] * n


def _pose12(Tcw):
    return (C.c_float * 12)(*np.asarray(Tcw, np.float32)[:3, :4].reshape(12).tolist())


def _vec3(Ow):
    return (C.c_float * 3)(*np.asarray(Ow, np.float32).reshape(3).tolist())


def _c_arrays(*pairs):
    """Contiguous copies of (array, dtype) pairs; None stays None."""
    return [np.ascontiguousarray(a, dt) if a is not None else None for a, dt in pairs]


def _mappoints_c(mps: "MapPointsView"):
    """(borb_mappoint_view, arrays to keep alive)."""
    arrs = _c_arrays((mps.mTrackProjX, np.float32), (mps.mTrackProjY, np.float32), (mps.mTrackProjXR, np.float32),
                     (mps.mnTrackScaleLevel, np.int32), (mps.mTrackViewCos, np.float32), (mps.descriptors, np.uint8), (mps.valid, np.uint8),
                     (mps.has_obs, np.uint8))
    return _MapPointViewC(len(arrs[0]), *[_p(a) for a in arrs]), arrs


def _lastframe_c(Last: "LastFrameView"):
    """(borb_lastframe_view, arrays to keep alive)."""
    arrs = _c_arrays((Last.mvKeysUn, KP_DTYPE), (Last.world_pos, np.float32), (Last.descriptors, np.uint8), (Last.valid, np.uint8),
                     (Last.has_obs, np.uint8))
    return _LastFrameViewC(len(arrs[0]), *[_p(a) for a in arrs]), arrs


def _prev_matched(vbPrevMatched):
    """vbPrevMatched as an (N,2) float32 copy that the library updates in place (at least one row, so that the pointer is valid)."""
    prev = np.ascontiguousarray(np.asarray(vbPrevMatched, np.float32).reshape(-1, 2)).copy()
    return prev if len(prev) else np.zeros((1, 2), np.float32)


def _local_points_outputs(nq: int):
    """The output arrays of SearchLocalPoints for nq points (at least one entry each, so that every pointer is valid)."""
    m1 = max(nq, 1)
    return dict(in_view=np.zeros(m1, np.uint8), proj_x=np.zeros(m1, np.float32), proj_y=np.zeros(m1, np.float32),
                proj_xr=np.zeros(m1, np.float32), level=np.zeros(m1, np.int32), view_cos=np.zeros(m1, np.float32),
                match=np.full(m1, -1, np.int32))


@dataclass
class FeatureVector:
    """DBoW2::FeatureVector as CSR: node ids ascending, feature indices ascending inside a node."""
    node_id: np.ndarray          # uint32 [n_nodes]
    start: np.ndarray            # int32  [n_nodes+1]
    feat_idx: np.ndarray         # uint32

    @staticmethod
    def from_nodes(node_of_feature: np.ndarray, keep: Optional[np.ndarray] = None) -> "FeatureVector":
        """fv.addFeature(nid, i_feature) for i_feature = 0..N-1 (TemplatedVocabulary.h:1160-1163)."""
        idx = np.arange(len(node_of_feature), dtype=np.uint32)
        nodes = np.asarray(node_of_feature, np.int64)
        if keep is not None:
            idx, nodes = idx[keep], nodes[keep]
        order = np.lexsort((idx, nodes))
        nodes, idx = nodes[order], idx[order]
        uniq, first = np.unique(nodes, return_index=True)
        start = np.append(first, len(nodes)).astype(np.int32)
        return FeatureVector(uniq.astype(np.uint32), start, np.ascontiguousarray(idx, np.uint32))

    def as_dict(self) -> Dict[int, List[int]]:
        return {int(n): self.feat_idx[self.start[i]:self.start[i + 1]].tolist() for i, n in enumerate(self.node_id)}


@dataclass
class FrameView:
    """What SearchByProjection reads of a Frame (include/Frame.h)."""
    mvKeysUn: np.ndarray
    mDescriptors: np.ndarray
    mvScaleFactors: np.ndarray
    bounds: Tuple[float, float, float, float]            # mnMinX, mnMinY, mnMaxX, mnMaxY
    mvuRight: Optional[np.ndarray] = None
    occupied: Optional[np.ndarray] = None                 # mvpMapPoints[i] && Observations()>0 (or != NULL, per overload)
    mfLogScaleFactor: Optional[float] = None              # Frame::mfLogScaleFactor; default logf(mvScaleFactors[1])
    mvInvLevelSigma2: Optional[np.ndarray] = None         # only read by Fuse(pKF, vpMapPoints, th)
    resident: Optional["ResidentFrame"] = None            # device-resident copy (borb_frame): only `occupied` travels per call
    has_mp: Optional[np.ndarray] = None                   # as a reference keyframe of SearchByBoWBatch: MapPoint present && !isBad()

    def _view(self, with_ur: bool = True):
        """(ctypes view, arrays to keep alive).  With a resident frame only `occupied` is read from the host."""
        oc = np.ascontiguousarray(self.occupied, np.uint8) if self.occupied is not None else None
        sf = np.ascontiguousarray(self.mvScaleFactors, np.float32)
        if self.resident is not None:
            return _FrameViewC(0, None, None, None, _p(oc), 0.0, 0.0, 0.0, 0.0, len(sf), None, self.resident._h), [oc, sf]
        k = np.ascontiguousarray(self.mvKeysUn, KP_DTYPE); d = np.ascontiguousarray(self.mDescriptors, np.uint8)
        ur = np.ascontiguousarray(self.mvuRight, np.float32) if (with_ur and self.mvuRight is not None) else None
        return _FrameViewC(len(k), _p(k), _p(d), _p(ur), _p(oc), *[float(x) for x in self.bounds], len(sf), _p(sf), None), [k, d, ur, oc, sf]

    def make_resident(self, matcher: "ORBmatcher") -> "FrameView":
        """Uploads the frame once (borb_frame_create: keypoints, descriptors, mvuRight, feature grid) and returns a view that
        refers to the device copy."""
        import dataclasses
        return dataclasses.replace(self, resident=ResidentFrame(matcher, self))


class ResidentFrame:
    """borb_frame: a Frame's features and 64x48 grid kept in HBM across the matcher calls of one Track()."""

    def __init__(self, matcher: "ORBmatcher", F: "FrameView"):
        self._lib = _lib.load()
        fv, keep = FrameView._view(dataclass_replace_resident(F), True)
        h = C.c_void_p()
        check(self._lib.borb_frame_create(matcher._h, C.byref(fv), C.byref(h)), "borb_frame_create")
        self._h = h
        self.n = len(F.mvKeysUn)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.borb_frame_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def read(self, stereo: bool = True) -> dict:
        """borb_debug_frame_read: what the device holds for this frame — keys_un, desc, u_right / depth (stereo / RGB-D frames) and
        the feature grid flattened as cell_start[64*48 + 1], cell_idx (cell = x*48 + y, insertion order)."""
        n = self.n
        k = np.zeros(max(n, 1), KP_DTYPE); d = np.zeros((max(n, 1), 32), np.uint8)
        ur = np.zeros(max(n, 1), np.float32) if stereo else None
        dp = np.zeros(max(n, 1), np.float32) if stereo else None
        cs = np.zeros(64 * 48 + 1, np.int32); ci = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_debug_frame_read(self._h, _p(k), _p(d), _p(ur), _p(dp), _p(cs), _p(ci)), "borb_debug_frame_read")
        return dict(keys_un=k[:n], desc=d[:n], u_right=ur[:n] if stereo else None, depth=dp[:n] if stereo else None, cell_start=cs,
                    cell_idx=ci[:cs[-1]])


class _CameraC(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3", "bf")]


def frames_from_extractor(matcher: "ORBmatcher", extractor, images, n_keys, K, dist=(0, 0, 0, 0, 0), bf: float = 0.0, mode: int = 0,
                          depth=None, depth_factor: float = 1.0, want_host: bool = True, depth_on_device: bool = False):
    """borb_frames_from_extractor: the Frame constructor tail (UndistortKeyPoints, ComputeStereoFromRGBD, AssignFeaturesToGrid,
    src/Frame.cc:404-434,643-664,230-245) on the device for images of the extractor's last batch.  K = (fx, fy, cx, cy),
    dist = (k1, k2, p1, p2, k3); mode 0 mono / 1 stereo / 2 RGB-D with depth = list of (h,w) float32 (metres) or uint16 (raw) maps.
    Host maps whose rows are contiguous keep their row stride (one padded stride shared by the batch); with depth_on_device the
    maps are tightly packed CUDA tensors (float32, or int16 / uint16 holding the raw values) and are read in place.
    Returns (frames, host) where frames[i] is a FrameView bound to the resident frame and host = dict(keys_un, u_right, depth, bounds)."""
    lib = _lib.load()
    images = np.ascontiguousarray(images, np.int32); nk = np.ascontiguousarray(n_keys, np.int32)
    nf = len(images)
    d5 = list(dist) + [0.0] * (5 - len(dist))
    cam = _CameraC(*[float(x) for x in K], *[float(x) for x in d5], float(bf))
    cap = int(nk.max()) if nf else 0
    ku = np.zeros((nf, max(cap, 1)), KP_DTYPE); ur = np.full((nf, max(cap, 1)), -1, np.float32); dp = np.full((nf, max(cap, 1)), -1, np.float32)
    b4 = np.zeros(4, np.float32)
    handles = (C.c_void_p * max(nf, 1))()
    dptr, dtype_flag, stride, keep = None, 0, 0, []
    if mode == 2 and depth_on_device:
        keep = list(depth)
        assert all(d.is_cuda and d.is_contiguous() and d.element_size() == keep[0].element_size() for d in keep)
        dtype_flag = (1 if keep[0].element_size() == 2 else 0) | 4
        dptr = (C.c_void_p * nf)(*[d.data_ptr() for d in keep])
    elif mode == 2:
        dtype_flag = 1 if np.asarray(depth[0]).dtype == np.uint16 else 0
        dt = np.uint16 if dtype_flag else np.float32
        keep = [np.asarray(d) for d in depth]
        if not all(d.dtype == dt and d.strides[1] == d.itemsize and d.strides[0] == keep[0].strides[0] for d in keep):
            keep = [np.ascontiguousarray(d, dt) for d in keep]
        stride = keep[0].strides[0]
        dptr = (C.c_void_p * nf)(*[d.ctypes.data for d in keep])
    check(lib.borb_frames_from_extractor(matcher._h, extractor._h, _p(images), nf, _p(nk), C.byref(cam), int(mode), dptr, dtype_flag,
                                         float(np.float32(depth_factor)), int(stride), _p(ku) if want_host else None,
                                         _p(ur) if want_host else None, _p(dp) if want_host else None, cap, _p(b4), handles),
          "borb_frames_from_extractor")
    sf = extractor.GetScaleFactors()
    out = []
    for i in range(nf):
        rf = ResidentFrame.__new__(ResidentFrame)
        rf._lib, rf._h, rf.n = lib, C.c_void_p(handles[i]), int(nk[i])
        n = int(nk[i])
        out.append(FrameView(mvKeysUn=ku[i, :n], mDescriptors=np.zeros((n, 32), np.uint8), mvScaleFactors=sf, bounds=tuple(float(x) for x in b4),
                             mvuRight=ur[i, :n] if mode else None, resident=rf))
    return out, dict(keys_un=[ku[i, :nk[i]] for i in range(nf)], u_right=[ur[i, :nk[i]] for i in range(nf)],
                     depth=[dp[i, :nk[i]] for i in range(nf)], bounds=b4)


class _FrameHostC(C.Structure):
    _fields_ = [("cap", C.c_int32)] + [(n, C.c_void_p) for n in ("keys", "desc", "keys_right", "desc_right", "keys_un", "u_right", "depth",
                                                                  "cell_start", "cell_idx")] + \
               [("n", C.c_int32), ("n_right", C.c_int32), ("bounds", C.c_float * 4)]


def frame_from_extractors(matcher: "ORBmatcher", left, right, K, dist=(0, 0, 0, 0, 0), bf: float = 0.0, fx: Optional[float] = None,
                          mode: int = 0, depth=None, depth_factor: float = 1.0):
    """borb_frame_from_extractors: one Frame constructor after left.extract_enqueue (and right.extract_enqueue for a stereo frame,
    mode 1; mb = bf/fx as float32, src/Frame.cc:114).  mode 2 takes one (h, w) float32 (metres) or uint16 (raw) depth map.
    Returns (frame, host): frame is a FrameView bound to the resident frame, host holds every member the constructor fills —
    mvKeys, mDescriptors, mvKeysRight, mDescriptorsRight, mvKeysUn, mvuRight, mvDepth, the grid as cell_start / cell_idx
    (borb_debug_frame_read's layout) and bounds."""
    lib = _lib.load()
    w, h = left._shape()
    cap = max(left.capacity(w, h), right.capacity(w, h) if right is not None else 0, 1)
    a = dict(keys=np.zeros(cap, KP_DTYPE), desc=np.zeros((cap, 32), np.uint8), keys_right=np.zeros(cap, KP_DTYPE),
             desc_right=np.zeros((cap, 32), np.uint8), keys_un=np.zeros(cap, KP_DTYPE), u_right=np.zeros(cap, np.float32),
             depth=np.zeros(cap, np.float32), cell_start=np.zeros(64 * 48 + 1, np.int32), cell_idx=np.zeros(cap, np.int32))
    hs = _FrameHostC(cap, *[_p(a[k]) for k in ("keys", "desc", "keys_right", "desc_right", "keys_un", "u_right", "depth", "cell_start",
                                               "cell_idx")])
    d5 = list(dist) + [0.0] * (5 - len(dist))
    cam = _CameraC(*[float(x) for x in K], *[float(x) for x in d5], float(bf))
    b = float(np.float32(bf) / np.float32(fx if fx is not None else K[0]))
    dptr, dtype_flag, stride = None, 0, 0
    if mode == 2:
        dmap = np.ascontiguousarray(depth)
        dtype_flag = 1 if dmap.dtype == np.uint16 else 0
        dmap = np.ascontiguousarray(dmap, np.uint16 if dtype_flag else np.float32)
        dptr, stride = dmap.ctypes.data, dmap.strides[0]
    out = C.c_void_p()
    check(lib.borb_frame_from_extractors(matcher._h, left._h, right._h if right is not None else None, C.byref(cam), int(mode), b, dptr,
                                         dtype_flag, float(np.float32(depth_factor)), int(stride), C.byref(hs), C.byref(out)),
          "borb_frame_from_extractors")
    n, nr = hs.n, hs.n_right
    rf = ResidentFrame.__new__(ResidentFrame)
    rf._lib, rf._h, rf.n = lib, out, n
    bounds = tuple(float(x) for x in hs.bounds)
    host = dict(mvKeys=a["keys"][:n], mDescriptors=a["desc"][:n], mvKeysRight=a["keys_right"][:nr], mDescriptorsRight=a["desc_right"][:nr],
                mvKeysUn=a["keys_un"][:n], mvuRight=a["u_right"][:n], mvDepth=a["depth"][:n], cell_start=a["cell_start"],
                cell_idx=a["cell_idx"][:a["cell_start"][-1]], bounds=bounds)
    F = FrameView(mvKeysUn=host["mvKeysUn"], mDescriptors=host["mDescriptors"], mvScaleFactors=left.GetScaleFactors(), bounds=bounds,
                  mvuRight=host["mvuRight"] if mode else None, resident=rf)
    return F, host


def dataclass_replace_resident(F):
    import dataclasses
    return dataclasses.replace(F, resident=None)


@dataclass
class MapPointsView:
    """Local map points after Frame::isInFrustum (src/Frame.cc:269-325), in vpMapPoints order."""
    mTrackProjX: np.ndarray
    mTrackProjY: np.ndarray
    mTrackProjXR: np.ndarray
    mnTrackScaleLevel: np.ndarray
    mTrackViewCos: np.ndarray
    descriptors: np.ndarray
    valid: Optional[np.ndarray] = None                    # mbTrackInView && !isBad()
    has_obs: Optional[np.ndarray] = None                  # Observations()>0


@dataclass
class WorldPointsView:
    """MapPoints with world-frame data for SearchByProjection(CurrentFrame, KeyFrame, ...) and (KeyFrame, Scw, ...)."""
    world_pos: np.ndarray                                  # (n,3) float32, GetWorldPos()
    descriptors: np.ndarray                                # (n,32), GetDescriptor()
    max_distance: np.ndarray                               # mfMaxDistance
    min_distance: np.ndarray                               # mfMinDistance
    normal: Optional[np.ndarray] = None                    # (n,3) GetNormal() — Sim3 overload
    angle: Optional[np.ndarray] = None                     # pKF->mvKeysUn[i].angle — keyframe overload, orientation check
    valid: Optional[np.ndarray] = None


def _libm_logf(x: float) -> float:
    """glibc logf — what Frame::mfLogScaleFactor = log(mfScaleFactor) evaluates to (src/Frame.cc:71)."""
    libm = C.CDLL("libm.so.6")
    libm.logf.restype = C.c_float
    libm.logf.argtypes = [C.c_float]
    return float(libm.logf(float(np.float32(x))))


@dataclass
class LastFrameView:
    """What SearchByProjection(CurrentFrame, LastFrame, ...) reads of LastFrame and of its MapPoints."""
    mvKeysUn: np.ndarray
    world_pos: np.ndarray                                  # (N,3) float32, pMP->GetWorldPos()
    descriptors: np.ndarray                                # (N,32), pMP->GetDescriptor()
    valid: Optional[np.ndarray] = None                     # mvpMapPoints[i] && !mvbOutlier[i]
    has_obs: Optional[np.ndarray] = None                   # Observations()>0


@dataclass
class KeyFrameView:
    """What the BoW-guided searches read of a KeyFrame / Frame."""
    mvKeysUn: np.ndarray
    mDescriptors: np.ndarray
    mFeatVec: FeatureVector
    has_mp: Optional[np.ndarray] = None                   # MapPoint present && !isBad(), per feature
    mvuRight: Optional[np.ndarray] = None
    mvScaleFactors: Optional[np.ndarray] = None
    mvLevelSigma2: Optional[np.ndarray] = None
    _keep: list = field(default_factory=list, repr=False)

    def _c(self) -> _KeyFrameViewC:
        k = np.ascontiguousarray(self.mvKeysUn, KP_DTYPE)
        d = np.ascontiguousarray(self.mDescriptors, np.uint8)
        hm = np.ascontiguousarray(self.has_mp, np.uint8) if self.has_mp is not None else None
        ur = np.ascontiguousarray(self.mvuRight, np.float32) if self.mvuRight is not None else None
        nd = np.ascontiguousarray(self.mFeatVec.node_id, np.uint32)
        st = np.ascontiguousarray(self.mFeatVec.start, np.int32)
        fi = np.ascontiguousarray(self.mFeatVec.feat_idx, np.uint32)
        sf = np.ascontiguousarray(self.mvScaleFactors, np.float32) if self.mvScaleFactors is not None else None
        sg = np.ascontiguousarray(self.mvLevelSigma2, np.float32) if self.mvLevelSigma2 is not None else None
        self._keep = [k, d, hm, ur, nd, st, fi, sf, sg]
        nl = len(sf) if sf is not None else (len(sg) if sg is not None else 0)
        return _KeyFrameViewC(len(k), _p(k), _p(d), _p(hm), _p(ur), _FeatVecC(len(nd), _p(nd), _p(st), _p(fi)), nl, _p(sf), _p(sg))


class ORBmatcher:
    """ORBmatcher(nnratio=0.6, checkOri=True) — include/ORBmatcher.h:41."""

    TH_LOW, TH_HIGH, HISTO_LENGTH = TH_LOW, TH_HIGH, HISTO_LENGTH

    def __init__(self, nnratio: float = 0.6, checkOri: bool = True, device: int = 0):
        self._lib = _lib.load()
        self.mfNNratio = float(np.float32(nnratio))
        self.mbCheckOrientation = bool(checkOri)
        h = C.c_void_p()
        check(self._lib.borb_matcher_create(device, C.byref(h)), "borb_matcher_create")
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.borb_matcher_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def DescriptorDistance(a: np.ndarray, b: np.ndarray) -> int:
        """256-bit Hamming distance (src/ORBmatcher.cc:1647-1663) — host convenience for tests."""
        return int(np.unpackbits(np.bitwise_xor(np.asarray(a, np.uint8), np.asarray(b, np.uint8))).sum())

    def SearchByProjection(self, F: FrameView, mps: MapPointsView, th: float = 3.0) -> Tuple[int, np.ndarray]:
        """src/ORBmatcher.cc:45-129.  Returns (nmatches, match_feat[n_mp]): frame feature that received map point i, or -1."""
        fv, keep = F._view()
        mv, arrs = _mappoints_c(mps)
        match = np.full(max(mv.n, 1), -1, np.int32)
        n = C.c_int32(0)
        check(self._lib.borb_search_by_projection(self._h, C.byref(fv), C.byref(mv), float(th), self.mfNNratio, _p(match), C.byref(n)),
              "borb_search_by_projection")
        return n.value, match[:mv.n]

    def SearchByProjectionBatch(self, frames: Sequence[FrameView], mps_list: Sequence[MapPointsView], th: float = 3.0):
        """borb_search_by_projection_batch: SearchByProjection(F, vpMapPoints, th) of many independent device-resident frames in one
        launch pair.  Returns [(nmatches, match_feat)] per job, each equal to the single call's result."""
        n = len(frames)
        assert n == len(mps_list)
        FV = (_FrameViewC * n)()
        MV = (_MapPointViewC * n)()
        keep, outs = [], []
        for j, (F, mps) in enumerate(zip(frames, mps_list)):
            FV[j], k = F._view()
            MV[j], arrs = _mappoints_c(mps)
            keep.append((k, arrs)); outs.append(np.full(max(MV[j].n, 1), -1, np.int32))
        ptrs = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_by_projection_batch(self._h, FV, MV, n, float(th), self.mfNNratio, ptrs, _p(nm)), "borb_search_by_projection_batch")
        return [(int(nm[j]), outs[j][:MV[j].n]) for j in range(n)]

    def SearchByProjectionLast(self, Cur: FrameView, Last: LastFrameView, Tcw: np.ndarray, K: Tuple[float, float, float, float], bf: float,
                               th: float, bForward: bool = False, bBackward: bool = False) -> Tuple[int, np.ndarray]:
        """SearchByProjection(CurrentFrame, LastFrame, th, bMono) — src/ORBmatcher.cc:1328-1470.  Tcw: (3,4) or (4,4) current pose;
        K = (fx, fy, cx, cy).  Returns (nmatches, state[cur.N]): >=0 last-frame index now matched, -1 untouched, -2 culled."""
        fv, keep = Cur._view()
        k = Cur.mvKeysUn
        lv, arrs = _lastframe_c(Last)
        T = np.ascontiguousarray(np.asarray(Tcw, np.float32)[:3, :4]).reshape(12)
        state = np.full(max(len(k), 1), -1, np.int32)
        n = C.c_int32(0)
        check(self._lib.borb_search_by_projection_last(self._h, C.byref(fv), C.byref(lv), _p(T), float(K[0]), float(K[1]), float(K[2]), float(K[3]),
                                                       float(bf), float(th), int(bForward), int(bBackward), int(self.mbCheckOrientation),
                                                       _p(state), C.byref(n)), "borb_search_by_projection_last")
        return n.value, state[:len(k)]

    def _points_call(self, F: FrameView, P: WorldPointsView, with_stereo: bool = False):
        fv, keep = F._view(with_stereo)
        k = F.mvKeysUn
        sf = np.ascontiguousarray(F.mvScaleFactors, np.float32)
        arrs = _c_arrays((P.world_pos, np.float32), (P.descriptors, np.uint8), (P.max_distance, np.float32), (P.min_distance, np.float32),
                         (P.normal, np.float32), (P.angle, np.float32), (P.valid, np.uint8))
        pv = _WorldPointsViewC(len(arrs[0]), *[_p(a) for a in arrs])
        logs = F.mfLogScaleFactor if F.mfLogScaleFactor is not None else _libm_logf(sf[1] if len(sf) > 1 else 1.2)
        return fv, pv, float(logs), len(k), keep + arrs

    def SearchByProjectionKF(self, Cur: FrameView, P: WorldPointsView, Tcw: np.ndarray, Ow: np.ndarray, K: Tuple[float, float, float, float],
                             th: float, ORBdist: int) -> Tuple[int, np.ndarray]:
        """SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) — src/ORBmatcher.cc:1472-1599 (relocalisation).
        P = the keyframe's MapPoints (valid = present, not bad, not already found); Cur.occupied = mvpMapPoints[i] != NULL;
        Ow = -Rcw.t()*tcw.  Returns (nmatches, state[cur.N]): >=0 index into P, -1 untouched, -2 culled by orientation."""
        fv, pv, logs, n, keep = self._points_call(Cur, P)
        T = np.ascontiguousarray(np.asarray(Tcw, np.float32)[:3, :4]).reshape(12)
        ow = np.ascontiguousarray(np.asarray(Ow, np.float32).reshape(3))
        state = np.full(max(n, 1), -1, np.int32)
        nm = C.c_int32(0)
        check(self._lib.borb_search_by_projection_kf(self._h, C.byref(fv), C.byref(pv), _p(T), _p(ow), float(K[0]), float(K[1]), float(K[2]),
                                                     float(K[3]), logs, float(th), int(ORBdist), int(self.mbCheckOrientation), _p(state),
                                                     C.byref(nm)), "borb_search_by_projection_kf")
        return nm.value, state[:n]

    def SearchByProjectionSim3(self, pKF: FrameView, P: WorldPointsView, Tcw: np.ndarray, Ow: np.ndarray,
                               K: Tuple[float, float, float, float], th: int) -> Tuple[int, np.ndarray]:
        """SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) — src/ORBmatcher.cc:290-403 (loop closing).  Tcw = [Rcw|tcw] with
        the Sim3 scale divided out, Ow = -Rcw.t()*tcw; pKF.occupied = vpMatched[idx] != NULL.  Returns (nmatches, state[kf.N])."""
        fv, pv, logs, n, keep = self._points_call(pKF, P)
        T = np.ascontiguousarray(np.asarray(Tcw, np.float32)[:3, :4]).reshape(12)
        ow = np.ascontiguousarray(np.asarray(Ow, np.float32).reshape(3))
        state = np.full(max(n, 1), -1, np.int32)
        nm = C.c_int32(0)
        check(self._lib.borb_search_by_projection_sim3(self._h, C.byref(fv), C.byref(pv), _p(T), _p(ow), float(K[0]), float(K[1]), float(K[2]),
                                                       float(K[3]), logs, int(th), _p(state), C.byref(nm)), "borb_search_by_projection_sim3")
        return nm.value, state[:n]

    def SearchLocalPoints(self, F: FrameView, P: WorldPointsView, Tcw: np.ndarray, Ow: np.ndarray, K: Tuple[float, float, float, float],
                          mbf: float, th: float = 1.0, has_obs: Optional[np.ndarray] = None, viewingCosLimit: float = 0.5):
        """Tracking::SearchLocalPoints (src/Tracking.cc:1148-1194): Frame::isInFrustum for every point of P, then
        SearchByProjection(F, vpMapPoints, th) on those in view, in one call.  Returns a dict with in_view, the MapPoint track
        fields (proj_x, proj_y, proj_xr, level, view_cos), match (feature per point or -1) and nmatches."""
        fv, pv, logs, n, keep = self._points_call(F, P, with_stereo=True)
        T = np.ascontiguousarray(np.asarray(Tcw, np.float32)[:3, :4]).reshape(12)
        ow = np.ascontiguousarray(np.asarray(Ow, np.float32).reshape(3))
        ho = np.ascontiguousarray(has_obs, np.uint8) if has_obs is not None else None
        nq = len(P.world_pos)
        out = _local_points_outputs(nq)
        nm = C.c_int32(0)
        check(self._lib.borb_search_local_points(self._h, C.byref(fv), C.byref(pv), _p(ho), _p(T), _p(ow), float(K[0]), float(K[1]), float(K[2]),
                                                 float(K[3]), float(mbf), float(viewingCosLimit), logs, float(th), self.mfNNratio,
                                                 _p(out["in_view"]), _p(out["proj_x"]), _p(out["proj_y"]), _p(out["proj_xr"]), _p(out["level"]),
                                                 _p(out["view_cos"]), _p(out["match"]), C.byref(nm)), "borb_search_local_points")
        out = {k: v[:nq] for k, v in out.items()}
        out["nmatches"] = nm.value
        return out

    def SearchLocalPointsBatch(self, frames: Sequence[FrameView], points: Sequence[WorldPointsView], poses, K, mbf, th=1.0,
                               has_obs=None, viewingCosLimit: float = 0.5):
        """borb_search_local_points_batch: SearchLocalPoints of many independent camera streams (device-resident frames) in one
        launch sequence.  poses[j] = (Tcw, Ow); K (fx, fy, cx, cy), mbf and th are one value for every job or one per job; has_obs is
        None or a per-job list (entries may be None).  Returns one dict per job, equal to what SearchLocalPoints returns."""
        n = len(frames)
        assert n == len(points) == len(poses)
        Ks, bfs, ths = _per_job(K, n, 1), _per_job(mbf, n), _per_job(th, n)
        obs = list(has_obs) if has_obs is not None else [None] * n
        jobs = (_LocalPointsJobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            fv, pv, logs, _, k = self._points_call(frames[j], points[j], with_stereo=True)
            ho = np.ascontiguousarray(obs[j], np.uint8) if obs[j] is not None else None
            nq = len(points[j].world_pos)
            out = _local_points_outputs(nq)
            Tcw, Ow = poses[j]
            J = jobs[j]
            J.frame, J.pts, J.has_obs, J.Tcw = fv, pv, _p(ho), _pose12(Tcw)
            J.Ow = (C.c_float * 3)(*np.asarray(Ow, np.float32).reshape(3).tolist())
            J.fx, J.fy, J.cx, J.cy = [float(x) for x in Ks[j]]
            J.mbf, J.log_scale_factor, J.th = float(bfs[j]), logs, float(ths[j])
            J.in_view, J.proj_x, J.proj_y, J.proj_xr = _p(out["in_view"]), _p(out["proj_x"]), _p(out["proj_y"]), _p(out["proj_xr"])
            J.level, J.view_cos, J.match_feat = _p(out["level"]), _p(out["view_cos"]), _p(out["match"])
            keep.append((k, ho)); outs.append((nq, out))
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_local_points_batch(self._h, jobs, n, float(viewingCosLimit), self.mfNNratio, _p(nm)),
              "borb_search_local_points_batch")
        res = []
        for j, (nq, out) in enumerate(outs):
            r = {k: v[:nq] for k, v in out.items()}
            r["nmatches"] = int(nm[j])
            res.append(r)
        return res

    def SearchByProjectionLastBatch(self, curs: Sequence[FrameView], lasts: Sequence[LastFrameView], poses, K, bf, th,
                                    forward=False, backward=False):
        """borb_search_by_projection_last_batch: SearchByProjection(CurrentFrame, LastFrame, th, bMono) of many independent camera
        streams (device-resident current frames) in one launch sequence.  poses[j] = Tcw; K, bf, th, forward and backward are one
        value for every job or one per job.  Returns [(nmatches, state)] per job, equal to what SearchByProjectionLast returns."""
        n = len(curs)
        assert n == len(lasts) == len(poses)
        Ks, bfs, ths = _per_job(K, n, 1), _per_job(bf, n), _per_job(th, n)
        fws, bws = _per_job(forward, n), _per_job(backward, n)
        jobs = (_LastFrameJobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            fv, k = curs[j]._view()
            lv, arrs = _lastframe_c(lasts[j])
            n_cur = len(curs[j].mvKeysUn)
            state = np.full(max(n_cur, 1), -1, np.int32)
            J = jobs[j]
            J.cur, J.last, J.Tcw = fv, lv, _pose12(poses[j])
            J.fx, J.fy, J.cx, J.cy = [float(x) for x in Ks[j]]
            J.bf, J.th, J.forward, J.backward, J.state_cur = float(bfs[j]), float(ths[j]), int(fws[j]), int(bws[j]), _p(state)
            keep.append((k, arrs)); outs.append((n_cur, state))
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_by_projection_last_batch(self._h, jobs, n, int(self.mbCheckOrientation), _p(nm)),
              "borb_search_by_projection_last_batch")
        return [(int(nm[j]), state[:n_cur]) for j, (n_cur, state) in enumerate(outs)]

    def SearchByProjectionKFBatch(self, curs: Sequence[FrameView], points: Sequence[WorldPointsView], poses, K, th, ORBdist):
        """borb_search_by_projection_kf_batch: SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) of many relocalising
        camera streams (device-resident current frames) in one launch sequence.  poses[j] = (Tcw, Ow); K, th and ORBdist are one
        value for every job or one per job.  Returns [(nmatches, state)] per job, equal to what SearchByProjectionKF returns."""
        n = len(curs)
        assert n == len(points) == len(poses)
        Ks, ths, ods = _per_job(K, n, 1), _per_job(th, n), _per_job(ORBdist, n)
        jobs = (_KfProjectionJobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            fv, pv, logs, n_cur, k = self._points_call(curs[j], points[j])
            state = np.full(max(n_cur, 1), -1, np.int32)
            Tcw, Ow = poses[j]
            J = jobs[j]
            J.cur, J.pts, J.Tcw, J.Ow = fv, pv, _pose12(Tcw), _vec3(Ow)
            J.fx, J.fy, J.cx, J.cy = [float(x) for x in Ks[j]]
            J.log_scale_factor, J.th, J.orb_dist, J.state_cur = logs, float(ths[j]), int(ods[j]), _p(state)
            keep.append(k); outs.append((n_cur, state))
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_by_projection_kf_batch(self._h, jobs, n, int(self.mbCheckOrientation), _p(nm)),
              "borb_search_by_projection_kf_batch")
        return [(int(nm[j]), state[:n_cur]) for j, (n_cur, state) in enumerate(outs)]

    def SearchByProjectionSim3Batch(self, kfs: Sequence[FrameView], points: Sequence[WorldPointsView], poses, K, th=10):
        """borb_search_by_projection_sim3_batch: SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) of many loop-closing streams
        (device-resident keyframes) in one launch sequence.  poses[j] = (Tcw, Ow) with the Sim3 scale divided out; K and th are one
        value for every job or one per job.  Returns [(nmatches, state)] per job, equal to what SearchByProjectionSim3 returns."""
        n = len(kfs)
        assert n == len(points) == len(poses)
        Ks, ths = _per_job(K, n, 1), _per_job(th, n)
        jobs = (_Sim3ProjectionJobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            fv, pv, logs, n_kf, k = self._points_call(kfs[j], points[j])
            state = np.full(max(n_kf, 1), -1, np.int32)
            Tcw, Ow = poses[j]
            J = jobs[j]
            J.kf, J.pts, J.Tcw, J.Ow = fv, pv, _pose12(Tcw), _vec3(Ow)
            J.fx, J.fy, J.cx, J.cy = [float(x) for x in Ks[j]]
            J.log_scale_factor, J.th, J.state_kf = logs, int(ths[j]), _p(state)
            keep.append(k); outs.append((n_kf, state))
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_by_projection_sim3_batch(self._h, jobs, n, _p(nm)), "borb_search_by_projection_sim3_batch")
        return [(int(nm[j]), state[:n_kf]) for j, (n_kf, state) in enumerate(outs)]

    def SearchBySim3Batch(self, kf1s: Sequence[FrameView], kf2s: Sequence[FrameView], P1s: Sequence[WorldPointsView],
                          P2s: Sequence[WorldPointsView], poses, sims, K, th=7.5):
        """borb_search_by_sim3_batch: SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) of many (keyframe, candidate) pairs on
        device-resident keyframes in three launches.  poses[j] = (T1w, T2w), sims[j] = (S12, S21) as for SearchBySim3; K (pKF1's)
        and th are one value for every job or one per job.  Returns [(nFound, match12)] per job, equal to what SearchBySim3 returns."""
        n = len(kf1s)
        assert n == len(kf2s) == len(P1s) == len(P2s) == len(poses) == len(sims)
        Ks, ths = _per_job(K, n, 1), _per_job(th, n)
        jobs = (_Sim3JobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            fv1, pv1, logs1, n1, k1 = self._points_call(kf1s[j], P1s[j])
            fv2, pv2, logs2, _, k2 = self._points_call(kf2s[j], P2s[j])
            match = np.full(max(n1, 1), -1, np.int32)
            J = jobs[j]
            J.kf1, J.kf2, J.pts1, J.pts2 = fv1, fv2, pv1, pv2
            J.T1w, J.T2w = _pose12(poses[j][0]), _pose12(poses[j][1])
            J.S12, J.S21 = _pose12(sims[j][0]), _pose12(sims[j][1])
            J.fx, J.fy, J.cx, J.cy = [float(x) for x in Ks[j]]
            J.log_scale_factor1, J.log_scale_factor2, J.th, J.match12 = logs1, logs2, float(ths[j]), _p(match)
            keep.append((k1, k2)); outs.append((n1, match))
        nf = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_by_sim3_batch(self._h, jobs, n, _p(nf)), "borb_search_by_sim3_batch")
        return [(int(nf[j]), match[:n1]) for j, (n1, match) in enumerate(outs)]

    def SearchForInitialization(self, F1: FrameView, F2: FrameView, vbPrevMatched: np.ndarray, windowSize: int = 10):
        """SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) — src/ORBmatcher.cc:405-520.
        Returns (nmatches, vnMatches12[F1.N], updated vbPrevMatched (N,2))."""
        views, keep = [], []
        for F in (F1, F2):
            k = np.ascontiguousarray(F.mvKeysUn, KP_DTYPE); d = np.ascontiguousarray(F.mDescriptors, np.uint8)
            sf = np.ascontiguousarray(F.mvScaleFactors, np.float32)
            views.append(_FrameViewC(len(k), _p(k), _p(d), None, None, *[float(x) for x in F.bounds], len(sf), _p(sf)))
            keep += [k, d, sf]
        n1 = views[0].n
        prev = _prev_matched(vbPrevMatched)
        m12 = np.full(max(n1, 1), -1, np.int32)
        nm = C.c_int32(0)
        check(self._lib.borb_search_for_initialization(self._h, C.byref(views[0]), C.byref(views[1]), _p(prev), int(windowSize), self.mfNNratio,
                                                       int(self.mbCheckOrientation), _p(m12), C.byref(nm)), "borb_search_for_initialization")
        return nm.value, m12[:n1], prev[:n1]

    def SearchForInitializationBatch(self, F1s: Sequence[FrameView], F2s: Sequence[FrameView], prevs, windowSize=100):
        """borb_search_for_initialization_batch: SearchForInitialization of many camera streams in two launches.  F1s[j] / F2s[j] =
        job j's initial and current frames, device-resident (FrameView.resident); prevs[j] = its vbPrevMatched (N1,2); windowSize is
        one value or one per job.  Returns [(nmatches, vnMatches12, updated vbPrevMatched)] per job, equal to what
        SearchForInitialization returns on host views of the same frames."""
        n = len(F1s)
        assert n == len(F2s) == len(prevs)
        wins = _per_job(windowSize, n)
        jobs = (_InitJobC * max(n, 1))()
        outs = []
        for j in range(n):
            F1, F2 = F1s[j], F2s[j]
            n1 = F1.resident.n if F1.resident is not None else len(F1.mvKeysUn)
            prev = _prev_matched(prevs[j])
            m12 = np.full(max(n1, 1), -1, np.int32)
            jobs[j] = _InitJobC(F1.resident._h if F1.resident is not None else None, F2.resident._h if F2.resident is not None else None,
                                _p(prev), int(wins[j]), _p(m12))
            outs.append((n1, m12, prev))
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_for_initialization_batch(self._h, jobs, n, self.mfNNratio, int(self.mbCheckOrientation), _p(nm)),
              "borb_search_for_initialization_batch")
        return [(int(nm[j]), m12[:n1], prev[:n1]) for j, (n1, m12, prev) in enumerate(outs)]

    def ComputeDistinctiveDescriptors(self, groups) -> np.ndarray:
        """MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307) for a batch of MapPoints: groups[p] = (N_p,32)
        uint8 descriptors of the point's observations.  Returns best[p] = index of the medoid-by-median descriptor (-1 if empty)."""
        groups = [np.ascontiguousarray(g, np.uint8).reshape(-1, 32) for g in groups]
        off = np.zeros(len(groups) + 1, np.int32)
        off[1:] = np.cumsum([len(g) for g in groups])
        desc = np.ascontiguousarray(np.concatenate(groups, 0)) if len(groups) and off[-1] > 0 else np.zeros((1, 32), np.uint8)
        best = np.full(max(len(groups), 1), -1, np.int32)
        check(self._lib.borb_distinctive_descriptors(self._h, _p(desc), _p(off), len(groups), _p(best)), "borb_distinctive_descriptors")
        return best[:len(groups)]

    def ComputeDistinctiveDescriptorsFrames(self, frames, groups) -> Tuple[np.ndarray, np.ndarray]:
        """borb_distinctive_descriptors_frames: ComputeDistinctiveDescriptors of many MapPoints (any number of streams) read from
        resident keyframes, no keyframe row crossing PCIe.  frames = ResidentFrames, or FrameViews carrying one; groups[p] = (frame
        indices, feature indices) of MapPoint p's non-bad observations in mObservations order.  Returns (best[p], descriptors
        (n_points,32)): best as ComputeDistinctiveDescriptors on the gathered rows, and the chosen row (zeros where best is -1)."""
        rfs = [F.resident if isinstance(F, FrameView) else F for F in frames]
        handles = (C.c_void_p * max(len(rfs), 1))(*[rf._h.value if rf is not None else None for rf in rfs])
        fi = [np.asarray(f, np.int32).reshape(-1) for f, _ in groups]
        ki = [np.asarray(k, np.int32).reshape(-1) for _, k in groups]
        assert all(len(a) == len(b) for a, b in zip(fi, ki))
        off = np.zeros(len(groups) + 1, np.int32)
        off[1:] = np.cumsum([len(a) for a in fi])
        obs_f = np.ascontiguousarray(np.concatenate(fi)) if off[-1] > 0 else np.zeros(1, np.int32)
        obs_k = np.ascontiguousarray(np.concatenate(ki)) if off[-1] > 0 else np.zeros(1, np.int32)
        best = np.full(max(len(groups), 1), -1, np.int32)
        desc = np.zeros((max(len(groups), 1), 32), np.uint8)
        check(self._lib.borb_distinctive_descriptors_frames(self._h, handles, len(rfs), _p(obs_f), _p(obs_k), _p(off), len(groups), _p(best),
                                                            _p(desc)), "borb_distinctive_descriptors_frames")
        return best[:len(groups)], desc[:len(groups)]

    def Fuse(self, pKF: FrameView, P: WorldPointsView, Tcw: np.ndarray, Ow: np.ndarray, K: Tuple[float, float, float, float], bf: float,
             th: float = 3.0, Scw: bool = False) -> Tuple[int, np.ndarray]:
        """Search part of Fuse(pKF, vpMapPoints, th) — src/ORBmatcher.cc:825-970 — or, with Scw=True, of
        Fuse(pKF, Scw, vpPoints, th, vpReplacePoint) — :972-1100.  Returns (n_found, best_idx[len(P)]); the MapPoint
        bookkeeping (Replace / AddObservation / vpReplacePoint) is the caller's, applied in order."""
        fv, pv, logs, n, keep = self._points_call(pKF, P, with_stereo=not Scw)
        inv = np.ascontiguousarray(pKF.mvInvLevelSigma2, np.float32) if pKF.mvInvLevelSigma2 is not None else None
        T = np.ascontiguousarray(np.asarray(Tcw, np.float32)[:3, :4]).reshape(12)
        ow = np.ascontiguousarray(np.asarray(Ow, np.float32).reshape(3))
        nq = len(P.world_pos)
        best = np.full(max(nq, 1), -1, np.int32)
        nf = C.c_int32(0)
        check(self._lib.borb_fuse(self._h, C.byref(fv), _p(inv), C.byref(pv), _p(T), _p(ow), float(K[0]), float(K[1]), float(K[2]), float(K[3]),
                                  float(bf), logs, float(th), int(Scw), _p(best), C.byref(nf)), "borb_fuse")
        return nf.value, best[:nq]

    def SearchBySim3(self, pKF1: FrameView, pKF2: FrameView, P1: WorldPointsView, P2: WorldPointsView, T1w: np.ndarray, T2w: np.ndarray,
                     S12: np.ndarray, S21: np.ndarray, K: Tuple[float, float, float, float], th: float) -> Tuple[int, np.ndarray]:
        """SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) — src/ORBmatcher.cc:1102-1326.  S12 = [s12*R12 | t12],
        S21 = [(1/s12)*R12^T | -sR21*t12] (3x4).  Returns (nFound, match12[kf1.N]): index in KF2 or -1."""
        fv1, pv1, logs1, n1, keep1 = self._points_call(pKF1, P1)
        fv2, pv2, logs2, n2, keep2 = self._points_call(pKF2, P2)
        mats = [np.ascontiguousarray(np.asarray(Mx, np.float32)[:3, :4]).reshape(12) for Mx in (T1w, T2w, S12, S21)]
        match = np.full(max(n1, 1), -1, np.int32)
        nf = C.c_int32(0)
        check(self._lib.borb_search_by_sim3(self._h, C.byref(fv1), C.byref(fv2), C.byref(pv1), C.byref(pv2), _p(mats[0]), _p(mats[1]),
                                            _p(mats[2]), _p(mats[3]), float(K[0]), float(K[1]), float(K[2]), float(K[3]), logs1, logs2,
                                            float(th), _p(match), C.byref(nf)), "borb_search_by_sim3")
        return nf.value, match[:n1]

    def SearchByBoW(self, pKF, F: KeyFrameView):
        """SearchByBoW(KeyFrame*, Frame&, vpMapPointMatches) — src/ORBmatcher.cc:159-288.  pKF may be one KeyFrameView or a
        sequence (batched candidates).  Returns (nmatches, match[F.N]) or lists of them: match[j] = keyframe feature whose
        MapPoint frame feature j received, or -1."""
        single = isinstance(pKF, KeyFrameView)
        kfs = [pKF] if single else list(pKF)
        arr = (_KeyFrameViewC * len(kfs))(*[kf._c() for kf in kfs])
        fc = F._c()
        nF = len(F.mvKeysUn)
        match = np.full((len(kfs), max(nF, 1)), -1, np.int32)
        nm = np.zeros(len(kfs), np.int32)
        check(self._lib.borb_search_by_bow(self._h, arr, len(kfs), C.byref(fc), self.mfNNratio, int(self.mbCheckOrientation), _p(match), _p(nm)),
              "borb_search_by_bow")
        match = match[:, :nF]
        return (int(nm[0]), match[0]) if single else (nm, match)

    def SearchByBoW_KF(self, pKF1: KeyFrameView, pKF2: KeyFrameView) -> Tuple[int, np.ndarray]:
        """SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) — src/ORBmatcher.cc:522-655.  match12[i] = index in KF2 or -1."""
        c1, c2 = pKF1._c(), pKF2._c()
        n1 = len(pKF1.mvKeysUn)
        match = np.full(max(n1, 1), -1, np.int32)
        nm = C.c_int32(0)
        check(self._lib.borb_search_by_bow_kf(self._h, C.byref(c1), C.byref(c2), self.mfNNratio, int(self.mbCheckOrientation), _p(match), C.byref(nm)),
              "borb_search_by_bow_kf")
        return nm.value, match[:n1]

    def ComputeBoWBatch(self, voc: "ORBVocabulary", frames: Sequence[FrameView], levelsup: int = 4, want_host: bool = True):
        """borb_frames_compute_bow: Frame::ComputeBoW (src/Frame.cc:395-402) of many device-resident frames in one launch pair.  The
        vectors stay with the frames (SearchByBoWBatch reads them).  Returns [(mBowVec as {word: value}, mFeatVec)] per frame, equal to
        what ORBVocabulary.ComputeBoW returns for the frame's descriptors; with want_host=False nothing is copied back and the result
        is None."""
        n = len(frames)
        hs = (C.c_void_p * max(n, 1))(*[F.resident._h.value if F.resident is not None else None for F in frames])
        sizes = [F.resident.n if F.resident is not None else len(F.mvKeysUn) for F in frames]
        outs = [(np.zeros(max(k, 1), np.uint32), np.zeros(max(k, 1), np.float64), np.zeros(max(k, 1), np.uint32), np.zeros(k + 1, np.int32),
                 np.zeros(max(k, 1), np.uint32)) for k in sizes]
        tables = [(C.c_void_p * max(n, 1))(*[o[t].ctypes.data for o in outs]) if want_host else None for t in range(5)]
        nb, nn = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_frames_compute_bow(self._h, voc._h, hs, n, int(levelsup), tables[0], tables[1], _p(nb), tables[2], tables[3],
                                                tables[4], _p(nn)), "borb_frames_compute_bow")
        if not want_host:
            return None
        return [_bow_result(*o, int(nb[j]), int(nn[j])) for j, o in enumerate(outs)]

    def SearchByBoWBatch(self, kfs, frames: Sequence[FrameView]):
        """borb_search_by_bow_batch: TrackReferenceKeyFrame's SearchByBoW(KeyFrame*, Frame&) (src/ORBmatcher.cc:159-288) of many
        independent camera streams in one launch.  frames[j] = device-resident FrameView whose BoW ComputeBoWBatch computed; kfs[j] =
        a KeyFrameView, or a resident FrameView with BoW and has_mp (then only has_mp crosses PCIe).  Returns [(nmatches, match)] per
        job, equal to what SearchByBoW returns on host views of the same data."""
        n = len(frames)
        assert n == len(kfs)
        jobs = (_BowJobC * max(n, 1))()
        keep, outs = [], []
        for j, (kf, F) in enumerate(zip(kfs, frames)):
            nF = F.resident.n if F.resident is not None else len(F.mvKeysUn)
            match = np.full(max(nF, 1), -1, np.int32)
            J = jobs[j]
            J.frame = F.resident._h.value if F.resident is not None else None
            J.kf, J.kf_frame, _ = self._kf_side(kf, keep)
            J.match = _p(match)
            outs.append((nF, match))
        nm = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_search_by_bow_batch(self._h, jobs, n, self.mfNNratio, int(self.mbCheckOrientation), _p(nm)), "borb_search_by_bow_batch")
        return [(int(nm[j]), match[:nF]) for j, (nF, match) in enumerate(outs)]

    @staticmethod
    def _db_jobs(dbs, n):
        """One database per job: a sequence, or one KeyFrameDatabase shared by every job."""
        dbs = [dbs] * n if isinstance(dbs, KeyFrameDatabase) else list(dbs)
        assert len(dbs) == n
        return dbs

    def KfdbQueryBatch(self, dbs, frames: Sequence[FrameView]):
        """borb_kfdb_query_batch: the KeyFrameDatabase query (KeyFrameDatabase.query) of many resident frames whose BoW ComputeBoWBatch
        computed, in one launch.  dbs[j] is job j's database (or one database for every job).  Returns [(common_words, score,
        first_word)] per job, equal to dbs[j].query() with the frame's BowVector.

        DetectRelocalizationCandidates of these queries is relocalization_candidates(cw, sc, fw, db._seq, covisibility,
        db._reloc_score) applied to the jobs IN JOB ORDER, each with its database's persistent mRelocScore dict: a query reads the
        mRelocScore that earlier queries left on keyframes below its own threshold, so the job order stands for the order of the
        sequential calls it replaces."""
        n = len(frames)
        dbs = self._db_jobs(dbs, n)
        sizes = [db.size()[0] if db is not None else 0 for db in dbs]
        while True:              # sized again when another thread added keyframes since (refused before any launch)
            jobs = (_KfdbQueryJobC * max(n, 1))()
            outs = []
            for j, (db, F, ns) in enumerate(zip(dbs, frames, sizes)):
                cw = np.zeros(max(ns, 1), np.int32); sc = np.zeros(max(ns, 1), np.float32); fw = np.zeros(max(ns, 1), np.uint32)
                nsl = np.zeros(1, np.int32)
                J = jobs[j]
                J.db = db._h.value if db is not None else None
                J.frame = F.resident._h.value if (F is not None and F.resident is not None) else None
                J.common_words, J.score, J.first_word, J.cap, J.n_slots = _p(cw), _p(sc), _p(fw), len(cw), _p(nsl)
                outs.append((cw, sc, fw, nsl))
            st = self._lib.borb_kfdb_query_batch(self._h, jobs, n)
            grown = [int(o[3][0]) > len(o[0]) for o in outs]
            if not (st == BORB_ERR_CAPACITY and any(grown)):
                break
            sizes = [max(ns, int(o[3][0])) for ns, o in zip(sizes, outs)]
        check(st, "borb_kfdb_query_batch")
        return [(cw[:int(nsl[0])], sc[:int(nsl[0])], fw[:int(nsl[0])]) for cw, sc, fw, nsl in outs]

    def KfdbAddFramesBatch(self, dbs, frames: Sequence[FrameView], has_mps) -> List[int]:
        """borb_kfdb_add_frames: KeyFrameDatabase.add of many resident frames whose BoW ComputeBoWBatch computed, in one launch; only
        the MapPoint masks cross PCIe.  dbs[j] is job j's database (or one database for every job); has_mps[j] = job j's mask (n
        entries, MapPoint present && !isBad()) or None.  Returns the new slots; each database ends as db.add() in job order leaves it
        with a host view of the frame and its BowVector.  The frames' FeatureVector level must be the databases' (caller's duty)."""
        n = len(frames)
        dbs = self._db_jobs(dbs, n)
        has_mps = list(has_mps) if has_mps is not None else [None] * n
        assert len(has_mps) == n
        jobs = (_KfdbAddJobC * max(n, 1))()
        slots = np.full(max(n, 1), -1, np.int32)
        keep = []
        for j, (db, F, hm) in enumerate(zip(dbs, frames, has_mps)):
            hm = np.ascontiguousarray(hm, np.uint8) if hm is not None else None
            keep.append(hm)
            J = jobs[j]
            J.db = db._h.value if db is not None else None
            J.frame = F.resident._h.value if (F is not None and F.resident is not None) else None
            J.has_mp, J.slot_out = _p(hm), slots.ctypes.data + 4 * j
        check(self._lib.borb_kfdb_add_frames(self._h, jobs, n), "borb_kfdb_add_frames")
        for db, F in zip(dbs, frames):
            db._appended(F.resident.n)
        return [int(s) for s in slots[:n]]

    @staticmethod
    def _bow_ref(x) -> "_BowRefC":
        """A BowVector on the device: a FrameView bound to a resident frame, or a (KeyFrameDatabase, slot) pair."""
        if isinstance(x, FrameView):
            return _BowRefC(x.resident._h.value if x.resident is not None else None, None, 0)
        db, slot = x
        return _BowRefC(None, db._h.value if db is not None else None, int(slot))

    def BowScoreBatch(self, jobs) -> List[np.ndarray]:
        """borb_bow_score_batch: TemplatedVocabulary::score(v1, v2) cast to float, as LoopClosing::DetectLoop takes it for minScore
        (src/LoopClosing.cc:121-140), between BowVectors already on the device, in one launch.  jobs = [(query, targets)], each
        BowVector a FrameView whose BoW ComputeBoWBatch computed or a (KeyFrameDatabase, slot) pair.  Returns one float32 array
        per job: score(query, targets[t])."""
        n = len(jobs)
        cj = (_BowScoreJobC * max(n, 1))()
        keep, outs = [], []
        for j, (query, targets) in enumerate(jobs):
            refs = (_BowRefC * max(len(targets), 1))(*[self._bow_ref(t) for t in targets])
            sc = np.zeros(max(len(targets), 1), np.float32)
            cj[j].query, cj[j].targets, cj[j].n_targets, cj[j].score = self._bow_ref(query), C.addressof(refs), len(targets), _p(sc)
            keep.append(refs)
            outs.append(sc[:len(targets)])
        check(self._lib.borb_bow_score_batch(self._h, cj, n), "borb_bow_score_batch")
        return outs

    def SearchByBoWDbBatch(self, dbs, slots_list, frames: Sequence[FrameView], pairs_cap=None):
        """borb_search_by_bow_db_batch: SearchByBoW(KeyFrame*, Frame&) (src/ORBmatcher.cc:159-288) of many resident frames with BoW
        against candidate keyframes of their databases, in one launch sequence.  slots_list[j] = slot list of job j (None: every
        slot); pairs_cap = None (room for every pair), one int for every job, or one per job.  Returns [(nmatches, pair_offset,
        pairs)] per job as KeyFrameDatabase.SearchByBoWPairs returns them."""
        n = len(frames)
        dbs = self._db_jobs(dbs, n)
        caps = pairs_cap if isinstance(pairs_cap, (list, tuple)) else [pairs_cap] * n
        jobs = (_BowDbJobC * max(n, 1))()
        outs = []
        for j, (db, sl, F, cap) in enumerate(zip(dbs, slots_list, frames, caps)):
            if sl is None:
                n_kf, sla = (db.size()[0] if db is not None else 0), None
            else:
                sla = np.ascontiguousarray(sl, np.int32); n_kf = len(sla)
            nF = F.resident.n if (F is not None and F.resident is not None) else 0
            cap = int(cap) if cap is not None else max(n_kf * nF, 1)
            nm = np.zeros(max(n_kf, 1), np.int32); off = np.zeros(max(n_kf, 1), np.int32)
            pairs = np.zeros(max(cap, 1), np.uint32); tot = np.zeros(1, np.int32)
            J = jobs[j]
            J.db = db._h.value if db is not None else None
            J.frame = F.resident._h.value if (F is not None and F.resident is not None) else None
            J.slots, J.n_kf = _p(sla), n_kf
            J.n_matches, J.pair_offset, J.pairs, J.pairs_cap, J.n_pairs_total = _p(nm), _p(off), _p(pairs), cap, _p(tot)
            outs.append((sla, n_kf, nm, off, pairs, tot))
        check(self._lib.borb_search_by_bow_db_batch(self._h, jobs, n, self.mfNNratio, int(self.mbCheckOrientation)),
              "borb_search_by_bow_db_batch")
        return [(nm[:n_kf], off[:n_kf], pairs[:int(tot[0])]) for _, n_kf, nm, off, pairs, tot in outs]

    def SearchByBoWKFDbBatch(self, dbs, query_slots, slots_list, pairs_cap=None):
        """borb_search_by_bow_kf_db_batch: SearchByBoW(KeyFrame*, KeyFrame*) (src/ORBmatcher.cc:522-655) of many loop-closing keyframes,
        each a slot of its database, against candidate slots of the same database, in one launch sequence.  slots_list[j] = the
        candidates of job j (None: every slot); pairs_cap as SearchByBoWDbBatch.  Returns [(nmatches, pair_offset, pairs)] per job as
        KeyFrameDatabase.SearchByBoWKFPairs returns them."""
        n = len(query_slots)
        dbs = self._db_jobs(dbs, n)
        caps = pairs_cap if isinstance(pairs_cap, (list, tuple)) else [pairs_cap] * n
        jobs = (_BowKfDbJobC * max(n, 1))()
        outs = []
        for j, (db, q, sl, cap) in enumerate(zip(dbs, query_slots, slots_list, caps)):
            if sl is None:
                n_kf, sla = (db.size()[0] if db is not None else 0), None
            else:
                sla = np.ascontiguousarray(sl, np.int32); n_kf = len(sla)
            cap = int(cap) if cap is not None else max(n_kf * (db._n_features(q) if db is not None else 0), 1)
            nm = np.zeros(max(n_kf, 1), np.int32); off = np.zeros(max(n_kf, 1), np.int32)
            pairs = np.zeros(max(cap, 1), np.uint32); tot = np.zeros(1, np.int32)
            J = jobs[j]
            J.db = db._h.value if db is not None else None
            J.query_slot, J.slots, J.n_kf = int(q), _p(sla), n_kf
            J.n_matches, J.pair_offset, J.pairs, J.pairs_cap, J.n_pairs_total = _p(nm), _p(off), _p(pairs), cap, _p(tot)
            outs.append((sla, n_kf, nm, off, pairs, tot))
        check(self._lib.borb_search_by_bow_kf_db_batch(self._h, jobs, n, self.mfNNratio, int(self.mbCheckOrientation)),
              "borb_search_by_bow_kf_db_batch")
        return [(nm[:n_kf], off[:n_kf], pairs[:int(tot[0])]) for _, n_kf, nm, off, pairs, tot in outs]

    def SearchForTriangulation(self, pKF1: KeyFrameView, pKF2: KeyFrameView, F12: np.ndarray, epipole: Tuple[float, float],
                               bOnlyStereo: bool = False) -> np.ndarray:
        """src/ORBmatcher.cc:657-823.  Returns vMatchedPairs as an (m,2) int array (idx1, idx2), ascending idx1."""
        c1, c2 = pKF1._c(), pKF2._c()
        f = np.ascontiguousarray(F12, np.float32).reshape(9)
        cap = max(len(pKF1.mvKeysUn), 1)
        pairs = np.zeros((cap, 2), np.int32)
        n = C.c_int32(0)
        check(self._lib.borb_search_for_triangulation(self._h, C.byref(c1), C.byref(c2), _p(f), float(epipole[0]), float(epipole[1]),
                                                      int(bOnlyStereo), int(self.mbCheckOrientation), _p(pairs), cap, C.byref(n)),
              "borb_search_for_triangulation")
        return pairs[:n.value]

    @staticmethod
    def _kf_side(kf, keep):
        """(borb_keyframe_view, resident frame handle, feature count) of the keyframe side of a batched BoW-guided search: a
        KeyFrameView, or a device-resident FrameView with BoW and has_mp (then only has_mp and mvLevelSigma2 = mvScaleFactors^2 in
        float, ORBextractor's definition, cross PCIe)."""
        if isinstance(kf, KeyFrameView):
            c = kf._c()
            keep.append(list(kf._keep))                  # the same view may serve several jobs: _c() replaces kf._keep
            return c, None, len(kf.mvKeysUn)
        if isinstance(kf, FrameView) and kf.resident is not None:
            hm = np.ascontiguousarray(kf.has_mp, np.uint8) if kf.has_mp is not None else None
            sf = np.asarray(kf.mvScaleFactors, np.float32)
            sg = np.ascontiguousarray(sf * sf, np.float32)
            keep.append((hm, sg))
            return _KeyFrameViewC(0, None, None, _p(hm), n_levels=len(sg), level_sigma2=_p(sg)), kf.resident._h.value, kf.resident.n
        raise ValueError("a KeyFrameView or a device-resident FrameView")

    _tri_side = _kf_side        # the name callers that assemble borb_triangulation_job tables by hand already use

    def SearchForTriangulationBatch(self, kf1s, kf2s, F12s, epipoles, bOnlyStereo=False, caps=None):
        """borb_search_for_triangulation_batch: SearchForTriangulation (src/ORBmatcher.cc:657-823) of many keyframe pairs in one launch.
        kf1s[j] / kf2s[j] = KeyFrameView or device-resident FrameView (BoW from ComputeBoWBatch, has_mp set); bOnlyStereo and caps
        (None: one pair per kf1 feature) are one value for every job or one per job.  Returns vMatchedPairs per job, equal to what
        SearchForTriangulation returns on host views of the same data."""
        n = len(kf1s)
        assert n == len(kf2s) == len(F12s) == len(epipoles)
        ost, cps = _per_job(bOnlyStereo, n), _per_job(caps, n)
        jobs = (_TriangulationJobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            J = jobs[j]
            J.kf1, J.kf1_frame, n1 = self._kf_side(kf1s[j], keep)
            J.kf2, J.kf2_frame, _ = self._kf_side(kf2s[j], keep)
            J.F12 = (C.c_float * 9)(*np.asarray(F12s[j], np.float32).reshape(9).tolist())
            J.ex, J.ey, J.only_stereo = float(epipoles[j][0]), float(epipoles[j][1]), int(ost[j])
            cap = n1 if cps[j] is None else int(cps[j])
            pairs, npairs = np.zeros((max(cap, 1), 2), np.int32), np.zeros(1, np.int32)
            J.pairs, J.cap, J.n_pairs = _p(pairs), cap, _p(npairs)
            outs.append((pairs, npairs))
        check(self._lib.borb_search_for_triangulation_batch(self._h, jobs, n, int(self.mbCheckOrientation)), "borb_search_for_triangulation_batch")
        return [pairs[:int(npairs[0])] for pairs, npairs in outs]

    def FuseBatch(self, kfs: Sequence[FrameView], points: Sequence[WorldPointsView], poses, K, bf, th=3.0, Scw=False):
        """borb_fuse_batch: the search part of Fuse (src/ORBmatcher.cc:825-970, or with Scw=True :972-1100) of many jobs in two launches.
        kfs[j] = device-resident FrameView (mvInvLevelSigma2 set unless Scw); poses[j] = (Tcw, Ow); K, bf, th and Scw are one value for
        every job or one per job.  Returns [(n_found, best_idx)] per job, equal to what Fuse returns."""
        n = len(kfs)
        assert n == len(points) == len(poses)
        Ks, bfs, ths, scws = _per_job(K, n, 1), _per_job(bf, n), _per_job(th, n), _per_job(Scw, n)
        jobs = (_FuseJobC * max(n, 1))()
        keep, outs = [], []
        for j in range(n):
            fv, pv, logs, _, k = self._points_call(kfs[j], points[j], with_stereo=not scws[j])
            inv = np.ascontiguousarray(kfs[j].mvInvLevelSigma2, np.float32) if kfs[j].mvInvLevelSigma2 is not None else None
            nq = len(points[j].world_pos)
            best = np.full(max(nq, 1), -1, np.int32)
            Tcw, Ow = poses[j]
            J = jobs[j]
            J.kf, J.inv_level_sigma2, J.pts, J.Tcw = fv, _p(inv), pv, _pose12(Tcw)
            J.Ow = (C.c_float * 3)(*np.asarray(Ow, np.float32).reshape(3).tolist())
            J.fx, J.fy, J.cx, J.cy = [float(x) for x in Ks[j]]
            J.bf, J.log_scale_factor, J.th, J.scw_variant, J.best_idx = float(bfs[j]), logs, float(ths[j]), int(scws[j]), _p(best)
            keep.append((k, inv)); outs.append((nq, best))
        nf = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_fuse_batch(self._h, jobs, n, _p(nf)), "borb_fuse_batch")
        return [(int(nf[j]), best[:nq]) for j, (nq, best) in enumerate(outs)]


def _sharing_order(cw, fw, seq, skip=()):
    """lKFsSharingWords: keyframes sharing a word with the query, in the order the inverted-file walk meets them — by first
    shared word id, then by insertion into that word's list (src/KeyFrameDatabase.cc:86-108, :211-224)."""
    s = [int(i) for i in np.nonzero(np.asarray(cw) > 0)[0] if int(i) not in skip]
    return sorted(s, key=lambda i: (int(fw[i]), seq[i]))


def relocalization_candidates(cw, sc, fw, seq, covisibility, reloc_score: Optional[dict] = None) -> list:
    """The host part of KeyFrameDatabase::DetectRelocalizationCandidates (src/KeyFrameDatabase.cc:226-310) from the per-keyframe
    shared-word counts `cw`, float L1 scores `sc` and first shared words `fw` (borb_kfdb_query).
    `reloc_score` is the database's persistent {slot: KeyFrame::mRelocScore}: the reference assigns mRelocScore only to keyframes
    above minCommonWords (:236-243) and the covisibility accumulation (:262-275) reads the field of EVERY neighbour that shares a
    word with the query — for a neighbour below the threshold that is the value an EARLIER query left there.  Passing the same
    dict to successive queries reproduces that; None (or a fresh dict) is a fresh database, where the field is 0."""
    if reloc_score is None:
        reloc_score = {}
    sharing = _sharing_order(cw, fw, seq)
    if not sharing:
        return []
    maxCommonWords = max(int(cw[s]) for s in sharing)
    minCommonWords = int(np.float32(maxCommonWords) * np.float32(0.8))
    scored = [(np.float32(sc[s]), s) for s in sharing if cw[s] > minCommonWords]
    for si, s in scored:
        reloc_score[s] = si                               # pKFi->mRelocScore = si (:241)
    if not scored:
        return []
    acc, bestAcc = [], np.float32(0)
    for si, s in scored:
        bestScore, accScore, best = si, si, s
        for s2 in covisibility(s):
            if cw[s2] <= 0:
                continue                                  # mnRelocQuery != F->mnId: shares no word with the query
            r = np.float32(reloc_score.get(s2, 0.0))      # pKF2->mRelocScore: this query's score, or the stale one (see above)
            accScore = np.float32(accScore + r)
            if r > bestScore:
                best, bestScore = s2, r
        acc.append((accScore, best))
        if accScore > bestAcc:
            bestAcc = accScore
    minScoreToRetain = np.float32(0.75) * bestAcc
    out, seen = [], set()
    for a, s in acc:
        if a > minScoreToRetain and s not in seen:
            out.append(s); seen.add(s)
    return out


def loop_candidates(cw, sc, fw, seq, connected, covisibility, minScore) -> list:
    """The host part of KeyFrameDatabase::DetectLoopCandidates (src/KeyFrameDatabase.cc:110-197); `connected` = slots of the
    query keyframe's connected keyframes (never candidates, :96-101)."""
    minScore = np.float32(minScore)
    sharing = _sharing_order(cw, fw, seq, skip=connected)
    if not sharing:
        return []
    maxCommonWords = max(int(cw[s]) for s in sharing)
    minCommonWords = int(np.float32(maxCommonWords) * np.float32(0.8))
    in_list = set(sharing)
    scored = [(np.float32(sc[s]), s) for s in sharing if cw[s] > minCommonWords and np.float32(sc[s]) >= minScore]
    if not scored:
        return []
    acc, bestAcc = [], minScore
    for si, s in scored:
        bestScore, accScore, best = si, si, s
        for s2 in covisibility(s):
            if s2 in in_list and cw[s2] > minCommonWords:                 # mnLoopQuery == pKF->mnId && mnLoopWords > minCommonWords (:157)
                r = np.float32(sc[s2])
                accScore = np.float32(accScore + r)
                if r > bestScore:
                    best, bestScore = s2, r
        acc.append((accScore, best))
        if accScore > bestAcc:
            bestAcc = accScore
    minScoreToRetain = np.float32(0.75) * bestAcc
    out, seen = [], set()
    for a, s in acc:
        if a > minScoreToRetain and s not in seen:
            out.append(s); seen.add(s)
    return out


def bow_and_featvec(word, weight, node):
    """The bookkeeping half of TemplatedVocabulary::transform (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1150-1194) from the
    per-feature results of the tree descent (word id, word weight, node id at level L-levelsup): BowVector::addWeight in
    feature order for every feature whose word weight is > 0 ("not stopped"), L1 normalisation with the norm summed in map
    (word id) order, FeatureVector::addFeature in feature order."""
    word = np.asarray(word); weight = np.asarray(weight, np.float64); node = np.asarray(node)
    bow: Dict[int, float] = {}
    keep = weight > 0
    for i in np.nonzero(keep)[0]:
        w = int(word[i])
        bow[w] = bow.get(w, 0.0) + float(weight[i])
    norm = 0.0                                   # plain left-to-right accumulation: Python >= 3.12's sum() is compensated, the
    for _, v in sorted(bow.items()):             # reference's `norm += fabs(it->second)` loop (BowVector.cpp:67-70) is not
        norm += abs(v)
    if norm > 0.0:
        bow = {k: v / norm for k, v in bow.items()}
    return dict(sorted(bow.items())), FeatureVector.from_nodes(node, keep)


def _bow_result(bw, bv, fn, fs, fi, nb: int, nn: int):
    """(mBowVec as {word: value}, mFeatVec) from the host copies of borb_compute_bow / borb_frames_compute_bow: nb words, nn nodes."""
    return dict(zip(bw[:nb].tolist(), bv[:nb].tolist())), FeatureVector(fn[:nn].copy(), fs[:nn + 1].copy(), fi[:fs[nn]].copy())


class KeyFrameDatabase:
    """KeyFrameDatabase (include/KeyFrameDatabase.h) with the keyframes resident in HBM.  add/erase/clear mirror
    src/KeyFrameDatabase.cc:41-73; query() is the data-parallel part of DetectLoopCandidates / DetectRelocalizationCandidates
    (shared-word count + L1 score for every keyframe in one launch); DetectRelocalizationCandidates() finishes the
    reference's procedure on the host from those arrays and the caller's covisibility lists."""

    def __init__(self, matcher: "ORBmatcher", device: int = 0):
        self._lib = _lib.load()
        self._m = matcher
        h = C.c_void_p()
        check(self._lib.borb_kfdb_create(device, C.byref(h)), "borb_kfdb_create")
        self._h = h
        self._seq = []                  # insertion sequence number per slot (inverted-file list order)
        self._reloc_score = {}          # KeyFrame::mRelocScore per slot, persistent across queries as in the reference
        self._n = []                    # features per slot (the default pair capacity of the searches from a slot)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.borb_kfdb_destroy(self._h)
            self._h = None

    @staticmethod
    def _bow_arrays(bow):
        w = np.fromiter(bow.keys(), np.uint32, len(bow)); v = np.fromiter(bow.values(), np.float64, len(bow))
        o = np.argsort(w, kind="stable")
        return np.ascontiguousarray(w[o]), np.ascontiguousarray(v[o])

    def add(self, pKF: KeyFrameView, mBowVec: Dict[int, float]) -> int:
        w, v = self._bow_arrays(mBowVec)
        slot = C.c_int32(-1)
        kc = pKF._c()
        check(self._lib.borb_kfdb_add(self._h, C.byref(kc), _p(w), _p(v), len(w), C.byref(slot)), "borb_kfdb_add")
        self._appended(len(pKF.mvKeysUn))
        return slot.value

    def _appended(self, n_features: int) -> None:
        """The host bookkeeping of a new slot (add() and ORBmatcher.KfdbAddFramesBatch): slots are handed out in call order."""
        self._seq.append(len(self._seq))
        self._n.append(n_features)

    def read_slot(self, slot: int) -> dict:
        """borb_debug_kfdb_read: what the database holds for a live slot — node, start, meta (row records, 2 u32 per row), desc (row
        order), bow_word, bow_value, host_meta (the host copy of the rows), block (the whole device block) and n (features)."""
        cnt = np.zeros(4, np.int32); nb = C.c_uint64(0)
        check(self._lib.borb_debug_kfdb_read(self._h, int(slot), _p(cnt), C.byref(nb), *([None] * 8)), "borb_debug_kfdb_read")
        nn, m, n, nbow = (int(x) for x in cnt)
        out = dict(node=np.zeros(max(nn, 1), np.uint32), start=np.zeros(nn + 1, np.int32), meta=np.zeros(max(2 * m, 1), np.uint32),
                   desc=np.zeros((max(m, 1), 32), np.uint8), bow_word=np.zeros(max(nbow, 1), np.uint32),
                   bow_value=np.zeros(max(nbow, 1), np.float64), host_meta=np.zeros(max(2 * m, 1), np.uint32),
                   block=np.zeros(nb.value, np.uint8))
        check(self._lib.borb_debug_kfdb_read(self._h, int(slot), None, None, *[_p(out[k]) for k in ("node", "start", "meta", "desc", "bow_word",
                                                                                                 "bow_value", "host_meta", "block")]),
              "borb_debug_kfdb_read")
        for k, ln in (("node", nn), ("meta", 2 * m), ("desc", m), ("bow_word", nbow), ("bow_value", nbow), ("host_meta", 2 * m)):
            out[k] = out[k][:ln]
        out["n"] = n
        return out

    def erase(self, slot: int) -> None:
        check(self._lib.borb_kfdb_erase(self._h, int(slot)), "borb_kfdb_erase")
        self._reloc_score.pop(int(slot), None)

    def clear(self) -> None:
        check(self._lib.borb_kfdb_clear(self._h), "borb_kfdb_clear")
        self._seq = []
        self._reloc_score = {}
        self._n = []

    def _n_features(self, slot: int) -> int:
        return self._n[slot] if 0 <= slot < len(self._n) else 0

    def set_has_mp(self, slot: int, has_mp: np.ndarray) -> None:
        hm = np.ascontiguousarray(has_mp, np.uint8)
        check(self._lib.borb_kfdb_set_has_mp(self._h, int(slot), _p(hm)), "borb_kfdb_set_has_mp")

    def set_has_mp_batch(self, slots, has_mps) -> None:
        """borb_kfdb_set_has_mp_batch: the MapPoint masks of several slots in one update that every search sees whole (a repeated
        slot takes its last mask).  A bad slot or a None mask anywhere refuses the whole batch and changes nothing."""
        sl = np.ascontiguousarray(slots, np.int32)
        keep = [np.ascontiguousarray(h, np.uint8) if h is not None else None for h in has_mps]
        assert len(keep) == len(sl)
        arr = (C.c_void_p * max(len(keep), 1))(*[h.ctypes.data if h is not None else None for h in keep])
        check(self._lib.borb_kfdb_set_has_mp_batch(self._h, len(sl), _p(sl), arr), "borb_kfdb_set_has_mp_batch")

    def size(self) -> Tuple[int, int]:
        n = C.c_int32(0); b = C.c_uint64(0)
        check(self._lib.borb_kfdb_size(self._h, C.byref(n), C.byref(b)), "borb_kfdb_size")
        return n.value, b.value

    def query(self, mBowVec: Dict[int, float]):
        """Returns (common_words[int32], score[float32], first_word[uint32]) with one entry per slot."""
        w, v = self._bow_arrays(mBowVec)
        ns = C.c_int32(self.size()[0])
        while True:              # sized again when another thread added keyframes since (refused before any launch)
            n = ns.value
            cw = np.zeros(max(n, 1), np.int32); sc = np.zeros(max(n, 1), np.float32); fw = np.zeros(max(n, 1), np.uint32)
            st = self._lib.borb_kfdb_query(self._m._h, self._h, _p(w), _p(v), len(w), _p(cw), _p(sc), _p(fw), len(cw), C.byref(ns))
            if not (st == BORB_ERR_CAPACITY and ns.value > len(cw)):
                break
        check(st, "borb_kfdb_query")
        return cw[:ns.value], sc[:ns.value], fw[:ns.value]

    def DetectRelocalizationCandidates(self, mBowVec: Dict[int, float], covisibility) -> list:
        """src/KeyFrameDatabase.cc:199-310.  covisibility(slot) -> up to 10 slots (GetBestCovisibilityKeyFrames(10))."""
        cw, sc, fw = self.query(mBowVec)
        return relocalization_candidates(cw, sc, fw, self._seq, covisibility, self._reloc_score)

    def DetectLoopCandidates(self, mBowVec: Dict[int, float], connected, covisibility, minScore: float) -> list:
        """src/KeyFrameDatabase.cc:76-197.  connected: slots of pKF->GetConnectedKeyFrames(); covisibility as above."""
        cw, sc, fw = self.query(mBowVec)
        return loop_candidates(cw, sc, fw, self._seq, set(int(c) for c in connected), covisibility, minScore)

    def SearchByBoW(self, slots, F: KeyFrameView):
        """SearchByBoW(pKF, F, vpMapPointMatches) (src/ORBmatcher.cc:159-288) for database keyframes `slots` against frame F."""
        sl = np.ascontiguousarray(slots, np.int32)
        fc = F._c()
        nF = len(F.mvKeysUn)
        match = np.full((len(sl), max(nF, 1)), -1, np.int32)
        nm = np.zeros(max(len(sl), 1), np.int32)
        m = self._m
        check(self._lib.borb_search_by_bow_db(m._h, self._h, _p(sl), len(sl), C.byref(fc), m.mfNNratio, int(m.mbCheckOrientation),
                                              _p(match), _p(nm)), "borb_search_by_bow_db")
        return nm[:len(sl)], match[:, :nF]


    def SearchByBoWPairs(self, slots, F: KeyFrameView, pairs_cap: Optional[int] = None, want_pairs: bool = True):
        """SearchByBoW of frame F against database keyframes `slots` (None = every slot) with compact results:
        returns (nmatches[n_kf], pair_offset[n_kf], pairs) where pairs[off[k]:off[k]+nm[k]] = (frame feature | keyframe feature << 16)."""
        m = self._m
        fc = F._c()
        if slots is None:
            n_kf, sl = self.size()[0], None
        else:
            sl = np.ascontiguousarray(slots, np.int32); n_kf = len(sl)
        nF = len(F.mvKeysUn)
        cap = int(pairs_cap) if pairs_cap is not None else max(n_kf * nF, 1)
        nm = np.zeros(max(n_kf, 1), np.int32); off = np.zeros(max(n_kf, 1), np.int32)
        pairs = np.zeros(cap if want_pairs else 1, np.uint32)
        tot = C.c_int32(0)
        check(self._lib.borb_search_by_bow_db_pairs(m._h, self._h, _p(sl), n_kf, C.byref(fc), m.mfNNratio, int(m.mbCheckOrientation), _p(nm),
                                                    _p(off), _p(pairs) if want_pairs else None, cap if want_pairs else 0, C.byref(tot)),
              "borb_search_by_bow_db_pairs")
        return nm[:n_kf], off[:n_kf], pairs[:tot.value] if want_pairs else None

    def SearchByBoWKFPairs(self, query_slot: int, slots, pairs_cap: Optional[int] = None):
        """SearchByBoW(KeyFrame*, KeyFrame*) (src/ORBmatcher.cc:522-655) of the keyframe in `query_slot` against the candidate slots
        `slots` (None = every slot), both read from the database with their current MapPoint masks: returns (nmatches[n_kf],
        pair_offset[n_kf], pairs) where pairs[off[k]:off[k]+nm[k]] = (query feature | candidate feature << 16) in the query's
        FeatureVector order."""
        m = self._m
        if slots is None:
            n_kf, sl = self.size()[0], None
        else:
            sl = np.ascontiguousarray(slots, np.int32); n_kf = len(sl)
        cap = int(pairs_cap) if pairs_cap is not None else max(n_kf * self._n_features(int(query_slot)), 1)
        nm = np.zeros(max(n_kf, 1), np.int32); off = np.zeros(max(n_kf, 1), np.int32)
        pairs = np.zeros(max(cap, 1), np.uint32)
        tot = C.c_int32(0)
        check(self._lib.borb_search_by_bow_kf_db_pairs(m._h, self._h, int(query_slot), _p(sl), n_kf, m.mfNNratio, int(m.mbCheckOrientation),
                                                       _p(nm), _p(off), _p(pairs), cap, C.byref(tot)),
              "borb_search_by_bow_kf_db_pairs")
        return nm[:n_kf], off[:n_kf], pairs[:tot.value]


class ORBVocabulary:
    """ORBVocabulary = DBoW2::TemplatedVocabulary<FORB> (include/ORBVocabulary.h), device resident."""

    def __init__(self, handle, lib):
        self._h, self._lib = handle, lib

    @staticmethod
    def from_arrays(parent, is_leaf, desc, weight, k: int, L: int, device: int = 0) -> "ORBVocabulary":
        lib = _lib.load()
        parent = np.ascontiguousarray(parent, np.int32); is_leaf = np.ascontiguousarray(is_leaf, np.uint8)
        desc = np.ascontiguousarray(desc, np.uint8); weight = np.ascontiguousarray(weight, np.float64)
        h = C.c_void_p()
        check(lib.borb_voc_create(_p(parent), _p(is_leaf), _p(desc), _p(weight), len(parent), k, L, device, C.byref(h)), "borb_voc_create")
        return ORBVocabulary(h, lib)

    @staticmethod
    def loadFromTextFile(path: str, device: int = 0) -> "ORBVocabulary":
        lib = _lib.load()
        h = C.c_void_p()
        check(lib.borb_voc_load_text(path.encode(), device, C.byref(h)), "borb_voc_load_text")
        return ORBVocabulary(h, lib)

    @staticmethod
    def from_blob(d_ptr: int, nbytes: int, device: int = 0) -> "ORBVocabulary":
        lib = _lib.load()
        h = C.c_void_p()
        check(lib.borb_voc_from_blob(C.c_void_p(d_ptr), nbytes, device, C.byref(h)), "borb_voc_from_blob")
        return ORBVocabulary(h, lib)

    def blob(self) -> Tuple[int, int]:
        p, n = C.c_void_p(), C.c_size_t()
        check(self._lib.borb_voc_blob(self._h, C.byref(p), C.byref(n)), "borb_voc_blob")
        return p.value, n.value

    def close(self):
        if getattr(self, "_h", None):
            self._lib.borb_voc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def transform_raw(self, descriptors: np.ndarray, levelsup: int = 4):
        """Per feature: word id, word weight, node id at level L-levelsup (TemplatedVocabulary.h:1218-1259)."""
        d = np.ascontiguousarray(descriptors, np.uint8)
        n = len(d)
        word = np.zeros(max(n, 1), np.int32); weight = np.zeros(max(n, 1), np.float64); node = np.zeros(max(n, 1), np.int32)
        check(self._lib.borb_bow_transform(self._h, _p(d), n, levelsup, _p(word), _p(weight), _p(node)), "borb_bow_transform")
        return word[:n], weight[:n], node[:n]

    def ComputeBoW(self, descriptors: np.ndarray, levelsup: int = 4):
        """Frame::ComputeBoW (src/Frame.cc:395-402) through borb_compute_bow: (mBowVec as {word: value}, mFeatVec), the tree
        descent and the ordered-map bookkeeping both on the device — same results as transform() below.  At most 8192 features."""
        d = np.ascontiguousarray(descriptors, np.uint8)
        n = len(d)
        bw = np.zeros(max(n, 1), np.uint32); bv = np.zeros(max(n, 1), np.float64)
        fn = np.zeros(max(n, 1), np.uint32); fs = np.zeros(n + 1, np.int32); fi = np.zeros(max(n, 1), np.uint32)
        nb, nn = C.c_int32(0), C.c_int32(0)
        check(self._lib.borb_compute_bow(self._h, _p(d), n, levelsup, _p(bw), _p(bv), C.byref(nb), _p(fn), _p(fs), _p(fi), C.byref(nn)), "borb_compute_bow")
        return _bow_result(bw, bv, fn, fs, fi, nb.value, nn.value)

    def transform(self, descriptors: np.ndarray, levelsup: int = 4):
        """transform(features, BowVector, FeatureVector, levelsup) (:1127-1194) for TF-IDF / L1 (ORBvoc.txt "10 6 0 0"):
        the tree descent runs on the GPU; the ordered-map bookkeeping is done on the host in feature order, as the reference does."""
        return bow_and_featvec(*self.transform_raw(descriptors, levelsup))
