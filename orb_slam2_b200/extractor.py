"""Host-side mirror of ORB_SLAM2::ORBextractor (reference include/ORBextractor.h:45-111) over libborb.

Same constructor arguments, call operator, getters and the public ``mvImagePyramid`` member as the
reference class, so parity tests read like calls into the reference; plus the batched entry points
(many independent frames per launch) that the design is built around.  All compute happens in
the CUDA library; this module only marshals numpy buffers through the C ABI.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import KP_DTYPE, ExtractorCfg, check, ptr

STAGES = ("upload", "pyramid", "fast_nms", "quadtree", "blur", "orient_brief", "stereo", "download")


class ORBextractor:
    """ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST) — ORBextractor.h:53-54."""

    HARRIS_SCORE = 0
    FAST_SCORE = 1

    def __init__(self, nfeatures: int = 2000, scaleFactor: float = 1.2, nlevels: int = 8, iniThFAST: int = 20,
                 minThFAST: int = 7, device: int = 0):
        self._lib = _lib.load()
        self.nfeatures, self.nlevels = int(nfeatures), int(nlevels)
        self.scaleFactor = float(np.float32(scaleFactor))
        self.iniThFAST, self.minThFAST = int(iniThFAST), int(minThFAST)
        self.device = int(device)
        cfg = ExtractorCfg(self.nfeatures, scaleFactor, self.nlevels, self.iniThFAST, self.minThFAST)
        h = C.c_void_p()
        check(self._lib.borb_extractor_create(C.byref(cfg), self.device, C.byref(h)), "borb_extractor_create")
        self._h = h
        L = self.nlevels
        self._scale = np.zeros(L, np.float32); self._inv_scale = np.zeros(L, np.float32)
        self._sigma2 = np.zeros(L, np.float32); self._inv_sigma2 = np.zeros(L, np.float32)
        self.mnFeaturesPerLevel = np.zeros(L, np.int32)
        f32p, i32p = _lib.f32p, _lib.i32p
        check(self._lib.borb_extractor_tables(self._h, self._scale.ctypes.data_as(f32p), self._inv_scale.ctypes.data_as(f32p),
                                              self._sigma2.ctypes.data_as(f32p), self._inv_sigma2.ctypes.data_as(f32p),
                                              self.mnFeaturesPerLevel.ctypes.data_as(i32p)), "borb_extractor_tables")
        self._last_n = 0
        self._keep = []      # host buffers referenced by an enqueue in flight

    def close(self):
        if getattr(self, "_h", None):
            self._lib.borb_extractor_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- getters (ORBextractor.h:63-83)
    def GetLevels(self) -> int: return self.nlevels
    def GetScaleFactor(self) -> float: return self.scaleFactor
    def GetScaleFactors(self) -> np.ndarray: return self._scale.copy()
    def GetInverseScaleFactors(self) -> np.ndarray: return self._inv_scale.copy()
    def GetScaleSigmaSquares(self) -> np.ndarray: return self._sigma2.copy()
    def GetInverseScaleSigmaSquares(self) -> np.ndarray: return self._inv_sigma2.copy()

    def _work_capacity(self, raw_w: int, raw_h: int) -> int:
        """Output capacity for frames of raw size (raw_w, raw_h): with rectification maps installed the extractor works on the
        maps' destination size, which may differ from the raw frame's."""
        rs = getattr(self, "_rect_size", None)
        return self.capacity(*rs) if rs is not None else self.capacity(raw_w, raw_h)

    def capacity(self, width: int, height: int) -> int:
        cap = C.c_int32()
        check(self._lib.borb_extractor_capacity(self._h, width, height, C.byref(cap)), "borb_extractor_capacity")
        return cap.value

    def reserve(self, width: int, height: int, max_images: int) -> None:
        check(self._lib.borb_extractor_reserve(self._h, width, height, max_images), "borb_extractor_reserve")

    # ---- operator() (ORBextractor.cc:1043): image -> (keypoints[N] KP_DTYPE, descriptors[N,32] u8)
    def set_input_format(self, channels: int, mbRGB: bool = True) -> None:
        """Colour frames (H, W, 3|4) are converted to gray on the GPU exactly as Tracking::GrabImage* does with cv::cvtColor
        (src/Tracking.cc:172-197); mbRGB = Camera.RGB of the settings file (1: RGB order, 0: BGR)."""
        self.mbRGB = bool(mbRGB)
        self._set_format(channels)

    def set_rectify_maps(self, which: int, map_x: Optional[np.ndarray], map_y: Optional[np.ndarray], src_size: Optional[Tuple[int, int]] = None) -> None:
        """cv::remap(im, imRect, M1, M2, INTER_LINEAR) of Examples/Stereo/stereo_euroc.cc:136-137 fused into the upload.  which: 0 mono /
        left, 1 right; map_x / map_y: (dst_h, dst_w) float32 maps from cv::initUndistortRectifyMap; src_size = (w, h) of the raw
        frames (default: same as the maps).  None removes the maps."""
        if map_x is None or map_y is None:
            check(self._lib.borb_extractor_set_rectify_maps(self._h, int(which), None, None, 0, 0, 0, 0), "borb_extractor_set_rectify_maps")
            if which == 0:
                self._rect_size = None
            return
        mx = np.ascontiguousarray(map_x, np.float32); my = np.ascontiguousarray(map_y, np.float32)
        assert mx.shape == my.shape and mx.ndim == 2
        dh, dw = mx.shape
        sw, sh = src_size if src_size is not None else (dw, dh)
        check(self._lib.borb_extractor_set_rectify_maps(self._h, int(which), ptr(mx), ptr(my), int(sw), int(sh), dw, dh),
              "borb_extractor_set_rectify_maps")
        if which == 0:
            self._rect_size = (dw, dh)

    def _set_format(self, channels: int) -> None:
        key = (int(channels), bool(getattr(self, "mbRGB", True)))
        if getattr(self, "_fmt", (1, True)) != key:
            check(self._lib.borb_extractor_set_input_format(self._h, key[0], int(key[1])), "borb_extractor_set_input_format")
            self._fmt = key

    def __call__(self, image: np.ndarray, mask=None) -> Tuple[np.ndarray, np.ndarray]:
        if image is None or image.size == 0:
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim in (2, 3), "CV_8UC1 expected (ORBextractor.cc:1050); 3/4 channels: see set_input_format"
        ch = 1 if image.ndim == 2 else image.shape[2]
        self._set_format(ch)
        if image.strides[-1] != 1 or (ch > 1 and image.strides[1] != ch):
            image = np.ascontiguousarray(image)
        h, w = image.shape[:2]
        cap = self._work_capacity(w, h)
        kps = np.zeros(cap, KP_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int32(0)
        check(self._lib.borb_extract(self._h, ptr(image), w, h, image.strides[0], ptr(kps), ptr(desc), cap, C.byref(n)), "borb_extract")
        self._last_n = 1
        return kps[:n.value].copy(), desc[:n.value].copy()

    # ---- batched: list of equally-sized images
    def extract_batch(self, images: Sequence[np.ndarray]) -> List[Tuple[np.ndarray, np.ndarray]]:
        n = len(images)
        if n == 0:
            return []
        images = [np.ascontiguousarray(im, np.uint8) for im in images]
        h, w = images[0].shape[:2]
        assert all(im.shape == images[0].shape for im in images), "a batch holds images of one size"
        self._set_format(1 if images[0].ndim == 2 else images[0].shape[2])
        cap = self._work_capacity(w, h)
        kps = np.zeros((n, cap), KP_DTYPE)
        desc = np.zeros((n, cap, 32), np.uint8)
        cnt = np.zeros(n, np.int32)
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in images])
        check(self._lib.borb_extract_batch(self._h, ptrs, n, w, h, images[0].strides[0], ptr(kps), ptr(desc), cap, ptr(cnt)),
              "borb_extract_batch")
        self._last_n = n
        return [(kps[i, :cnt[i]].copy(), desc[i, :cnt[i]].copy()) for i in range(n)]

    def extract_enqueue(self, image: np.ndarray) -> None:
        """borb_extract_batch_enqueue of one CV_8UC1 image with no host copies: the keypoints stay on the device for
        matcher.frame_from_extractors (the Frame constructors' ExtractORB, src/Frame.cc:247-253)."""
        image = np.ascontiguousarray(image, np.uint8)
        assert image.ndim == 2, "CV_8UC1 expected"
        self._set_format(1)
        h, w = image.shape
        ptrs = (C.c_void_p * 1)(image.ctypes.data)
        check(self._lib.borb_extract_batch_enqueue(self._h, ptrs, 1, w, h, image.strides[0], None, None, 0, None),
              "borb_extract_batch_enqueue")
        self._last_n = 1

    # ---- mvImagePyramid (ORBextractor.h:85) of image `image` of the last call
    def pyramid(self, level: int, image: int = 0) -> np.ndarray:
        w, h = C.c_int32(), C.c_int32()
        check(self._lib.borb_extractor_pyramid(self._h, image, level, None, C.byref(w), C.byref(h)), "borb_extractor_pyramid")
        out = np.zeros((h.value, w.value), np.uint8)
        check(self._lib.borb_extractor_pyramid(self._h, image, level, ptr(out), C.byref(w), C.byref(h)), "borb_extractor_pyramid")
        return out

    @property
    def mvImagePyramid(self) -> List[np.ndarray]:
        return [self.pyramid(l, 0) for l in range(self.nlevels)]

    # ---- stereo (Frame::ComputeStereoMatches, Frame.cc:466) on the last batch
    def stereo_match(self, n_pairs: int, bf: float, fx: float, left_idx=None, right_idx=None):
        b = np.float32(bf) / np.float32(fx)       # mb = mbf/fx (Frame.cc:114)
        cap = self.capacity(*self._shape())
        ur = np.zeros((n_pairs, cap), np.float32)
        dp = np.zeros((n_pairs, cap), np.float32)
        li = np.ascontiguousarray(left_idx, np.int32) if left_idx is not None else None
        ri = np.ascontiguousarray(right_idx, np.int32) if right_idx is not None else None
        check(self._lib.borb_stereo_match(self._h, n_pairs, ptr(li), ptr(ri), float(bf), float(b), ptr(ur), ptr(dp), cap),
              "borb_stereo_match")
        return ur, dp

    def _shape(self):
        w, h = C.c_int32(), C.c_int32()
        check(self._lib.borb_extractor_pyramid(self._h, 0, 0, None, C.byref(w), C.byref(h)), "borb_extractor_pyramid")
        return w.value, h.value

    def stereo_frames(self, lefts: Sequence[np.ndarray], rights: Sequence[np.ndarray], bf: float, fx: float):
        """Frame::Frame stereo ctor hot path for a batch of pairs (Frame.cc:61-117): returns a list of dicts
        with mvKeys, mDescriptors, mvKeysRight, mDescriptorsRight, mvuRight, mvDepth."""
        n = len(lefts)
        assert n == len(rights) and n > 0
        lefts = [np.ascontiguousarray(im, np.uint8) for im in lefts]
        rights = [np.ascontiguousarray(im, np.uint8) for im in rights]
        h, w = lefts[0].shape
        cap = self._work_capacity(w, h)
        b = np.float32(bf) / np.float32(fx)
        kl = np.zeros((n, cap), KP_DTYPE); kr = np.zeros((n, cap), KP_DTYPE)
        dl = np.zeros((n, cap, 32), np.uint8); dr = np.zeros((n, cap, 32), np.uint8)
        nl = np.zeros(n, np.int32); nr = np.zeros(n, np.int32)
        ur = np.zeros((n, cap), np.float32); dp = np.zeros((n, cap), np.float32)
        pl = (C.c_void_p * n)(*[im.ctypes.data for im in lefts])
        pr = (C.c_void_p * n)(*[im.ctypes.data for im in rights])
        check(self._lib.borb_stereo_frames(self._h, pl, pr, n, w, h, lefts[0].strides[0], float(bf), float(b), ptr(kl), ptr(dl),
                                           ptr(nl), ptr(kr), ptr(dr), ptr(nr), ptr(ur), ptr(dp), cap), "borb_stereo_frames")
        self._last_n = 2 * n
        out = []
        for i in range(n):
            out.append(dict(mvKeys=kl[i, :nl[i]].copy(), mDescriptors=dl[i, :nl[i]].copy(),
                            mvKeysRight=kr[i, :nr[i]].copy(), mDescriptorsRight=dr[i, :nr[i]].copy(),
                            mvuRight=ur[i, :nl[i]].copy(), mvDepth=dp[i, :nl[i]].copy()))
        return out

    # ---- per-stage intermediates of the last batch (parity tests)
    def _debug_list(self, fn, image, level):
        n = C.c_int32()
        check(fn(self._h, image, level, None, 0, C.byref(n)), "borb_debug")
        out = np.zeros((max(n.value, 1), 3), np.int32)
        check(fn(self._h, image, level, ptr(out), n.value, C.byref(n)), "borb_debug")
        return out[:n.value]

    def debug_candidates(self, level: int, image: int = 0) -> np.ndarray:
        return self._debug_list(self._lib.borb_debug_candidates, image, level)

    def debug_selected(self, level: int, image: int = 0) -> np.ndarray:
        return self._debug_list(self._lib.borb_debug_selected, image, level)

    def debug_blurred(self, level: int, image: int = 0) -> np.ndarray:
        w, h = C.c_int32(), C.c_int32()
        check(self._lib.borb_debug_blurred(self._h, image, level, None, C.byref(w), C.byref(h)), "borb_debug_blurred")
        out = np.zeros((h.value, w.value), np.uint8)
        check(self._lib.borb_debug_blurred(self._h, image, level, ptr(out), C.byref(w), C.byref(h)), "borb_debug_blurred")
        return out

    def launch_count(self) -> int:
        n = C.c_uint64()
        check(self._lib.borb_launch_count(self._h, C.byref(n)), "borb_launch_count")
        return n.value

    def set_timing(self, on: bool) -> None:
        check(self._lib.borb_set_timing(self._h, int(on)), "borb_set_timing")

    def stage_times(self) -> dict:
        ms = np.zeros(8, np.float32)
        check(self._lib.borb_stage_times(self._h, ms.ctypes.data_as(_lib.f32p)), "borb_stage_times")
        return dict(zip(STAGES, ms.tolist()))
