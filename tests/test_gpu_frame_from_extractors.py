"""GPU: borb_frame_from_extractors, one Frame constructor (src/Frame.cc:61-117 stereo, :119-178 RGB-D, :180-233 monocular) on the
frame's own extractor handles after their extractions were enqueued.  Every host member it returns equals what the existing entry
points return for the same images — the extraction (borb_extract_batch), the two-handle association (borb_stereo_match2), the
constructor tail (borb_frames_from_extractor) and the feature grid of the resident frame (borb_debug_frame_read) — each of which
other tests pin to the port and the verbatim reference; the resident frame searches as its host view does; refusals name the
argument."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import frame_input_cases as fic

pytestmark = pytest.mark.gpu

KITTI_K = (718.856, 718.856, 607.1928, 185.2157)
KITTI_BF = 386.1448
EUROC_K = (435.2047, 435.2047, 367.4517, 252.2005)
EUROC_BF = 47.90639384423901


def _M():
    from orb_slam2_b200 import matcher as M
    return M


def _X(n, **kw):
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor(n, **kw)


def _grid(F):
    g = F.resident.read(stereo=False)
    return g["cell_start"], g["cell_idx"], g["keys_un"]


def _check_grid(F, host):
    cs, ci, ku = _grid(F)
    assert np.array_equal(host["cell_start"], cs) and np.array_equal(host["cell_idx"], ci)
    assert np.array_equal(host["mvKeysUn"], ku)


def _stereo_reference(L, R, nl, nr, K, bf):
    """mvKeys / mvKeysRight from borb_extract_batch on two fresh handles, mvuRight / mvDepth from borb_stereo_match2 on them."""
    from orb_slam2_b200 import _lib
    GL, GR = _X(nl), _X(nr)
    (kl, dl), = GL.extract_batch([L])
    (kr, dr), = GR.extract_batch([R])
    cap = max(GL.capacity(*L.shape[::-1]), 1)
    ur = np.zeros(cap, np.float32); dp = np.zeros(cap, np.float32)
    b = np.float32(bf) / np.float32(K[0])
    _lib.check(_lib.load().borb_stereo_match2(GL._h, GR._h, float(bf), float(b), _lib.ptr(ur), _lib.ptr(dp), cap), "borb_stereo_match2")
    return kl, dl, kr, dr, ur[:len(kl)], dp[:len(kl)]


def _stereo_ctor(L, R, nl, nr, K, bf, mt=None):
    M = _M()
    XL, XR = _X(nl), _X(nr)
    XL.extract_enqueue(L)
    XR.extract_enqueue(R)
    return M.frame_from_extractors(mt or M.ORBmatcher(0.8, True), XL, XR, K, bf=bf, mode=1)


@pytest.mark.parametrize("shape,nl,nr,K,bf", [((1242, 375), 2000, 2000, KITTI_K, KITTI_BF),
                                              ((752, 480), 1200, 1500, EUROC_K, EUROC_BF),
                                              ((752, 480), 1500, 1200, EUROC_K, EUROC_BF)],
                         ids=["kitti_2000", "euroc_1200_1500", "euroc_1500_1200"])
def test_stereo_constructor(shape, nl, nr, K, bf):
    L, R, _ = synth.stereo_pair(7, 0, 0, *shape)
    F, host = _stereo_ctor(L, R, nl, nr, K, bf)
    kl, dl, kr, dr, ur, dp = _stereo_reference(L, R, nl, nr, K, bf)
    assert len(kl) > 500 and len(kr) > 500 and (ur >= 0).sum() > 100
    assert np.array_equal(host["mvKeys"], kl) and np.array_equal(host["mDescriptors"], dl)
    assert np.array_equal(host["mvKeysRight"], kr) and np.array_equal(host["mDescriptorsRight"], dr)
    assert np.array_equal(host["mvKeysUn"], kl)                   # no distortion: mvKeysUn = mvKeys (Frame.cc:406-410)
    assert np.array_equal(host["mvuRight"], ur) and np.array_equal(host["mvDepth"], dp)
    _check_grid(F, host)
    dev = F.resident.read(stereo=True)
    assert np.array_equal(dev["u_right"], ur) and np.array_equal(dev["depth"], dp)
    assert host["bounds"] == (0.0, 0.0, float(shape[0]), float(shape[1]))
    F.resident.close()


def test_stereo_constructor_empty_images_on_reused_handles():
    """On the same two handles, frame after frame (the counts change between calls and are only read on the device): a full
    pair, a right image without keypoints (every mvuRight -1), a blank left image (N = 0: every per-feature member empty, an
    empty grid), then a full pair again, each equal to the separate entry points."""
    M = _M()
    L, R, _ = synth.stereo_pair(3, 0, 0, 752, 480)
    L2, R2, _ = synth.stereo_pair(5, 0, 0, 752, 480)
    blank = np.zeros_like(L)
    XL, XR, mt = _X(1200), _X(1300), M.ORBmatcher(0.8, True)
    for left, right in ((L, R), (L, blank), (blank, R), (L2, R2)):
        XL.extract_enqueue(left)
        XR.extract_enqueue(right)
        F, host = M.frame_from_extractors(mt, XL, XR, EUROC_K, bf=EUROC_BF, mode=1)
        kl, dl, kr, dr, ur, dp = _stereo_reference(left, right, 1200, 1300, EUROC_K, EUROC_BF)
        assert np.array_equal(host["mvKeys"], kl) and np.array_equal(host["mDescriptors"], dl)
        assert np.array_equal(host["mvKeysRight"], kr) and np.array_equal(host["mDescriptorsRight"], dr)
        assert np.array_equal(host["mvKeysUn"], kl)
        assert np.array_equal(host["mvuRight"], ur) and np.array_equal(host["mvDepth"], dp)
        _check_grid(F, host)
        if right is blank:
            assert len(kl) > 500 and len(kr) == 0 and np.all(ur == -1.0) and np.all(dp == -1.0)
        if left is blank:
            assert len(kr) > 500 and len(host["mvKeys"]) == 0 and len(host["mvKeysUn"]) == 0
            assert len(host["mvuRight"]) == 0 and len(host["mvDepth"]) == 0
            assert np.all(host["cell_start"] == 0) and len(host["cell_idx"]) == 0
            n = C.c_int32()
            assert F.resident._lib.borb_frame_info(F.resident._h, C.byref(n), None, None) == 0 and n.value == 0
        F.resident.close()


def test_rgbd_constructor():
    """TUM-shaped RGB-D with k1 != 0 and a raw CV_16U depth map with mDepthMapFactor, against borb_frames_from_extractor."""
    M = _M()
    K, dist = fic.DIST_CASES["tum1_5"]
    img = synth.mono_frame(11, 0, 0, 640, 480)
    raw = fic.edge_depth_raw(5)
    factor = 1.0 / 5000.0
    X = _X(1000)
    X.extract_enqueue(img)
    mt = M.ORBmatcher(0.8, True)
    F, host = M.frame_from_extractors(mt, X, None, K, dist, bf=40.0, mode=2, depth=raw, depth_factor=factor)
    X2 = _X(1000)
    (k, d), = X2.extract_batch([img])
    (G,), ref = M.frames_from_extractor(mt, X2, [0], [len(k)], K, dist, bf=40.0, mode=2, depth=[raw], depth_factor=factor)
    assert np.array_equal(host["mvKeys"], k) and np.array_equal(host["mDescriptors"], d) and len(host["mvKeysRight"]) == 0
    assert np.array_equal(host["mvKeysUn"], ref["keys_un"][0]) and not np.array_equal(host["mvKeysUn"], k)
    assert np.array_equal(host["mvuRight"], ref["u_right"][0]) and np.array_equal(host["mvDepth"], ref["depth"][0])
    assert (host["mvDepth"] > 0).sum() > 100
    assert np.array_equal(np.float32(host["bounds"]), ref["bounds"])
    _check_grid(F, host)
    assert np.array_equal(host["cell_start"], _grid(G)[0]) and np.array_equal(host["cell_idx"], _grid(G)[1])
    F.resident.close(); G.resident.close()


def test_monocular_constructor_initialisation_extractor():
    """Monocular with the initialisation extractor (2 x nFeatures, src/Tracking.cc:158-159), distorted camera."""
    M = _M()
    K, dist = fic.DIST_CASES["tum1_5"]
    img = synth.mono_frame(12, 0, 0, 640, 480)
    X = _X(4000)
    X.extract_enqueue(img)
    mt = M.ORBmatcher(0.9, True)
    F, host = M.frame_from_extractors(mt, X, None, K, dist)
    X2 = _X(4000)
    (k, d), = X2.extract_batch([img])
    (G,), ref = M.frames_from_extractor(mt, X2, [0], [len(k)], K, dist)
    assert len(k) > 2000
    assert np.array_equal(host["mvKeys"], k) and np.array_equal(host["mDescriptors"], d)
    assert np.array_equal(host["mvKeysUn"], ref["keys_un"][0])
    assert np.all(host["mvuRight"] == -1.0) and np.all(host["mvDepth"] == -1.0)       # Frame.cc:219-220
    _check_grid(F, host)
    assert np.array_equal(host["cell_start"], _grid(G)[0]) and np.array_equal(host["cell_idx"], _grid(G)[1])
    F.resident.close(); G.resident.close()


def test_resident_frame_searches_like_its_host_view():
    """SearchByProjection on the resident frame the constructor made equals the same search on its host members."""
    M = _M()
    L, R, _ = synth.stereo_pair(9, 0, 0, 1242, 375)
    mt = M.ORBmatcher(0.8, True)
    F, host = _stereo_ctor(L, R, 2000, 2000, KITTI_K, KITTI_BF, mt)
    kl = host["mvKeys"]
    ur = host["mvuRight"]
    rng = np.random.default_rng(0)
    sel = np.nonzero(ur >= 0)[0][:400]
    mps = M.MapPointsView((kl["x"][sel] + rng.normal(0, 1.0, len(sel))).astype(np.float32),
                          (kl["y"][sel] + rng.normal(0, 1.0, len(sel))).astype(np.float32),
                          (ur[sel] + rng.normal(0, 1.0, len(sel))).astype(np.float32),
                          kl["octave"][sel].astype(np.int32), np.full(len(sel), 0.9, np.float32), host["mDescriptors"][sel])
    V = M.FrameView(host["mvKeysUn"], host["mDescriptors"], F.mvScaleFactors, host["bounds"], mvuRight=ur)
    n_r, m_r = mt.SearchByProjection(F, mps, 3.0)
    n_h, m_h = mt.SearchByProjection(V, mps, 3.0)
    assert n_r == n_h and np.array_equal(m_r, m_h) and n_r > 100
    F.resident.close()


def test_refusals():
    from orb_slam2_b200 import _lib
    M = _M()
    so = _lib.load()
    mt = M.ORBmatcher(0.8, True)
    L, R, _ = synth.stereo_pair(4, 0, 0, 752, 480)
    XL, XR, fresh = _X(1200), _X(1200), _X(1200)
    cam = M._CameraC(*EUROC_K, 0, 0, 0, 0, 0, EUROC_BF)
    cap = XL.capacity(752, 480)
    host = M._FrameHostC(cap)
    out = C.c_void_p()

    def call(left, right, mode=1, b=0.11, h=host, m=mt._h, depth=None):
        return so.borb_frame_from_extractors(m, left, right, C.byref(cam), mode, b, depth, 0, 1.0, 0, C.byref(h) if h is not None else None,
                                             C.byref(out))

    def refused(status, text, **kw):
        args = {k: kw.pop(k) for k in ("left", "right") if k in kw}
        assert call(args.get("left", XL._h), args.get("right", XR._h), **kw) == status
        assert text in so.borb_last_error().decode(), so.borb_last_error()
        assert not out.value

    refused(6, "no extracted batch")                                 # neither handle has extracted anything yet
    XL.extract_enqueue(L); XR.extract_enqueue(R)
    refused(1, "argument: m", m=None)
    refused(1, "argument: left", left=None)
    refused(1, "argument: host", h=None)
    refused(1, "right", right=None)                                  # stereo without a right handle
    refused(1, "right", mode=0)                                      # monocular with one
    refused(1, "right", right=XL._h)
    refused(1, "b:", b=0.0)
    refused(6, "before extract", right=fresh._h)
    refused(1, "bad mode", mode=2, right=None)                       # RGB-D without a depth map
    refused(5, "host->cap", h=M._FrameHostC(cap - 1))                # below the handles' capacity
    small = _X(1200)
    small.extract_enqueue(np.ascontiguousarray(R[:, :640]))
    refused(1, "geometry", right=small._h)
    assert call(XL._h, XR._h) == 0 and out.value and host.n > 0 and host.n_right > 0
    assert so.borb_frame_destroy(out) == 0
