"""GPU parity for Frame::ComputeStereoMatches (reference src/Frame.cc:466-640) through the C ABI."""
import ctypes as C
import os

import numpy as np
import pytest

from orb_slam2_b200 import synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BF, FX = 386.1448, 718.856          # Examples/Stereo/KITTI00-02.yaml Camera.bf / Camera.fx


@pytest.fixture(scope="module")
def X():
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor


def oracle_stereo(oracle, L, R, nf, bf=BF, fx=FX):
    EL, ER = oracle.PortExtractor(nf), oracle.PortExtractor(nf)
    kl, dl = EL(L)
    kr, dr = ER(R)
    ur, dp, sad = oracle.port_stereo(kl, dl, kr, dr, [EL.level(i) for i in range(8)], [ER.level(i) for i in range(8)],
                                     EL.scale, EL.inv_scale, bf, fx)
    return kl, dl, kr, dr, ur, dp


def test_matches_golden_stereo(X):
    g = np.load(os.path.join(GOLD, "stereo_kitti_2000.npz"))
    w, h, nf, seed = g["meta"].tolist()
    bf, fx = g["cam"].tolist()
    L, R, _ = synth.stereo_pair(seed, 0, 0, w, h)
    out = X(nf).stereo_frames([L], [R], bf, fx)[0]
    assert np.array_equal(out["mvKeys"], g["kl"]) and np.array_equal(out["mDescriptors"], g["dl"])
    assert np.array_equal(out["mvKeysRight"], g["kr"]) and np.array_equal(out["mDescriptorsRight"], g["dr"])
    dev = np.abs(out["mvuRight"] - g["u_right"]).max()
    assert dev <= 1e-4 and np.array_equal(out["mvuRight"], g["u_right"]), dev
    assert np.array_equal(out["mvDepth"], g["depth"])


@pytest.mark.parametrize("shape,nf,cam", [(synth.KITTI, 2000, (BF, FX)), (synth.EUROC, 1200, (47.90639384423901, 435.2046959714599)),
                                          ((640, 480), 1000, (40.0, 525.0))])
def test_matches_oracle_batched_pairs(X, oracle, shape, nf, cam):
    w, h = shape
    bf, fx = cam
    pairs = [synth.stereo_pair(300 + i, 0, 0, w, h) for i in range(3)]
    outs = X(nf).stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], bf, fx)
    for (L, R, _), out in zip(pairs, outs):
        kl, dl, kr, dr, ur, dp = oracle_stereo(oracle, L, R, nf, bf, fx)
        assert np.array_equal(out["mvKeys"], kl) and np.array_equal(out["mvKeysRight"], kr)
        assert np.array_equal(out["mDescriptors"], dl) and np.array_equal(out["mDescriptorsRight"], dr)
        assert (ur >= 0).sum() > 100
        assert np.array_equal(out["mvuRight"], ur), int((out["mvuRight"] != ur).sum())
        assert np.array_equal(out["mvDepth"], dp)
        assert np.all(out["mvuRight"][ur < 0] == -1.0) and np.all(out["mvDepth"][ur < 0] == -1.0)   # sentinel contract


def test_two_handle_path_equals_batched_path(X, oracle):
    """mpORBextractorLeft / mpORBextractorRight as separate objects (Frame.cc:78-81) + borb_stereo_match2."""
    from orb_slam2_b200 import _lib
    L, R, _ = synth.stereo_pair(400, 0, 0)
    GL, GR = X(2000), X(2000)
    kl, dl = GL(L)
    kr, dr = GR(R)
    cap = GL.capacity(*synth.KITTI)
    ur = np.zeros(cap, np.float32); dp = np.zeros(cap, np.float32)
    b = np.float32(BF) / np.float32(FX)
    _lib.check(_lib.load().borb_stereo_match2(GL._h, GR._h, float(BF), float(b), _lib.ptr(ur), _lib.ptr(dp), cap), "borb_stereo_match2")
    want = X(2000).stereo_frames([L], [R], BF, FX)[0]
    assert np.array_equal(ur[:len(kl)], want["mvuRight"]) and np.array_equal(dp[:len(kl)], want["mvDepth"])
    _, _, _, _, our, odp = oracle_stereo(oracle, L, R, 2000)
    assert np.array_equal(ur[:len(kl)], our) and np.array_equal(dp[:len(kl)], odp)


def test_results_of_the_device_resident_call_read_back_equal_the_host_call(X):
    """borb_stereo_frames_device leaves keypoints, descriptors and the association in HBM; borb_stereo_frames_results copies
    them out afterwards and they equal what borb_stereo_frames returns for the same pairs."""
    import torch
    from orb_slam2_b200 import _lib
    from orb_slam2_b200._lib import KP_DTYPE
    lib = _lib.load()
    w, h = synth.KITTI
    pairs = [synth.stereo_pair(500 + i, 0, 0, w, h) for i in range(2)]
    G = X(2000)
    cap = G.capacity(w, h)
    d_img = torch.from_numpy(np.stack([im for p in pairs for im in p[:2]])).cuda()
    b = float(np.float32(BF) / np.float32(FX))
    nl, nr = np.zeros(2, np.int32), np.zeros(2, np.int32)
    _lib.check(lib.borb_stereo_frames_device(G._h, d_img.data_ptr(), 2, w, h, w, w * h, BF, b, _lib.ptr(nl), _lib.ptr(nr), None, None, cap),
               "borb_stereo_frames_device")
    kl, kr = np.zeros((2, cap), KP_DTYPE), np.zeros((2, cap), KP_DTYPE)
    dl, dr = np.zeros((2, cap, 32), np.uint8), np.zeros((2, cap, 32), np.uint8)
    ml, mr = np.zeros(2, np.int32), np.zeros(2, np.int32)
    ur, dp = np.zeros((2, cap), np.float32), np.zeros((2, cap), np.float32)
    _lib.check(lib.borb_stereo_frames_results(G._h, 2, kl.ctypes.data, dl.ctypes.data, ml.ctypes.data, kr.ctypes.data, dr.ctypes.data,
                                              mr.ctypes.data, ur.ctypes.data, dp.ctypes.data, cap), "borb_stereo_frames_results")
    assert np.array_equal(ml, nl) and np.array_equal(mr, nr)
    want = X(2000).stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], BF, FX)
    for p, o in enumerate(want):
        n, m = nl[p], nr[p]
        assert np.array_equal(kl[p, :n], o["mvKeys"]) and np.array_equal(dl[p, :n], o["mDescriptors"])
        assert np.array_equal(kr[p, :m], o["mvKeysRight"]) and np.array_equal(dr[p, :m], o["mDescriptorsRight"])
        assert np.array_equal(ur[p, :n], o["mvuRight"]) and np.array_equal(dp[p, :n], o["mvDepth"])
    # a buffer smaller than a pair's keypoint count is reported, as borb_stereo_frames does
    small = int(min(nl.min(), nr.min())) - 1
    with pytest.raises(_lib.BorbError) as ex:
        _lib.check(lib.borb_stereo_frames_results(G._h, 1, kl.ctypes.data, dl.ctypes.data, ml.ctypes.data, kr.ctypes.data,
                                                  dr.ctypes.data, mr.ctypes.data, ur.ctypes.data, dp.ctypes.data, small), "results")
    assert ex.value.status == 5                                                    # BORB_ERR_CAPACITY
    with pytest.raises(_lib.BorbError) as ex:                                      # more pairs than the stereo call associated
        _lib.check(lib.borb_stereo_frames_results(G._h, 3, None, None, None, None, None, None, None, None, cap), "results")
    assert ex.value.status == 6                                                    # BORB_ERR_STATE
    G(pairs[0][0])                                                                 # a mono extraction replaces the batch
    with pytest.raises(_lib.BorbError) as ex:
        _lib.check(lib.borb_stereo_frames_results(G._h, 1, None, None, None, None, None, None, ur.ctypes.data, dp.ctypes.data, cap),
                   "results")
    assert ex.value.status == 6


def test_explicit_pair_indices_and_no_match_cases(X, oracle):
    G = X(1000)
    L, R, _ = synth.stereo_pair(500, 0, 0, 640, 480)
    blank = np.full((480, 640), 90, np.uint8)
    G.extract_batch([R, L, blank, L])
    ur, dp = G.stereo_match(3, 40.0, 525.0, left_idx=[1, 3, 1], right_idx=[0, 2, 1])
    kl, dl, kr, dr, our, odp = oracle_stereo(oracle, L, R, 1000, 40.0, 525.0)
    assert np.array_equal(ur[0, :len(kl)], our) and np.array_equal(dp[0, :len(kl)], odp)
    assert np.all(ur[1, :len(kl)] == -1.0) and np.all(dp[1, :len(kl)] == -1.0)        # right image has no keypoints
    # left matched against itself: zero disparity -> clamped to 0.01 (Frame.cc:614-618) where SAD is unambiguous
    _, _, _, _, sur, sdp = oracle_stereo(oracle, L, L, 1000, 40.0, 525.0)
    assert np.array_equal(ur[2, :len(kl)], sur) and np.array_equal(dp[2, :len(kl)], sdp)


def test_stereo_before_extract_is_a_state_error(X):
    from orb_slam2_b200._lib import BorbError
    G = X(1000)
    with pytest.raises(BorbError) as ei:
        G._lib.borb_stereo_match   # noqa: B018  (binding exists)
        import numpy as _np
        ur = _np.zeros(8, _np.float32)
        from orb_slam2_b200 import _lib
        _lib.check(G._lib.borb_stereo_match(G._h, 1, None, None, 40.0, 0.1, _lib.ptr(ur), _lib.ptr(ur), 8), "borb_stereo_match")
    assert ei.value.status == 6


def test_constant_shift_property_full_size(X):
    """Right = left shifted by an integer disparity: every accepted match recovers it to sub-pixel accuracy."""
    L = synth.mono_frame(600, 0, 0, *synth.KITTI)
    d = 23
    R = np.empty_like(L); R[:, :-d] = L[:, d:]; R[:, -d:] = L[:, -1:]
    out = X(2000).stereo_frames([L] * 4, [R] * 4, BF, FX)
    for o in out:
        m = o["mvuRight"] >= 0
        assert m.sum() > 800
        disp = o["mvKeys"]["x"][m] - o["mvuRight"][m]
        # sub-pixel resolution is one level pixel, i.e. up to mvScaleFactor[7]=3.58 px at the coarsest octave
        scale = np.float32(1.2) ** o["mvKeys"]["octave"][m]
        assert np.all(np.abs(disp - d) < 0.75 * scale) and np.median(np.abs(disp - d)) < 0.3
        assert np.allclose(o["mvDepth"][m], np.float32(BF) / disp, rtol=1e-6)
    assert all(np.array_equal(out[0]["mvuRight"], o["mvuRight"]) for o in out[1:])


def test_rectification_fused_into_upload_equals_cv2_remap():
    """Examples/Stereo/stereo_euroc.cc:136-137 rectify every frame with cv::remap before TrackStereo; with the maps installed on
    the handle the RAW frames are uploaded and rectified on the GPU: level 0 must equal cv2.remap's output bit for bit, and
    keypoints / descriptors / stereo matches those of the pre-rectified path."""
    cv2 = pytest.importorskip("cv2")
    from orb_slam2_b200.extractor import ORBextractor
    w, h = synth.EUROC

    def maps(flip):
        K = np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1]])
        D = np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05]) * flip
        R = cv2.Rodrigues(np.array([0.003, -0.002, 0.001]) * flip)[0]
        P = np.array([[435.2, 0, 367.45], [0, 435.2, 252.2], [0, 0, 1]])
        return cv2.initUndistortRectifyMap(K, D, R, P, (w, h), cv2.CV_32F)
    M1l, M2l = maps(1.0)
    M1r, M2r = maps(0.9)
    pairs = [synth.stereo_pair(80 + i, 0, 0, w, h)[:2] for i in range(3)]
    rect = [(cv2.remap(L, M1l, M2l, cv2.INTER_LINEAR), cv2.remap(R, M1r, M2r, cv2.INTER_LINEAR)) for L, R in pairs]
    bf, fx = 47.9, 435.2
    ref = ORBextractor(1200).stereo_frames([p[0] for p in rect], [p[1] for p in rect], bf, fx)
    G = ORBextractor(1200)
    G.set_rectify_maps(0, M1l, M2l)
    G.set_rectify_maps(1, M1r, M2r)
    got = G.stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], bf, fx)
    for i in range(3):
        assert np.array_equal(G.pyramid(0, image=2 * i), rect[i][0]) and np.array_equal(G.pyramid(0, image=2 * i + 1), rect[i][1])
        for k in ("mvKeys", "mDescriptors", "mvKeysRight", "mDescriptorsRight", "mvuRight", "mvDepth"):
            assert np.array_equal(got[i][k], ref[i][k]), (i, k)
        assert (got[i]["mvuRight"] >= 0).sum() > 100
    # monocular call on the same handle: set 0 only
    km, dm = G(pairs[1][0])
    kr, dr = ORBextractor(1200)(rect[1][0])
    assert np.array_equal(km, kr) and np.array_equal(dm, dr)
    # a raw frame of the wrong size is an error, removing the maps restores the plain path
    from orb_slam2_b200._lib import BorbError
    with pytest.raises(BorbError):
        G(pairs[0][0][:400])
    G.set_rectify_maps(0, None, None)
    kp, dp = G(rect[1][0])
    assert np.array_equal(kp, kr) and np.array_equal(dp, dr)
