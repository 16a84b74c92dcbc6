"""GPU: the stereo association of the CUDA library (k_stereo.cu) equals the port bit for bit — keypoints, descriptors, mvuRight
and mvDepth — on every envelope case of tests/stereo_envelope.py, through every stereo entry point: borb_stereo_frames,
borb_stereo_match with permuted and repeated pair indices, borb_stereo_frames_device + borb_stereo_frames_results, and
borb_stereo_match2 on two handles whose nfeatures differ either way round."""
import numpy as np
import pytest

from orb_slam2_b200 import _lib
from orb_slam2_b200._lib import KP_DTYPE, BorbError
from tests import stereo_envelope as E

pytestmark = pytest.mark.gpu

ONE_HANDLE = [n for n in E.NAMES if E.CASES[n]["left"] == E.CASES[n]["right"]]
BORB_ERR_INVALID_ARG = 1


@pytest.fixture(scope="module")
def X():
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor


def _b(cam):
    bf, fx = cam
    return float(np.float32(bf) / np.float32(fx))


def assert_pair(name, p, kl, dl, kr, dr, ur, dp):
    assert np.array_equal(kl, p["kl"]) and np.array_equal(dl, p["dl"]), name
    assert np.array_equal(kr, p["kr"]) and np.array_equal(dr, p["dr"]), name
    n = len(p["kl"])
    bad = int((ur[:n] != p["ur"]).sum())
    assert bad == 0, f"{name}: mvuRight differs at {bad} of {n} left keypoints (rows {np.sort(p['kl']['y'][ur[:n] != p['ur']])[:8]})"
    assert np.array_equal(dp[:n], p["dp"]), name


@pytest.mark.parametrize("name", ONE_HANDLE)
def test_stereo_frames(X, oracle, name):
    c = E.CASES[name]
    p = E.run_port(oracle, name)
    L, R = E.images(name)
    o = X(*c["left"]).stereo_frames([L], [R], *c["cam"])[0]
    assert_pair(name, p, o["mvKeys"], o["mDescriptors"], o["mvKeysRight"], o["mDescriptorsRight"], o["mvuRight"], o["mvDepth"])


@pytest.mark.parametrize("name", ONE_HANDLE)
def test_stereo_match_permuted_and_repeated_pairs(X, oracle, name):
    """Images [R, L, L, R]: the same pair three times under different index tables; a second call of the same length with
    other indices replaces the cached pair table, a third goes back to the first one."""
    c = E.CASES[name]
    p = E.run_port(oracle, name)
    L, R = E.images(name)
    G = X(*c["left"])
    G.extract_batch([R, L, L, R])
    for li, ri in (([1, 2, 1], [0, 3, 3]), ([2, 1, 2], [3, 0, 0]), ([1, 2, 1], [0, 3, 3])):
        ur, dp = G.stereo_match(3, *c["cam"], left_idx=li, right_idx=ri)
        for q in range(3):
            assert_pair(name, p, p["kl"], p["dl"], p["kr"], p["dr"], ur[q], dp[q])


@pytest.mark.parametrize("name", ONE_HANDLE)
def test_device_resident_frames_and_results(X, oracle, name):
    import torch
    c = E.CASES[name]
    p = E.run_port(oracle, name)
    L, R = E.images(name)
    w, h = c["w"], c["h"]
    G = X(*c["left"])
    lib = G._lib
    cap = G.capacity(w, h)
    d_img = torch.from_numpy(np.stack([L, R])).cuda()
    nl, nr = np.zeros(1, np.int32), np.zeros(1, np.int32)
    _lib.check(lib.borb_stereo_frames_device(G._h, d_img.data_ptr(), 1, w, h, w, w * h, float(c["cam"][0]), _b(c["cam"]),
                                             _lib.ptr(nl), _lib.ptr(nr), None, None, cap), "borb_stereo_frames_device")
    kl, kr = np.zeros(cap, KP_DTYPE), np.zeros(cap, KP_DTYPE)
    dl, dr = np.zeros((cap, 32), np.uint8), np.zeros((cap, 32), np.uint8)
    ml, mr = np.zeros(1, np.int32), np.zeros(1, np.int32)
    ur, dp = np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    _lib.check(lib.borb_stereo_frames_results(G._h, 1, kl.ctypes.data, dl.ctypes.data, ml.ctypes.data, kr.ctypes.data,
                                              dr.ctypes.data, mr.ctypes.data, ur.ctypes.data, dp.ctypes.data, cap),
               "borb_stereo_frames_results")
    assert ml[0] == nl[0] == len(p["kl"]) and mr[0] == nr[0] == len(p["kr"])
    assert_pair(name, p, kl[:ml[0]], dl[:ml[0]], kr[:mr[0]], dr[:mr[0]], ur, dp)


def _match2(GL, GR, cam, cap):
    ur, dp = np.zeros(cap, np.float32), np.zeros(cap, np.float32)
    _lib.check(_lib.load().borb_stereo_match2(GL._h, GR._h, float(cam[0]), _b(cam), _lib.ptr(ur), _lib.ptr(dp), cap),
               "borb_stereo_match2")
    return ur, dp


@pytest.mark.parametrize("name", E.NAMES)
def test_two_handles(X, oracle, name):
    """mpORBextractorLeft / mpORBextractorRight (Frame.cc:78-81) as two handles; in the kitti_L* cases their nfeatures differ,
    so the right keypoints' bin records need a buffer sized by the right handle."""
    c = E.CASES[name]
    p = E.run_port(oracle, name)
    L, R = E.images(name)
    GL, GR = X(*c["left"]), X(*c["right"])
    kl, dl = GL(L)
    kr, dr = GR(R)
    ur, dp = _match2(GL, GR, c["cam"], GL.capacity(c["w"], c["h"]))
    assert_pair(name, p, kl, dl, kr, dr, ur, dp)


def test_two_handles_with_differing_scale_factors_are_refused(X):
    L, R = E.images("kitti_1.2x8")
    for right in ((2000, 1.25, 8), (2000, 1.2, 7)):
        GL, GR = X(2000, 1.2, 8), X(*right)
        GL(L)
        GR(R)
        with pytest.raises(BorbError) as ex:
            _match2(GL, GR, E.KITTI_CAM, GL.capacity(E.KW, E.KH))
        assert ex.value.status == BORB_ERR_INVALID_ARG


def test_batch_of_envelope_blank_and_identical_pairs(X, oracle):
    """One batch at KITTI size: natural, shifted and maxD-edge pairs next to a blank pair (no keypoints at all) and L = R pairs."""
    names = ["kitti_1.2x8", "shift_23", "periodic_48"]
    L0, _ = E.images("shift_23")
    blank = np.full((E.KH, E.KW), 90, np.uint8)
    lefts = [E.images(n)[0] for n in names] + [blank, L0, blank]
    rights = [E.images(n)[1] for n in names] + [blank, L0, L0]
    out = X(2000).stereo_frames(lefts, rights, *E.KITTI_CAM)
    for i, n in enumerate(names):
        o = out[i]
        assert_pair(n, E.run_port(oracle, n), o["mvKeys"], o["mDescriptors"], o["mvKeysRight"], o["mDescriptorsRight"],
                    o["mvuRight"], o["mvDepth"])
    assert len(out[3]["mvKeys"]) == len(out[3]["mvKeysRight"]) == 0 and len(out[5]["mvKeys"]) == 0
    EL = oracle.PortExtractor(2000)
    kl, dl = EL(L0)
    pyr = [EL.level(i) for i in range(8)]
    ur, dp, _ = oracle.port_stereo(kl, dl, kl, dl, pyr, pyr, EL.scale, EL.inv_scale, *E.KITTI_CAM)
    o = out[4]
    assert_pair("L=R", dict(kl=kl, dl=dl, kr=kl, dr=dl, ur=ur, dp=dp), o["mvKeys"], o["mDescriptors"], o["mvKeysRight"],
                o["mDescriptorsRight"], o["mvuRight"], o["mvDepth"])


@pytest.mark.parametrize("name", ["kitti_1.2x8", "vga_1.2x12", "kitti_11200", "tall_2120x4095"])
def test_handle_reused_after_another_size_equals_the_port(X, oracle, name):
    """A handle that first associated a batch of another size (its workspace is then rebuilt) gives what a fresh one gives."""
    from orb_slam2_b200 import synth
    c = E.CASES[name]
    p = E.run_port(oracle, name)
    G = X(*c["left"])
    oL, oR, _ = synth.stereo_pair(730, 0, 0, 720, 540)
    G.stereo_frames([oL, oL, oL], [oR, oR, oR], *c["cam"])
    L, R = E.images(name)
    o = G.stereo_frames([L], [R], *c["cam"])[0]
    assert_pair(name, p, o["mvKeys"], o["mDescriptors"], o["mvKeysRight"], o["mDescriptorsRight"], o["mvuRight"], o["mvDepth"])
