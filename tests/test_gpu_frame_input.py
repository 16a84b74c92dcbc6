"""GPU sweep of the frame input path: the uploads that turn a camera frame into level 0 (repack / remap kernels of k_pyramid.cu,
host and device entry points of borb_host.cu), the pipelined enqueue calls, and the Frame constructor tail of k_frame.cu
(UndistortKeyPoints, ComputeStereoFromRGBD, AssignFeaturesToGrid) read back field by field, grid included.  Everything is
compared bit for bit with the CPU restatements under oracle/ (pinned to cv2 and to the verbatim Frame.cc by
tests/test_oracle_prims.py and tests/test_oracle_frame_ref.py) or with the host-buffer path of the same library."""
import ctypes as C
import dataclasses
import threading

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import frame_input_cases as fic
from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu

BF, FX = 40.0, 525.0


@pytest.fixture(scope="module")
def L():
    from orb_slam2_b200 import _lib
    return _lib


def _X(nf=1000):
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor(nf)


def _raw(seed, w, h):
    return synth.mono_frame(seed, 0, 0, w, h)


def _extract_slots(L, G, images, contiguous):
    """borb_extract_batch with the images in one block (one H2D copy) or in scattered buffers (one 2-D copy each)."""
    n = len(images)
    h, w = images[0].shape
    if contiguous:
        block = np.ascontiguousarray(np.stack(images))
        slots = [block[i] for i in range(n)]
    else:
        slots = [np.pad(im, ((0, 0), (0, 9)), constant_values=77)[:, :w] for im in images]      # own buffers, rows w + 9 apart
        assert all(s.strides[0] == w + 9 for s in slots)
    stride = slots[0].strides[0]
    cap = G._work_capacity(w, h)
    kps, desc, cnt = np.zeros((n, cap), L.KP_DTYPE), np.zeros((n, cap, 32), np.uint8), np.zeros(n, np.int32)
    ptrs = (C.c_void_p * n)(*[s.ctypes.data for s in slots])
    L.check(L.load().borb_extract_batch(G._h, ptrs, n, w, h, stride, L.ptr(kps), L.ptr(desc), cap, L.ptr(cnt)), "borb_extract_batch")
    G._last_n = n
    return [(kps[i, :cnt[i]].copy(), desc[i, :cnt[i]].copy()) for i in range(n)]


def _device_block(images, pitch, image_stride):
    """The images in one device buffer: rows `pitch` bytes apart, images `image_stride` apart, every other byte 0xA5."""
    import torch
    n = len(images)
    h, w = images[0].shape
    buf = np.full(n * image_stride + pitch, 0xA5, np.uint8)
    for i, im in enumerate(images):
        for y in range(h):
            o = i * image_stride + y * pitch
            buf[o:o + w] = im[y]
    return torch.from_numpy(buf).cuda()


def _extract_device(L, G, d, n, w, h, pitch, image_stride):
    cap = G._work_capacity(w, h)
    kps, desc, cnt = np.zeros((n, cap), L.KP_DTYPE), np.zeros((n, cap, 32), np.uint8), np.zeros(n, np.int32)
    L.check(L.load().borb_extract_batch_device(G._h, d.data_ptr(), n, w, h, pitch, image_stride, L.ptr(kps), L.ptr(desc), cap, L.ptr(cnt)),
            "borb_extract_batch_device")
    G._last_n = n
    return [(kps[i, :cnt[i]].copy(), desc[i, :cnt[i]].copy()) for i in range(n)]


def _same_extraction(a, b):
    return len(a) == len(b) and all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))


def _maps(src, dst, seed):
    """The adversarial maps of the CPU pin plus a smooth rectification map with a special value in every 11th entry."""
    mx, my = fic.radial_rectify_maps(src, dst)
    sp = fic.SPECIAL_MAP_VALUES
    mx.reshape(-1)[5::11] = sp[np.arange(len(mx.reshape(-1)[5::11])) % len(sp)]
    my.reshape(-1)[::13] = sp[(3 * np.arange(len(my.reshape(-1)[::13]))) % len(sp)]
    return [(mx, my)] + fic.adversarial_remap_maps(src, dst, seed)


# ------------------------------------------------------------------------------------------------------ 1. rectified upload
@pytest.mark.parametrize("src,dst", [((752, 480), (752, 480)), ((347, 263), (301, 229)), ((250, 190), (389, 271))])
def test_rectified_upload_equals_port_remap(L, oracle, src, dst):
    """Level 0 of a rectifying upload equals the port's cv::remap for every map (NaN, +-inf, out-of-int-range values, ties, edge
    taps), through one contiguous H2D copy and through scattered per-image copies; the keypoints equal those of the
    pre-rectified frames on a handle without maps."""
    sw, sh = src
    raws = [_raw(70 + i, sw, sh) for i in range(3)]
    G, P = _X(), _X()
    for k, (mx, my) in enumerate(_maps(src, dst, sum(src))):
        want = [oracle.port_remap(r, mx, my) for r in raws]
        G.set_rectify_maps(0, mx, my, src_size=src)
        plain = P.extract_batch(want)
        for contiguous in (True, False):
            got = _extract_slots(L, G, raws, contiguous)
            for i in range(3):
                assert np.array_equal(G.pyramid(0, image=i), want[i]), (k, contiguous, i)
            assert _same_extraction(got, plain), (k, contiguous)
        if k == 0:                                                        # the smooth map: a natural frame for the port extractor
            kp, dp = oracle.PortExtractor(1000)(want[1])
            assert len(kp) > 100 and np.array_equal(plain[1][0], kp) and np.array_equal(plain[1][1], dp)


def test_rectified_stereo_one_and_two_map_sets_mono_call_and_removal(L, oracle):
    """Stereo with two sets (even images set 0, odd images set 1), with one set (both images set 0), a mono call on a handle with
    set 1 installed (set 0 only), and the removal of the sets (plain upload again)."""
    src, dst = (400, 300), (373, 281)
    m0 = fic.radial_rectify_maps(src, dst)
    m1 = fic.radial_rectify_maps(src, dst, k1=-0.2, k2=0.03, shift=(4.5, -2.25))
    m1[0].reshape(-1)[::17] = np.nan                                      # NaN entries in the right set only
    pairs = [synth.stereo_pair(90 + i, 0, 0, *src)[:2] for i in range(3)]
    G, P = _X(), _X()
    G.set_rectify_maps(0, *m0, src_size=src)
    G.set_rectify_maps(1, *m1, src_size=src)
    for sets in (2, 1):
        mr = m1 if sets == 2 else m0
        got = G.stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], BF, FX)
        rect = [(oracle.port_remap(l, *m0), oracle.port_remap(r, *mr)) for l, r in pairs]
        want = P.stereo_frames([r[0] for r in rect], [r[1] for r in rect], BF, FX)
        for i in range(3):
            assert np.array_equal(G.pyramid(0, image=2 * i), rect[i][0]) and np.array_equal(G.pyramid(0, image=2 * i + 1), rect[i][1]), (sets, i)
            for key in want[i]:
                assert np.array_equal(got[i][key], want[i][key]), (sets, i, key)
        if sets == 2:
            km, dm = G(pairs[0][1])                                        # mono call: set 0 even with set 1 installed
            assert np.array_equal(G.pyramid(0), oracle.port_remap(pairs[0][1], *m0))
            kr, dr = P(oracle.port_remap(pairs[0][1], *m0))
            assert np.array_equal(km, kr) and np.array_equal(dm, dr)
            G.set_rectify_maps(1, None, None)                              # set 0 stays
    G.set_rectify_maps(0, None, None)
    km, dm = G(rect[0][0])
    assert np.array_equal(G.pyramid(0), rect[0][0])
    kr, dr = P(rect[0][0])
    assert np.array_equal(km, kr) and np.array_equal(dm, dr)


# ------------------------------------------------------------------------------------------------------ 2. device input
@pytest.mark.parametrize("n", [1, 3, 8])
@pytest.mark.parametrize("layout", ["stride_multiple_of_pitch", "stride_not_multiple"])
def test_extract_batch_device_equals_host_path(L, n, layout):
    """borb_extract_batch_device with pitch > width: a multiple image stride moves the batch as one 3-D copy, any other stride
    as one 2-D copy per image; either way level 0 and the keypoints equal the host path's."""
    w, h = 640, 480
    pitch = 704
    image_stride = pitch * (h + 3) if layout == "stride_multiple_of_pitch" else pitch * h + 37
    imgs = [_raw(10 + i, w, h) for i in range(n)]
    d = _device_block(imgs, pitch, image_stride)
    G = _X()
    got = _extract_device(L, G, d, n, w, h, pitch, image_stride)
    for i in range(n):
        assert np.array_equal(G.pyramid(0, image=i), imgs[i])
    assert _same_extraction(got, _X().extract_batch(imgs))


@pytest.mark.parametrize("layout", ["stride_multiple_of_pitch", "stride_not_multiple"])
def test_device_input_is_rectified_and_ignores_the_colour_format(L, oracle, layout):
    """With maps installed the device entry points take RAW frames and rectify them (set 1 on the odd images of the stereo call);
    a colour input format set on the handle does not apply to device images (always CV_8UC1)."""
    import torch
    src, dst = (400, 300), (373, 281)
    m0 = fic.radial_rectify_maps(src, dst)
    m1 = fic.radial_rectify_maps(src, dst, k1=-0.2, k2=0.03, shift=(4.5, -2.25))
    m0[1].reshape(-1)[::19] = np.nan
    pitch = 448
    image_stride = pitch * (src[1] + 1) if layout == "stride_multiple_of_pitch" else pitch * src[1] + 5
    pairs = [synth.stereo_pair(95 + i, 0, 0, *src)[:2] for i in range(4)]
    flat = [im for p in pairs for im in p]
    d = _device_block(flat, pitch, image_stride)
    G, H = _X(), _X()
    G.set_input_format(3)
    for X in (G, H):
        X.set_rectify_maps(0, *m0, src_size=src)
        X.set_rectify_maps(1, *m1, src_size=src)
    # mono: set 0 on every image
    got = _extract_device(L, G, d, 4, src[0], src[1], pitch, image_stride)
    for i in range(4):
        assert np.array_equal(G.pyramid(0, image=i), oracle.port_remap(flat[i], *m0)), i
    assert _same_extraction(got, H.extract_batch(flat[:4]))
    # stereo: set 0 left, set 1 right; results read back with borb_stereo_frames_results
    cap = G._work_capacity(*src)
    nl, nr = np.zeros(4, np.int32), np.zeros(4, np.int32)
    ur, dp = np.zeros((4, cap), np.float32), np.zeros((4, cap), np.float32)
    b = float(np.float32(BF) / np.float32(FX))
    lib = L.load()
    L.check(lib.borb_stereo_frames_device(G._h, d.data_ptr(), 4, src[0], src[1], pitch, image_stride, BF, b, L.ptr(nl), L.ptr(nr), L.ptr(ur),
                                          L.ptr(dp), cap), "borb_stereo_frames_device")
    torch.cuda.synchronize()
    want = H.stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], BF, FX)
    for i in range(4):
        assert np.array_equal(G.pyramid(0, image=2 * i), oracle.port_remap(pairs[i][0], *m0))
        assert np.array_equal(G.pyramid(0, image=2 * i + 1), oracle.port_remap(pairs[i][1], *m1))
        assert nl[i] == len(want[i]["mvKeys"]) and nr[i] == len(want[i]["mvKeysRight"])
        assert np.array_equal(ur[i, :nl[i]], want[i]["mvuRight"]) and np.array_equal(dp[i, :nl[i]], want[i]["mvDepth"])


# ------------------------------------------------------------------------------------------------------ 3. pipelined handles
def _pinned(L, shape, dtype):
    p = C.c_void_p()
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    L.check(L.load().borb_host_alloc(C.byref(p), n), "borb_host_alloc")
    arr = np.ctypeslib.as_array((C.c_uint8 * n).from_address(p.value)).view(dtype).reshape(shape)
    return p, arr


def test_pipelined_enqueues_on_several_handles_equal_synchronous_calls(L):
    """Several handles, each with several stereo enqueues in flight before borb_sync, as the benchmark drives them: host-buffer
    enqueues land in their own pinned buffers, device enqueues in their own count / association buffers, and
    borb_stereo_frames_results returns the last batch of each handle.  Every batch equals one synchronous call."""
    w, h, n_pairs, depth_q, n_handles = 640, 480, 2, 3, 3
    lib = L.load()
    b = float(np.float32(BF) / np.float32(FX))
    batches = [[synth.stereo_pair(200 + 10 * hd + q * 3 + p, 0, 0, w, h)[:2] for p in range(n_pairs)] for hd in range(n_handles) for q in range(depth_q)]
    R = _X()
    want = [R.stereo_frames([p[0] for p in bt], [p[1] for p in bt], BF, FX) for bt in batches]
    Gs = [_X() for _ in range(n_handles)]
    cap = Gs[0].capacity(w, h)
    pinned, keep, outs = [], [], []
    for hd, G in enumerate(Gs):
        for q in range(depth_q):
            bt = batches[hd * depth_q + q]
            p_img, imgs = _pinned(L, (2 * n_pairs, h, w), np.uint8)
            p_out, out = _pinned(L, (n_pairs * cap * (28 * 2 + 64 + 8) + 8 * n_pairs,), np.uint8)
            pinned += [p_img, p_out]
            for p in range(n_pairs):
                imgs[2 * p], imgs[2 * p + 1] = bt[p]
            o = np.cumsum([0, n_pairs * cap * 28, n_pairs * cap * 28, n_pairs * cap * 32, n_pairs * cap * 32, n_pairs * cap * 4,
                           n_pairs * cap * 4, 8 * n_pairs])
            v = dict(kl=out[o[0]:o[1]].view(L.KP_DTYPE).reshape(n_pairs, cap), kr=out[o[1]:o[2]].view(L.KP_DTYPE).reshape(n_pairs, cap),
                     dl=out[o[2]:o[3]].reshape(n_pairs, cap, 32), dr=out[o[3]:o[4]].reshape(n_pairs, cap, 32),
                     ur=out[o[4]:o[5]].view(np.float32).reshape(n_pairs, cap), dp=out[o[5]:o[6]].view(np.float32).reshape(n_pairs, cap),
                     nl=out[o[6]:o[7]].view(np.int32)[:n_pairs], nr=out[o[6]:o[7]].view(np.int32)[n_pairs:])
            pl = (C.c_void_p * n_pairs)(*[imgs[2 * p].ctypes.data for p in range(n_pairs)])
            pr = (C.c_void_p * n_pairs)(*[imgs[2 * p + 1].ctypes.data for p in range(n_pairs)])
            keep.append((pl, pr, imgs))
            L.check(lib.borb_stereo_frames_enqueue(G._h, pl, pr, n_pairs, w, h, w, BF, b, L.ptr(v["kl"]), L.ptr(v["dl"]), L.ptr(v["nl"]),
                                                   L.ptr(v["kr"]), L.ptr(v["dr"]), L.ptr(v["nr"]), L.ptr(v["ur"]), L.ptr(v["dp"]), cap),
                    "borb_stereo_frames_enqueue")
            outs.append(v)
    for G in Gs:
        L.check(lib.borb_sync(G._h), "borb_sync")
    for j, v in enumerate(outs):
        for p in range(n_pairs):
            nl, nr, o = v["nl"][p], v["nr"][p], want[j][p]
            assert np.array_equal(v["kl"][p, :nl], o["mvKeys"]) and np.array_equal(v["dl"][p, :nl], o["mDescriptors"]), (j, p)
            assert np.array_equal(v["kr"][p, :nr], o["mvKeysRight"]) and np.array_equal(v["dr"][p, :nr], o["mDescriptorsRight"]), (j, p)
            assert np.array_equal(v["ur"][p, :nl], o["mvuRight"]) and np.array_equal(v["dp"][p, :nl], o["mvDepth"]), (j, p)
    # device enqueues: several in flight per handle, then the resident results of each handle's last batch
    dev = [_device_block([im for p in bt for im in p], w, w * h) for bt in batches]
    douts = []
    for hd, G in enumerate(Gs):
        for q in range(depth_q):
            v = dict(nl=np.zeros(n_pairs, np.int32), nr=np.zeros(n_pairs, np.int32), ur=np.zeros((n_pairs, cap), np.float32),
                     dp=np.zeros((n_pairs, cap), np.float32))
            L.check(lib.borb_stereo_frames_device_enqueue(G._h, dev[hd * depth_q + q].data_ptr(), n_pairs, w, h, w, w * h, BF, b, L.ptr(v["nl"]),
                                                          L.ptr(v["nr"]), L.ptr(v["ur"]), L.ptr(v["dp"]), cap), "borb_stereo_frames_device_enqueue")
            douts.append(v)
    for G in Gs:
        L.check(lib.borb_sync(G._h), "borb_sync")
    for j, v in enumerate(douts):
        for p in range(n_pairs):
            o = want[j][p]
            assert v["nl"][p] == len(o["mvKeys"]) and v["nr"][p] == len(o["mvKeysRight"]), (j, p)
            assert np.array_equal(v["ur"][p, :v["nl"][p]], o["mvuRight"]) and np.array_equal(v["dp"][p, :v["nl"][p]], o["mvDepth"]), (j, p)
    for hd, G in enumerate(Gs):
        kl, kr = np.zeros((n_pairs, cap), L.KP_DTYPE), np.zeros((n_pairs, cap), L.KP_DTYPE)
        dl, dr = np.zeros((n_pairs, cap, 32), np.uint8), np.zeros((n_pairs, cap, 32), np.uint8)
        nl, nr = np.zeros(n_pairs, np.int32), np.zeros(n_pairs, np.int32)
        L.check(lib.borb_stereo_frames_results(G._h, n_pairs, L.ptr(kl), L.ptr(dl), L.ptr(nl), L.ptr(kr), L.ptr(dr), L.ptr(nr), None, None, cap),
                "borb_stereo_frames_results")
        for p in range(n_pairs):
            o = want[hd * depth_q + depth_q - 1][p]
            assert np.array_equal(kl[p, :nl[p]], o["mvKeys"]) and np.array_equal(dr[p, :nr[p]], o["mDescriptorsRight"]), (hd, p)
            assert np.array_equal(kr[p, :nr[p]], o["mvKeysRight"]) and np.array_equal(dl[p, :nl[p]], o["mDescriptors"]), (hd, p)
    for p in pinned:
        L.check(lib.borb_host_free(p), "borb_host_free")


# ------------------------------------------------------------------------------------------------------ 4. frame tail envelope
ENVELOPE_N = [0, 1, 31, 32, 33, 1023, 1024, 1025, 2048, 4097, 8192]


@pytest.fixture(scope="module")
def kitti_8192():
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(8192)
    img = synth.stereo_pair(9, 0, 0, *synth.KITTI)[0]
    keys, desc = X.extract_batch([img])[0]
    assert len(keys) >= 8192
    return X, keys, desc


@pytest.mark.parametrize("case", ["tum1_5", "tum1_4", "pincushion", "icdist_negative", "k1_neg_zero", "k1_zero_rest_nonzero"])
def test_frame_tail_envelope_in_one_batch(oracle, kitti_8192, case):
    """borb_frames_from_extractor on subsets of one 8192+-keypoint extraction, all in ONE batch with mixed sizes (the per-job
    sort size against the batch's shared-memory size; 32 / 1024 / 8192 keys fill the sort to its last slot): mvKeysUn,
    mvuRight, mvDepth (edge depths) and the bounds equal the port, and the feature grid read back from the device equals the
    port's build_grid cell by cell."""
    from orb_slam2_b200 import matcher as M
    X, keys, desc = kitti_8192
    w, h = synth.KITTI
    K, dist = fic.DIST_CASES[case]
    depth = fic.edge_depth_float(21, w, h)
    mt = M.ORBmatcher(0.8, True)
    frames, host = M.frames_from_extractor(mt, X, [0] * len(ENVELOPE_N), ENVELOPE_N, K, dist, bf=BF, mode=2, depth=[depth] * len(ENVELOPE_N))
    outside = 0
    for j, n in enumerate(ENVELOPE_N):
        p = oracle.port_rgbd_frame(keys[:n], np.array(K, np.float32), np.array(dist, np.float32), BF, depth)
        assert np.array_equal(host["bounds"], p["bounds"])
        got = frames[j].resident.read()
        for f in ("keys_un", "u_right", "depth"):
            assert host[f][j].tobytes() == p[f].tobytes(), (n, f)
            assert got[f].tobytes() == p[f].tobytes(), (n, f)
        assert np.array_equal(got["desc"], desc[:n])
        cs, ci = oracle.port_assign_grid(p["keys_un"], p["bounds"])
        assert np.array_equal(got["cell_start"], cs) and np.array_equal(got["cell_idx"], ci), n
        outside += n - int(cs[-1])
        frames[j].resident.close()
    if case in ("pincushion", "icdist_negative"):
        assert outside > 0                                                 # undistorted keys that miss the grid


# ------------------------------------------------------------------------------------------------------ 5. RGB-D depth
@pytest.mark.parametrize("factor", fic.DEPTH_FACTORS)
def test_rgbd_depth_host_padded_device_and_mixed(oracle, factor):
    """Host uint16 / float32 maps with a padded row stride, device maps (+4) with the host copies off (read back from the resident
    frames), and a mixed batch of both kinds of frames from one extraction: every frame equals the port on the edge depths."""
    import torch
    from orb_slam2_b200 import matcher as M
    w, h = 640, 480
    K, dist = fic.DIST_CASES["tum1_5"]
    X = _X(1500)
    outs = X.extract_batch([_raw(30 + i, w, h) for i in range(3)])
    raws = [fic.edge_depth_raw(40 + i) for i in range(3)]
    floats = [fic.edge_depth_float(50 + i) for i in range(3)]
    mt = M.ORBmatcher(0.8, True)
    nk = [len(o[0]) for o in outs]
    K4, D = np.array(K, np.float32), np.array(dist, np.float32)

    def check(frames, host, metres, sel):
        for j, i in enumerate(sel):
            p = oracle.port_rgbd_frame(outs[i][0], K4, D, BF, metres[j])
            got = frames[j].resident.read()
            for f in ("keys_un", "u_right", "depth"):
                assert got[f].tobytes() == p[f].tobytes(), (i, f)
                if host is not None:
                    assert host[f][j].tobytes() == p[f].tobytes(), (i, f)
            assert fic.keys_on_depth_specials(outs[i][0], metres[j]) > 20
            frames[j].resident.close()

    sel = [2, 0, 1]
    for raw16 in (True, False):
        maps = [raws[i] if raw16 else floats[i] for i in sel]
        metres = [oracle.port_depth_to_float(m, factor) if raw16 else m for m in maps]
        padded = [np.pad(m, ((0, 0), (0, 24)), constant_values=7)[:, :w] for m in maps]        # depth_stride_bytes > row
        assert padded[0].strides[0] == (w + 24) * padded[0].itemsize
        frames, host = M.frames_from_extractor(mt, X, sel, [nk[i] for i in sel], K, dist, bf=BF, mode=2, depth=padded,
                                               depth_factor=factor if raw16 else 1.0)
        check(frames, host, metres, sel)
        dev = [torch.from_numpy(m.view(np.int16) if raw16 else m).cuda() for m in maps]
        frames, _ = M.frames_from_extractor(mt, X, sel, [nk[i] for i in sel], K, dist, bf=BF, mode=2, depth=dev,
                                            depth_factor=factor if raw16 else 1.0, want_host=False, depth_on_device=True)
        check(frames, None, metres, sel)
    # a mixed batch: the same image as several frames with different depth maps, next to an empty frame
    maps = [raws[0], raws[1], raws[2]]
    metres = [oracle.port_depth_to_float(m, factor) for m in maps]
    frames, host = M.frames_from_extractor(mt, X, [1, 1, 1], [nk[1]] * 3, K, dist, bf=BF, mode=2, depth=maps, depth_factor=factor)
    check(frames, host, metres, [1, 1, 1])
    frames, host = M.frames_from_extractor(mt, X, [0, 2], [0, nk[2]], K, dist, bf=BF, mode=2, depth=[raws[0], raws[2]], depth_factor=factor)
    assert frames[0].resident.read()["cell_start"].max() == 0
    check(frames[1:], dict((k, v[1:]) for k, v in host.items() if k != "bounds"), [metres[2]], [2])
    frames[0].resident.close()


# ------------------------------------------------------------------------------------------------------ 6. config-2 pass, threads
def _projection_jobs(oracle, X, outs, depths, factor, K, dist, seed):
    """The host path: per frame the port's RGB-D frame, map points projected into it, and the port's SearchByProjection."""
    from orb_slam2_b200 import matcher as M
    jobs = []
    for i, (keys, desc) in enumerate(outs):
        p = oracle.port_rgbd_frame(keys, np.array(K, np.float32), np.array(dist, np.float32), BF, oracle.port_depth_to_float(depths[i], factor))
        v = dict(w=640, h=480, kl=p["keys_un"], dl=desc, kr=p["keys_un"], dr=desc, ur=p["u_right"], disp=np.zeros((480, 640), np.float32),
                 scale=X.GetScaleFactors(), sigma2=X.GetScaleSigmaSquares())
        F, mps = mf.projection_case(v, seed + i, n_mp=300)
        F = M.FrameView(p["keys_un"], desc, X.GetScaleFactors(), tuple(float(x) for x in p["bounds"]), mvuRight=p["u_right"], occupied=F.occupied)
        jobs.append((F, mps, oracle.port_search_by_projection(F, mps, 3.0, 0.8)))
    return jobs


def test_config2_pass_under_threads_equals_host_path_and_port(L, oracle):
    """Several host threads, each with its own extractor and matcher, repeat the resident RGB-D pass: device images through
    borb_extract_batch_device, borb_frames_from_extractor with device depth maps (+4, no host copies), SearchByProjectionBatch.
    Every thread's matches equal the single-threaded host path and the port."""
    import torch
    from orb_slam2_b200 import matcher as M
    w, h, B, reps, n_threads = 640, 480, 4, 3, 4
    K, dist = fic.DIST_CASES["tum1_5"]
    factor = 1.0 / 5000.0
    imgs = [_raw(60 + i, w, h) for i in range(B)]
    raws = [fic.edge_depth_raw(80 + i) for i in range(B)]
    X = _X()
    outs = X.extract_batch(imgs)
    jobs = _projection_jobs(oracle, X, outs, raws, factor, K, dist, 3)
    mt = M.ORBmatcher(0.8, True)
    frames, _ = M.frames_from_extractor(mt, X, list(range(B)), [len(o[0]) for o in outs], K, dist, bf=BF, mode=2, depth=raws, depth_factor=factor)
    host = mt.SearchByProjectionBatch([dataclasses.replace(f, occupied=j[0].occupied) for f, j in zip(frames, jobs)], [j[1] for j in jobs], 3.0)
    for (n_g, m_g), (_, _, (n_o, m_o)) in zip(host, jobs):
        assert n_g == n_o > 30 and np.array_equal(m_g, m_o)
    d_img = _device_block(imgs, w, w * h)
    d_depth = [torch.from_numpy(r.view(np.int16)).cuda() for r in raws]
    torch.cuda.synchronize()
    errors = []

    def worker(t):
        try:
            Xt, mtt = _X(), M.ORBmatcher(0.8, True)
            for r in range(reps):
                o = _extract_device(L, Xt, d_img, B, w, h, w, w * h)
                assert _same_extraction(o, outs), (t, r)
                fr, _ = M.frames_from_extractor(mtt, Xt, list(range(B)), [len(k) for k, _ in o], K, dist, bf=BF, mode=2, depth=d_depth,
                                                depth_factor=factor, want_host=False, depth_on_device=True)
                got = mtt.SearchByProjectionBatch([dataclasses.replace(f, occupied=j[0].occupied) for f, j in zip(fr, jobs)], [j[1] for j in jobs], 3.0)
                for b, ((n_g, m_g), (n_h, m_h)) in enumerate(zip(got, host)):
                    assert n_g == n_h and np.array_equal(m_g, m_h), (t, r, b)
                for f in fr:
                    f.resident.close()
        except Exception as ex:                                            # reported on the main thread
            errors.append(repr(ex))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
