"""GPU: borb_frame_from_extractors against the reference's own Frame constructors (src/Frame.cc:61-228, run unmodified by
oracle.ref_frame on what the verbatim ORBextractor.cc finds on the same images).  Every host member — mvKeys, mDescriptors,
mvKeysRight, mDescriptorsRight, mvKeysUn, mvuRight, mvDepth, the grid and the bounds — and what the resident frame holds
(borb_debug_frame_read: keys, mvuRight, mvDepth, grid; the scale tables and level count) are bit-equal to the constructor's,
floats compared as uint32 so that NaN payloads and -0 count.  Stereo frames with distortion, odd and smallest image sizes, level
and scale variants, a handle at BORB_MATCH_MAX_FEATURES, blank images, RGB-D edge depths, sequences that keep the reference's
statics, and four streams on four threads.  The bounds are the reference's statics (:96-112): they are compared once the
reference has computed them for the frame's camera, i.e. not for a first frame without keypoints."""
import ctypes as C
import threading

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import frame_input_cases as fic

pytestmark = pytest.mark.gpu

KITTI_K = (718.856, 718.856, 607.1928, 185.2157)
KITTI_BF = 386.1448
EUROC_K = (435.2047, 435.2047, 367.4517, 252.2005)
EUROC_BF = 47.90639384423901
MODE = {"mono": 0, "stereo": 1, "rgbd": 2}


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_framector() and oracle.have_ref()):
        pytest.skip("oracle/_ref/libframector.so / liborbref.so not built")
    return oracle


def _M():
    from orb_slam2_b200 import matcher as M
    return M


def _X(n, sf=1.2, nl=8):
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor(n, sf, nl)


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Stream:
    """One camera: a matcher and the frame's own extractor handles, reused frame after frame."""

    def __init__(self, kind, nf=(2000, 2000), sf=1.2, nl=8):
        M = _M()
        self.kind, self.nf, self.sf, self.nl = kind, tuple(nf), sf, nl
        self.mt = M.ORBmatcher(0.8, True)
        self.XL = _X(nf[0], sf, nl)
        self.XR = _X(nf[1], sf, nl) if kind == "stereo" else None

    def frame(self, left, right=None, K=EUROC_K, dist=(0, 0, 0, 0), bf=EUROC_BF, depth=None, factor=1.0):
        self.XL.extract_enqueue(left)
        if self.XR is not None:
            self.XR.extract_enqueue(right)
        return _M().frame_from_extractors(self.mt, self.XL, self.XR, K, dist, bf=bf, mode=MODE[self.kind], depth=depth,
                                          depth_factor=factor)


def check(O, S, F, host, ref, bounds=True):
    """Every member the constructor fills equals the verbatim constructor's, on the host and on the device."""
    assert host["mvKeys"].shape == ref["mvKeys"].shape and _bits(host["mvKeys"]) == _bits(ref["mvKeys"])
    assert _bits(host["mDescriptors"]) == _bits(ref["mDescriptors"])
    assert _bits(host["mvKeysRight"]) == _bits(ref["mvKeysRight"]) and _bits(host["mDescriptorsRight"]) == _bits(ref["mDescriptorsRight"])
    N = ref["N"]
    assert len(host["mvKeys"]) == N
    if N == 0:                                    # the reference returned before UndistortKeyPoints (Frame.cc:85/140/195)
        assert len(ref["mvKeysUn"]) == len(ref["mvuRight"]) == len(ref["mvDepth"]) == 0
    assert _bits(host["mvKeysUn"]) == _bits(ref["mvKeysUn"])
    if S.kind == "mono" and N > 0:
        assert np.all(ref["mvuRight"] == -1) and np.all(ref["mvDepth"] == -1)
    assert np.array_equal(_u32(host["mvuRight"]), _u32(ref["mvuRight"])) and np.array_equal(_u32(host["mvDepth"]), _u32(ref["mvDepth"]))
    assert np.array_equal(host["cell_start"], ref["cell_start"]) and np.array_equal(host["cell_idx"], ref["cell_idx"])
    if bounds:
        assert np.array_equal(_u32(host["bounds"]), _u32(ref["bounds"])), (host["bounds"], ref["bounds"])
    dev = F.resident.read(stereo=S.kind != "mono")
    assert _bits(dev["keys_un"]) == _bits(ref["mvKeysUn"]) and _bits(dev["desc"]) == _bits(ref["mDescriptors"])
    if S.kind != "mono":
        assert np.array_equal(_u32(dev["u_right"]), _u32(ref["mvuRight"])) and np.array_equal(_u32(dev["depth"]), _u32(ref["mvDepth"]))
    assert np.array_equal(dev["cell_start"], ref["cell_start"]) and np.array_equal(dev["cell_idx"], ref["cell_idx"])
    n, nl = C.c_int32(), C.c_int32()
    assert F.resident._lib.borb_frame_info(F.resident._h, C.byref(n), C.byref(nl), None) == 0
    assert n.value == N and nl.value == ref["mnScaleLevels"]
    for got, f in ((F.mvScaleFactors, "mvScaleFactors"), (S.XL.GetInverseScaleFactors(), "mvInvScaleFactors"),
                   (S.XL.GetScaleSigmaSquares(), "mvLevelSigma2"), (S.XL.GetInverseScaleSigmaSquares(), "mvInvLevelSigma2")):
        assert _bits(np.float32(got)) == _bits(ref[f]), f
    assert np.float32(S.XL.GetScaleFactor()) == ref["mfScaleFactor"]
    F.resident.close()


def run(O, S, left, right=None, K=EUROC_K, dist=(0, 0, 0, 0), bf=EUROC_BF, depth=None, factor=1.0, ref_depth=None, fresh=True):
    F, host = S.frame(left, right, K, dist, bf, depth, factor)
    ref = O.ref_frame(S.kind, left, right, nfeatures=S.nf, scale_factor=S.sf, nlevels=S.nl, K=K, dist=dist, bf=bf,
                      depth=ref_depth if ref_depth is not None else depth, fresh=fresh)
    check(O, S, F, host, ref, bounds=not ref["mbInitialComputations"])
    return ref


# ---------------------------------------------------------------------------------------------------------------- stereo
@pytest.mark.parametrize("shape,nf,K,bf", [((1242, 375), (2000, 2000), KITTI_K, KITTI_BF),
                                           ((752, 480), (1200, 1500), EUROC_K, EUROC_BF),
                                           ((752, 480), (1500, 1200), EUROC_K, EUROC_BF),
                                           ((1241, 376), (2000, 2000), KITTI_K, KITTI_BF),
                                           ((753, 479), (1200, 1200), EUROC_K, EUROC_BF),
                                           ((221, 221), (500, 500), EUROC_K, EUROC_BF)],
                         ids=["kitti_2000", "euroc_1200_1500", "euroc_1500_1200", "odd_1241x376", "odd_753x479", "smallest_221"])
def test_stereo_sizes(O, shape, nf, K, bf):
    L, R, _ = synth.stereo_pair(7, 0, 0, *shape)
    ref = run(O, Stream("stereo", nf), L, R, K, bf=bf)
    assert ref["N"] > (50 if shape[0] < 300 else 500) and (ref["mvuRight"] >= 0).sum() > (5 if shape[0] < 300 else 100)


@pytest.mark.parametrize("case", ["barrel_4", "tum1_5", "icdist_negative", "pincushion", "k1_zero_rest_nonzero"])
def test_stereo_distorted(O, case):
    """The first stereo frames with k1 != 0: mvKeysUn undistorted, the grid and the bounds from the undistorted corners, while the
    association runs on the distorted keypoints."""
    K, dist = fic.DIST_CASES[case]
    L, R, _ = synth.stereo_pair(8, 0, 0, 752, 480)
    ref = run(O, Stream("stereo", (1500, 1500)), L, R, K, dist, bf=EUROC_BF)
    assert (dist[0] == 0) == (_bits(ref["mvKeysUn"]) == _bits(ref["mvKeys"]))
    assert (ref["mvuRight"] >= 0).sum() > 100


@pytest.mark.parametrize("sf,nl", [(1.2, 1), (1.1, 12), (1.5, 4)])
def test_stereo_levels(O, sf, nl):
    L, R, _ = synth.stereo_pair(9, 0, 0, 752, 480)
    ref = run(O, Stream("stereo", (1500, 1500), sf, nl), L, R, EUROC_K, fic.DIST_CASES["barrel_4"][1], bf=EUROC_BF)
    assert ref["mnScaleLevels"] == nl and ref["N"] > 500


def test_stereo_handle_at_feature_limit(O):
    """Handles whose capacity is exactly BORB_MATCH_MAX_FEATURES (the largest the call accepts)."""
    lo, hi = 1000, 8192
    while lo < hi:                                        # the largest nfeatures whose capacity stays within the limit
        mid = (lo + hi + 1) // 2
        if _X(mid).capacity(1242, 375) <= 8192:
            lo = mid
        else:
            hi = mid - 1
    assert _X(lo).capacity(1242, 375) == 8192, "no nfeatures gives a capacity of exactly 8192 at 1242x375"
    L, R, _ = synth.stereo_pair(10, 0, 0, 1242, 375)
    ref = run(O, Stream("stereo", (lo, lo)), L, R, KITTI_K, bf=KITTI_BF)
    assert ref["N"] > 4000


def test_stereo_blank_images(O):
    """A blank right image: N > 0 and every mvuRight -1 (the reference reaches :627 with an empty vDistIdx).  A blank left image:
    N = 0, the reference returns at :85; as a first frame it leaves the statics alone."""
    L, R, _ = synth.stereo_pair(11, 0, 0, 752, 480)
    blank = np.zeros_like(L)
    S = Stream("stereo", (1200, 1200))
    ref = run(O, S, L, blank, K=EUROC_K, dist=fic.DIST_CASES["barrel_4"][1])
    assert ref["N"] > 500 and len(ref["mvKeysRight"]) == 0 and np.all(ref["mvuRight"] == -1) and np.all(ref["mvDepth"] == -1)
    ref = run(O, Stream("stereo", (1200, 1200)), blank, R)
    assert ref["N"] == 0 and len(ref["mvKeysRight"]) > 500 and ref["mbInitialComputations"]


# ----------------------------------------------------------------------------------------------------------------- RGB-D
@pytest.mark.parametrize("case", ["tum1_5", "k1_zero_rest_nonzero", "pincushion", "icdist_negative"])
def test_rgbd_distortion(O, case):
    K, dist = fic.DIST_CASES[case]
    depth = fic.edge_depth_float(21)
    ref = run(O, Stream("rgbd", (1500, 0)), synth.mono_frame(21, 0, 0, 640, 480), K=K, dist=dist, bf=40.0, depth=depth)
    assert (ref["mvDepth"] > 0).sum() > 100


@pytest.mark.parametrize("factor", fic.DEPTH_FACTORS)
def test_rgbd_raw_depth(O, factor):
    """Raw CV_16U maps: the reference is fed Tracking::GrabImageRGBD's conversion (src/Tracking.cc:227-228)."""
    K, dist = fic.DIST_CASES["tum1_5"]
    raw = fic.edge_depth_raw(22)
    img = synth.mono_frame(22, 0, 0, 640, 480)
    ref = run(O, Stream("rgbd", (1500, 0)), img, K=K, dist=dist, bf=40.0, depth=raw, factor=factor,
              ref_depth=O.port_depth_to_float(raw, factor))
    assert fic.keys_on_depth_specials(ref["mvKeys"], O.port_depth_to_float(raw, factor)) > 50
    assert (ref["mvDepth"] > 0).sum() > 100


def test_rgbd_edge_float_depth_padded_stride(O):
    """Float maps with NaN, +-inf, -0, subnormal and negative depths, handed over with a padded row stride."""
    K, dist = fic.DIST_CASES["tum1_5"]
    depth = fic.edge_depth_float(23)
    padded = np.full((480, 640 + 24), np.float32(7.5))
    padded[:, :640] = depth
    view = padded[:, :640]
    assert view.strides[0] == (640 + 24) * 4
    img = synth.mono_frame(23, 0, 0, 640, 480)
    ref = run(O, Stream("rgbd", (1500, 0)), img, K=K, dist=dist, bf=40.0, depth=view, ref_depth=depth)
    assert fic.keys_on_depth_specials(ref["mvKeys"], depth) > 50


# ------------------------------------------------------------------------------------------------------------- monocular
@pytest.mark.parametrize("case", sorted(fic.DIST_CASES))
def test_monocular_initialisation_extractor(O, case):
    """The initialisation extractor: 2 x nFeatures (src/Tracking.cc:158-159)."""
    K, dist = fic.DIST_CASES[case]
    ref = run(O, Stream("mono", (4000, 0)), synth.mono_frame(24, 0, 0, 640, 480), K=K, dist=dist)
    assert ref["N"] > 2000


# ------------------------------------------------------------------------------------------------------------- sequences
@pytest.mark.parametrize("kind", ["stereo", "rgbd", "mono"])
def test_sequence(O, kind):
    """12 frames on the same handles and matcher, starting with a blank frame; the reference starts a process once (fresh for
    frame 0 only), as Tracking does, so frame 0 leaves the statics alone and frame 1 computes them."""
    K, dist = fic.DIST_CASES["barrel_4"]
    S = Stream(kind, (1200, 1000))
    blank = np.zeros((480, 752), np.uint8)
    ids = []
    for t in range(12):
        L, R, _ = synth.stereo_pair(100 + t, 0, 0, 752, 480)
        if t == 0:
            L = R = blank
        elif t == 5 and kind == "stereo":
            R = blank
        depth = fic.edge_depth_float(200 + t, 752, 480) if kind == "rgbd" else None
        ref = run(O, S, L, R if kind == "stereo" else None, K, dist, EUROC_BF, depth=depth, fresh=t == 0)
        ids.append(ref["mnId"])
        assert (ref["N"] == 0) == (t == 0) and ref["mbInitialComputations"] == (t == 0)
    assert ids == list(range(ids[0], ids[0] + 12))


# --------------------------------------------------------------------------------------------------------------- threads
def test_four_streams_on_four_threads(O):
    """Four streams, each with its own matcher and handle pair on its own thread, build 8 stereo frames each at the same time;
    every frame equals the verbatim constructor, run on one thread afterwards."""
    K, dist = fic.DIST_CASES["barrel_4"]
    imgs = [[synth.stereo_pair(300 + 10 * s + t, 0, 0, 752, 480)[:2] for t in range(8)] for s in range(4)]
    streams = [Stream("stereo", (1000 + 100 * s, 1100)) for s in range(4)]
    out = [[None] * 8 for _ in range(4)]
    errors = []
    start = threading.Barrier(4)

    def work(s):
        try:
            start.wait()
            for t in range(8):
                F, host = streams[s].frame(*imgs[s][t], K, dist, EUROC_BF)
                dev = F.resident.read(stereo=True)
                out[s][t] = (F, {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in host.items()}, dev)
        except Exception as e:                      # noqa: BLE001 - reported below
            errors.append(e)

    th = [threading.Thread(target=work, args=(s,)) for s in range(4)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
    for s in range(4):
        for t in range(8):
            F, host, dev = out[s][t]
            ref = O.ref_frame("stereo", *imgs[s][t], nfeatures=streams[s].nf, K=K, dist=dist, bf=EUROC_BF, fresh=True)
            check(O, streams[s], F, host, ref)
            assert _bits(dev["keys_un"]) == _bits(ref["mvKeysUn"]) and np.array_equal(_u32(dev["u_right"]), _u32(ref["mvuRight"]))
            assert np.array_equal(dev["cell_idx"], ref["cell_idx"])
