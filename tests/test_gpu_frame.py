"""GPU parity of the device-side Frame constructor tail (borb_frames_from_extractor: UndistortKeyPoints, ComputeStereoFromRGBD,
AssignFeaturesToGrid — reference src/Frame.cc:404-434, 643-664, 230-245) against oracle/orb_port_frame.cpp (itself pinned to the
verbatim Frame.cc and to cv2.undistortPoints in tests/test_oracle_frame_ref.py), and of the matcher calls that run on the resulting
resident frames.  BASELINE configs[2]: RGB-D TUM-shaped 640x480."""
import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu

TUM1_K = (517.306408, 516.469215, 318.643040, 255.313989)
TUM1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)


def _depth_raw(seed, w=640, h=480):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    raw = (5000.0 * (1.5 + 0.8 * np.sin(xx / 90.0 + seed) * np.cos(yy / 70.0))).astype(np.uint16)
    raw[rng.random((h, w)) < 0.15] = 0
    return raw


@pytest.mark.parametrize("dist", [TUM1_DIST, (0.0, 0.0, 0.0, 0.0, 0.0)])
@pytest.mark.parametrize("raw16", [True, False])
def test_rgbd_frames_from_extractor(oracle, dist, raw16):
    from orb_slam2_b200 import matcher as M
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(1000)
    imgs = [synth.mono_frame(40 + i, 0, 0, 640, 480) for i in range(3)]
    outs = X.extract_batch(imgs)
    raws = [_depth_raw(i) for i in range(3)]
    factor = np.float32(1.0 / 5000.0)
    depths_f = [oracle.port_depth_to_float(r, factor) for r in raws]
    mt = M.ORBmatcher(0.8, True)
    sel = [2, 0]                                                     # any subset / order of the batch
    frames, host = M.frames_from_extractor(mt, X, sel, [len(outs[i][0]) for i in sel], TUM1_K, dist, bf=40.0, mode=2,
                                           depth=[raws[i] if raw16 else depths_f[i] for i in sel], depth_factor=factor if raw16 else 1.0)
    K4 = np.array(TUM1_K, np.float32)
    for j, i in enumerate(sel):
        keys, desc = outs[i]
        want = oracle.port_rgbd_frame(keys, K4, np.array(dist, np.float32), 40.0, depths_f[i])
        assert np.array_equal(host["keys_un"][j], want["keys_un"])
        assert np.array_equal(host["u_right"][j], want["u_right"]) and np.array_equal(host["depth"][j], want["depth"])
        assert np.array_equal(host["bounds"], want["bounds"])
        assert (want["depth"] > 0).sum() > 500
        # a matcher call on the resident frame == the same call on the host view built from the oracle's frame
        v = dict(w=640, h=480, kl=want["keys_un"], dl=desc, kr=want["keys_un"], dr=desc, ur=want["u_right"],
                 disp=np.zeros((480, 640), np.float32), scale=X.GetScaleFactors(), sigma2=X.GetScaleSigmaSquares())
        F, mps = mf.projection_case(v, 5 + i, n_mp=300)
        F = M.FrameView(want["keys_un"], desc, X.GetScaleFactors(), tuple(float(x) for x in want["bounds"]), mvuRight=want["u_right"], occupied=F.occupied)
        n_o, m_o = oracle.port_search_by_projection(F, mps, 3.0, 0.8)
        import dataclasses
        FR = dataclasses.replace(frames[j], occupied=F.occupied)
        n_g, m_g = mt.SearchByProjection(FR, mps, 3.0)
        assert n_g == n_o > 50 and np.array_equal(m_g, m_o)


def test_mono_and_stereo_frames_from_extractor(oracle):
    from orb_slam2_b200 import matcher as M
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(1000)
    L, R, _ = synth.stereo_pair(3, 0, 0, 640, 360)
    L2, R2, _ = synth.stereo_pair(4, 0, 0, 640, 360)
    bf, fx = 386.1448, 718.856
    res = X.stereo_frames([L, L2], [R, R2], bf, fx)
    mt = M.ORBmatcher(0.9, True)
    K = (fx, fx, 320.0, 180.0)
    frames, host = M.frames_from_extractor(mt, X, [0, 2], [len(res[0]["mvKeys"]), len(res[1]["mvKeys"])], K, bf=bf, mode=1)
    for j in range(2):
        assert np.array_equal(host["keys_un"][j], res[j]["mvKeys"])                      # no distortion: mvKeysUn = mvKeys
        assert np.array_equal(host["u_right"][j], res[j]["mvuRight"]) and np.array_equal(host["depth"][j], res[j]["mvDepth"])
    assert np.array_equal(host["bounds"], np.array([0, 0, 640, 360], np.float32))
    # the motion-model search on the resident stereo frame == on the host view of the same frame
    v = dict(w=640, h=360, kl=res[0]["mvKeys"], dl=res[0]["mDescriptors"], kr=res[0]["mvKeysRight"], dr=res[0]["mDescriptorsRight"],
             ur=res[0]["mvuRight"], disp=np.zeros((360, 640), np.float32), scale=X.GetScaleFactors(), sigma2=X.GetScaleSigmaSquares())
    Cur, Last, Tcw, Kc = mf.last_frame_case(v, 21, K=(fx, fx, 320.0, 180.0))
    import dataclasses
    CurR = dataclasses.replace(frames[0], occupied=Cur.occupied)
    a = mt.SearchByProjectionLast(Cur, Last, Tcw, Kc, bf, 7.0)
    b = mt.SearchByProjectionLast(CurR, Last, Tcw, Kc, bf, 7.0)
    o = oracle.port_search_by_projection_last(Cur, Last, Tcw, Kc, bf, 7.0, False, False, True)
    assert a[0] == b[0] == o[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[1], o[1])
    # monocular frames: no mvuRight
    fm, hm = M.frames_from_extractor(mt, X, [1], [len(res[0]["mvKeysRight"])], K, mode=0)
    assert np.array_equal(hm["keys_un"][0], res[0]["mvKeysRight"]) and fm[0].mvuRight is None


def test_host_view_grids_share_one_launch(oracle):
    """One grid_sort_jobs_kernel builds every feature grid: a matcher call builds the grids of all its host views in one launch,
    and borb_frame_create builds the grid borb_frames_from_extractor builds for the same keypoints."""
    import ctypes as C
    from orb_slam2_b200 import matcher as M
    from orb_slam2_b200.extractor import ORBextractor
    mt = M.ORBmatcher(0.75, True)

    def launches():
        n = C.c_uint64(0)
        assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
        return n.value

    # SearchBySim3 on two host keyframes: the resident batch's launches plus one for both grids, and the same matches
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = mf.sim3_case(mf.two_views(oracle, 7), 21)
    c0 = launches()
    host = mt.SearchBySim3(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K, 7.5)
    n_host = launches() - c0
    R1, R2 = KF1.make_resident(mt), KF2.make_resident(mt)
    c0 = launches()
    batch = mt.SearchBySim3Batch([R1], [R2], [P1], [P2], [(T1w, T2w)], [(S12, S21)], K, 7.5)[0]
    assert n_host == launches() - c0 + 1
    o = oracle.port_search_by_sim3(KF1, KF2, P1, P2, T1w, T2w, S12, S21, K, 7.5)
    assert host[0] == batch[0] == o[0] > 100 and np.array_equal(host[1], batch[1]) and np.array_equal(host[1], o[1])
    # borb_frame_create on the keypoints borb_frames_from_extractor undistorted, within its bounds
    X = ORBextractor(1000)
    outs = X.extract_batch([synth.mono_frame(50, 0, 0, 640, 480)])
    frames, h = M.frames_from_extractor(mt, X, [0], [len(outs[0][0])], TUM1_K, TUM1_DIST, mode=0)
    created = M.FrameView(h["keys_un"][0], outs[0][1], X.GetScaleFactors(), tuple(float(x) for x in h["bounds"])).make_resident(mt)
    a, b = frames[0].resident.read(stereo=False), created.resident.read(stereo=False)
    assert len(a["cell_idx"]) > 500
    assert np.array_equal(a["cell_start"], b["cell_start"]) and np.array_equal(a["cell_idx"], b["cell_idx"])
