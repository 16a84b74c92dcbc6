"""CPU: the reference's three Frame constructors (src/Frame.cc:61-228), run unmodified through libframector.so's framector_run on
what the verbatim ORBextractor.cc finds on the same images (oracle.ref_frame).  Pins the whole constructor — its order of steps,
its early return on an empty mvKeys, the once-per-process statics and the mb it reads before assigning it — to the pieces that
tests/test_oracle_frame_ref.py already pins (ComputeStereoMatches, the RGB-D leg, the grid) and to their restatements.
tests/test_gpu_frame_ctor_ref.py holds borb_frame_from_extractors to the same constructor."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import frame_input_cases as fic


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_framector() and oracle.have_ref()):
        pytest.skip("oracle/_ref/libframector.so / liborbref.so not built (reference tree absent)")
    return oracle


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _logf(x):
    f = C.CDLL("libm.so.6").logf
    f.restype, f.argtypes = C.c_float, [C.c_float]
    return np.float32(f(float(np.float32(x))))


def _images(kind, seed, w=640, h=480):
    if kind == "stereo":
        L, R, _ = synth.stereo_pair(seed, 0, 0, w, h)
        return L, R
    return synth.mono_frame(seed, 0, 0, w, h), None


@pytest.mark.parametrize("case", sorted(fic.DIST_CASES))
@pytest.mark.parametrize("kind", ["mono", "stereo", "rgbd"])
def test_constructor_equals_pinned_pieces(O, kind, case):
    """Every member of the verbatim constructor equals the extraction, ref_stereo / ref_rgbd_frame / ref_assign_grid on it, and the
    restatements (port_stereo, port_rgbd_frame, port_assign_grid).  Stereo frames with k1 != 0 undistort mvKeysUn and bound the
    grid by the undistorted corners, while ComputeStereoMatches works on the distorted mvKeys."""
    K, dist = fic.DIST_CASES[case]
    bf = 40.0
    left, right = _images(kind, 21)
    depth = fic.edge_depth_float(3) if kind == "rgbd" else np.zeros((480, 640), np.float32)
    r = O.ref_frame(kind, left, right, nfeatures=(1500, 1300), K=K, dist=dist, bf=bf, th_depth=35.0, depth=depth)
    (kl, dl), (kr, dr) = r["extractor_keys"]
    N = len(kl)
    assert r["N"] == N > 1000
    assert _bits(r["mvKeys"]) == _bits(kl) and _bits(r["mDescriptors"]) == _bits(dl)
    assert _bits(r["mvKeysRight"]) == _bits(kr if kind == "stereo" else kr[:0])
    assert _bits(r["mDescriptorsRight"]) == _bits(dr if kind == "stereo" else dr[:0])
    K4, D = np.array(K, np.float32), np.array(dist, np.float32)
    leg = O.ref_rgbd_frame(kl, K4, D, bf, depth)                  # UndistortKeyPoints + ComputeImageBounds (+ the depth lookup)
    port = O.port_rgbd_frame(kl, K4, D, bf, depth)
    assert _bits(port["keys_un"]) == _bits(leg["keys_un"]) and _bits(port["bounds"]) == _bits(leg["bounds"])
    assert _bits(r["mvKeysUn"]) == _bits(leg["keys_un"]) and _bits(r["bounds"]) == _bits(leg["bounds"])
    assert (D[0] == 0) == (_bits(r["mvKeysUn"]) == _bits(kl))
    if kind == "stereo":
        E = r["extractor_tables"]
        scale, inv = E[:8], E[8:16]
        ur, dp = O.ref_stereo(kl, dl, kr, dr, r["pyramid"], r["pyramid_right"], scale, inv, bf, K[0])
        ur_p, dp_p, _ = O.port_stereo(kl, dl, kr, dr, r["pyramid"], r["pyramid_right"], scale, inv, bf, K[0])
        assert _bits(r["mvuRight"]) == _bits(ur) == _bits(ur_p) and _bits(r["mvDepth"]) == _bits(dp) == _bits(dp_p)
        assert (ur >= 0).sum() > 100
    elif kind == "rgbd":
        assert _bits(r["mvuRight"]) == _bits(leg["u_right"]) and _bits(r["mvDepth"]) == _bits(leg["depth"]) and leg["count"] > 100
    else:
        assert np.all(r["mvuRight"] == -1) and np.all(r["mvDepth"] == -1) and len(r["mvuRight"]) == N     # Frame.cc:201-202
    cs, ci = O.ref_assign_grid(r["mvKeysUn"], r["bounds"])
    cs_p, ci_p = O.port_assign_grid(r["mvKeysUn"], r["bounds"])
    assert np.array_equal(r["cell_start"], cs) and np.array_equal(r["cell_idx"], ci)
    assert np.array_equal(cs, cs_p) and np.array_equal(ci, ci_p)
    assert r["mbf"] == np.float32(bf) and r["mThDepth"] == np.float32(35.0)


def test_statics_follow_the_first_frame(O):
    """mnId counts every constructor, N = 0 frames included; an N = 0 first frame returns (Frame.cc:85/140/195) before the
    once-per-process block (:96-112), so the bounds, grid inverses and fx..invfy stay as they were and the next frame computes
    them; a later frame with another camera keeps the first frame's statics, and its mb = mbf/fx uses that first fx (:114)."""
    Ka, da = fic.DIST_CASES["barrel_4"]
    Kb, db = fic.DIST_CASES["tum1_5"]
    Kc, dc = fic.DIST_CASES["pincushion"]
    img = synth.mono_frame(31, 0, 0, 640, 480)
    blank = np.zeros((480, 640), np.uint8)
    a = O.ref_frame("mono", img, nfeatures=1000, K=Ka, dist=da, fresh=True)
    assert not a["mbInitialComputations"]
    e = O.ref_frame("mono", blank, nfeatures=1000, K=Kb, dist=db, fresh=True)
    assert e["N"] == 0 and e["mnId"] == a["mnId"] + 1 and e["mbInitialComputations"]
    assert len(e["mvKeysUn"]) == len(e["mvuRight"]) == len(e["cell_idx"]) == 0 and np.all(e["cell_start"] == 0)
    for f in ("bounds", "grid_inv", "fx", "fy", "cx", "cy", "invfx", "invfy"):
        assert _bits(e[f]) == _bits(a[f]), f                                            # untouched by the empty frame
    b = O.ref_frame("rgbd", img, nfeatures=1000, K=Kb, dist=db, bf=40.0, depth=fic.edge_depth_float(4), fresh=False)
    assert b["mnId"] == e["mnId"] + 1 and not b["mbInitialComputations"]
    leg = O.ref_rgbd_frame(b["mvKeys"], np.float32(Kb), np.float32(db), 40.0, fic.edge_depth_float(4))
    assert _bits(b["bounds"]) == _bits(leg["bounds"]) and not np.array_equal(b["bounds"], a["bounds"])
    bx = b["bounds"]
    assert b["grid_inv"][0] == np.float32(64) / np.float32(bx[2] - bx[0]) and b["grid_inv"][1] == np.float32(48) / np.float32(bx[3] - bx[1])
    assert (b["fx"], b["fy"], b["cx"], b["cy"]) == tuple(np.float32(Kb))
    assert b["invfx"] == np.float32(1) / np.float32(Kb[0]) and b["invfy"] == np.float32(1) / np.float32(Kb[1])
    c = O.ref_frame("stereo", *synth.stereo_pair(32, 0, 0, 640, 480)[:2], nfeatures=(1000, 1000), K=Kc, dist=dc, bf=40.0, fresh=False)
    assert c["mnId"] == b["mnId"] + 1
    for f in ("bounds", "grid_inv", "fx", "fy", "cx", "cy", "invfx", "invfy"):
        assert _bits(c[f]) == _bits(b[f]), f                                            # the first frame's camera
    assert c["mb"] == np.float32(40.0) / np.float32(Kb[0]) != np.float32(40.0) / np.float32(Kc[0])
    cs, ci = O.ref_assign_grid(c["mvKeysUn"], b["bounds"])                             # the grid uses the kept bounds
    assert np.array_equal(c["cell_start"], cs) and np.array_equal(c["cell_idx"], ci)


def test_stereo_mb_prefill(O):
    """ComputeStereoMatches reads mb (Frame.cc:496-498) before the constructor assigns it (:114), so the reference's result depends
    on what the Frame's storage held: an indeterminate value.  borb (like frameref_stereo) uses mbf/fx, the value :114 assigns and
    the search limits are evidently meant to use; ref_frame pre-fills it by default for that reason.  A huge mb
    makes maxD tiny and rejects every match; mb = 0 makes maxD infinite and, on this KITTI-shaped pair, admits one match more."""
    L, R, _ = synth.stereo_pair(7, 0, 0, 1242, 375)
    K, bf = (718.856, 718.856, 607.1928, 185.2157), 386.1448
    base = O.ref_frame("stereo", L, R, nfeatures=(2000, 2000), K=K, bf=bf)
    zero = O.ref_frame("stereo", L, R, nfeatures=(2000, 2000), K=K, bf=bf, mb=0.0)
    huge = O.ref_frame("stereo", L, R, nfeatures=(2000, 2000), K=K, bf=bf, mb=1e30)
    n = [int((x["mvuRight"] >= 0).sum()) for x in (base, zero, huge)]
    assert n == [1146, 1147, 0], n
    for x in (base, zero, huge):                                                         # the constructor's own mb afterwards
        assert x["mb"] == np.float32(bf) / np.float32(K[0])
    E = base["extractor_tables"]
    (kl, dl), (kr, dr) = base["extractor_keys"]
    ur, dp = O.ref_stereo(kl, dl, kr, dr, base["pyramid"], base["pyramid_right"], E[:8], E[8:16], bf, K[0])
    assert _bits(ur) == _bits(base["mvuRight"]) and _bits(dp) == _bits(base["mvDepth"])
    diff = np.nonzero(zero["mvuRight"] != base["mvuRight"])[0]
    assert len(diff) == 1 and base["mvuRight"][diff[0]] == -1


@pytest.mark.parametrize("sf,nl", [(1.2, 8), (1.2, 1), (1.1, 12), (1.5, 4)])
def test_scale_members(O, sf, nl):
    """mnScaleLevels, mfScaleFactor (the extractor's scaleFactor, also with one level), mfLogScaleFactor = logf(mfScaleFactor) and
    the four scale tables equal what the verbatim ORBextractor computes (orbref_tables), for every kind."""
    for kind in ("mono", "stereo", "rgbd"):
        left, right = _images(kind, 40, 640, 480)
        r = O.ref_frame(kind, left, right, nfeatures=(1000, 1000), scale_factor=sf, nlevels=nl, K=fic.TUM1_K, bf=40.0,
                        depth=fic.edge_depth_float(5))
        E = O.ref_extractor(1000, sf, nl)
        assert r["mnScaleLevels"] == nl and r["mfScaleFactor"] == np.float32(sf)
        assert _bits(r["mfLogScaleFactor"]) == _bits(_logf(sf))
        for f, t in (("mvScaleFactors", E.scale), ("mvInvScaleFactors", E.inv_scale), ("mvLevelSigma2", E.sigma2),
                     ("mvInvLevelSigma2", E.inv_sigma2)):
            assert _bits(r[f]) == _bits(t), f
        assert r["N"] > 300
