"""CPU: the stereo port (oracle/orb_port_stereo.cpp) equals the verbatim Frame::ComputeStereoMatches on the envelope cases of
tests/stereo_envelope.py — scale factors 1.05 to 2.5, 3 to 12 levels, 11200-feature frames, a 4095-row frame, periodic, shifted,
identical, blank and nearly blank pairs, two handles with differing nfeatures — and those cases reach every coverage class listed
in stereo_envelope.CLASSES.  tests/test_gpu_stereo_envelope.py pins the CUDA library to the port on the same cases."""
import numpy as np
import pytest

from tests import stereo_envelope as E


@pytest.fixture(scope="module")
def O(oracle):
    if not oracle.have_frameref():
        pytest.skip("oracle/_ref/libframeref.so not built (reference tree absent)")
    return oracle


def test_every_case_is_an_accepted_geometry():
    for name in E.NAMES:
        assert E.geometry_ok(E.CASES[name]) is None, (name, E.geometry_ok(E.CASES[name]))


@pytest.mark.parametrize("name", E.NAMES)
def test_port_equals_numpy_restatement(oracle, name):
    p = E.run_port(oracle, name)
    ur, dp, _, _ = E.restate(oracle, name)
    assert np.array_equal(p["ur"], ur), int((p["ur"] != ur).sum())
    assert np.array_equal(p["dp"], dp), int((p["dp"] != dp).sum())


@pytest.mark.parametrize("name", E.NAMES)
def test_port_equals_reference(O, name):
    c = E.CASES[name]
    p = E.run_port(O, name)
    if not E.ref_eligible(O, name):
        # reference-asserting windows, or nothing accepted (UB in the reference): the port's own answer is pinned above
        assert c["ref_asserts"] or not (p["ur"] >= 0).any()
        pytest.skip("the reference cannot run this case (cv::Mat range / empty vDistIdx)")
    bf, fx = c["cam"]
    ur, dp = O.ref_stereo(p["kl"], p["dl"], p["kr"], p["dr"], p["pyrL"], p["pyrR"], p["scale"], p["inv_scale"], bf, fx)
    assert np.array_equal(p["ur"], ur), int((p["ur"] != ur).sum())
    assert np.array_equal(p["dp"], dp), int((p["dp"] != dp).sum())


def test_cases_reach_every_coverage_class(oracle):
    hit = {}
    for name in E.NAMES:
        for k in E.coverage(oracle, name):
            hit.setdefault(k, name)
    assert set(hit) == set(E.CLASSES), sorted(set(E.CLASSES) - set(hit))
    assert not set(E.UNREACHABLE) & set(E.CLASSES)
    # only the reference-asserting case may claim the class that marks it
    assert all(E.CASES[n]["ref_asserts"] for n in E.NAMES if "sad_window_left_of_level" in E.coverage(oracle, n))
    assert all(len(E.run_port(oracle, n)["kr"]) < 1 << E.IR_BITS for n in E.NAMES)       # iR fits the packed key


def test_right_records_exceed_the_left_handles_stride(oracle):
    """Two handles, left 1000 / right 4000 features: the right keypoints need more bin records than a buffer sized from the left
    handle's geometry holds, so the record stride must come from the right handle (borb_stereo_match2)."""
    c = E.CASES["kitti_L1000_R4000"]
    n = E.record_count(oracle, "kitti_L1000_R4000")
    assert n > E.rec_stride(c["w"], c["h"], *c["left"]), (n, E.rec_stride(c["w"], c["h"], *c["left"]))
    assert n <= E.rec_stride(c["w"], c["h"], *c["right"])
    # the stride bounds every case's records by the right geometry
    for name in E.NAMES:
        c = E.CASES[name]
        assert E.record_count(oracle, name) <= E.rec_stride(c["w"], c["h"], *c["right"]), name


def test_restated_constants_match_the_geometry():
    # KITTI at 1000 features (1.2 x 8): 1048 keypoint slots, 4 bins per band -> 4192 records
    assert E.sel_image_stride(1242, 375, 1000, 1.2, 8) == 1048
    assert E.rec_stride(1242, 375, 1000, 1.2, 8) == 4192
    assert E.n_bins(4095) == E.SBIN_MAX and E.n_bins(375) == 47


def test_clamped_zero_disparity_matches_survive_the_cull(oracle):
    """half_same_LR: zero-disparity matches of the identical half reach the output as uL - 0.01 (in double) and bf / 0.01f,
    next to the shifted half that keeps the median SAD above zero."""
    c = E.CASES["half_same_LR"]
    p = E.run_port(oracle, "half_same_LR")
    uL = p["kl"]["x"]
    clamped = p["ur"] == (uL.astype(np.float64) - 0.01).astype(np.float32)
    assert clamped.any() and (p["ur"] >= 0).sum() > 100
    assert np.all(p["dp"][clamped] == np.float32(c["cam"][0]) / np.float32(0.01))
