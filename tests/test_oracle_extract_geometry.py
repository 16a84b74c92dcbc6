"""CPU checks of the geometry sweep: the Python restatement of build_geometry (tests/extract_geometry.py) against the port's
own pyramid, the coverage of the committed size list, and the port against the reference's ORBextractor.cc compiled
verbatim at every swept size, at the quadtree's on-chip boundary and at the node-capacity envelope."""
import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import extract_geometry as EG

ENVELOPE, DOT_CASES, DOT_NFEATURES = EG.ENVELOPE, EG.DOT_CASES, EG.DOT_NFEATURES


@pytest.mark.parametrize("size", EG.SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_restated_level_shapes_equal_port(oracle, size):
    w, h = size
    P = oracle.PortExtractor(1000)
    P(synth.mono_frame(3, 0, 0, w, h))
    assert [P.level(l).shape for l in range(8)] == EG.level_shapes(w, h)


def test_restated_tables_equal_port(oracle):
    for nf, sf, nl in [(1000, 1.2, 8), (2000, 1.2, 8), (11200, 1.2, 8), (600, 2.0, 3), (3243, 3.0, 2), (1500, 1.1, 12)]:
        P = oracle.PortExtractor(nf, sf, nl)
        scale, inv_scale, quota = EG.scale_tables(nf, sf, nl)
        assert np.array_equal(P.scale, np.array(scale, np.float32)) and np.array_equal(P.inv_scale, np.array(inv_scale, np.float32))
        assert P.per_level.tolist() == quota


def test_sizes_cover_every_edge_class():
    cov = EG.coverage(EG.SIZES)
    missing = [c for c, hit in cov.items() if not hit]
    assert not missing, missing
    assert 20 <= len(EG.SIZES) <= 30 and len(set(EG.SIZES)) == len(EG.SIZES)


def test_refusal_conditions():
    assert EG.accepted(221, 221) and not EG.accepted(220, 221) and not EG.accepted(221, 220)
    assert EG.accepted(221, 300) and EG.accepted(640, 221)
    assert not EG.accepted(221, 480)                 # 189/448 rounds to zero quadtree roots
    assert not EG.accepted(4096, 480) and EG.accepted(4095, 480)
    for sf, nl, nf in ENVELOPE:
        assert EG.accepted(*synth.KITTI, nfeatures=nf, scale_factor=sf, nlevels=nl)
        assert not EG.accepted(*synth.KITTI, nfeatures=nf + 1, scale_factor=sf, nlevels=nl)
        levels, _ = EG.geometry(*synth.KITTI, nfeatures=nf, scale_factor=sf, nlevels=nl)
        assert max(lv["smem"] for lv in levels) <= EG.QT_SMEM_LIMIT < EG.quadtree_smem_bytes(levels[0]["node_cap"] + 4)
    assert EG.accepted(1280, 720, nfeatures=DOT_NFEATURES)


def test_envelope_cases_take_both_resize_kernels():
    """The envelope is checked through the table-driven resize kernel and through the generic one."""
    windowed = [[lv["x_windowed"] for lv in EG.geometry(*synth.KITTI, nfeatures=nf, scale_factor=sf, nlevels=nl)[0][1:]]
                for sf, nl, nf in ENVELOPE]
    assert windowed == [[True] * 7, [False]]


def test_dot_images_hit_their_candidate_counts(oracle):
    for target, n, (w, h), seed in DOT_CASES:
        P = oracle.PortExtractor(DOT_NFEATURES)
        P(EG.dot_image(n, w, h, seed))
        got = len(P.candidates(0))
        print(f"dot image {w}x{h} seed {seed}: {got} level-0 candidates")
        assert got == target


@pytest.mark.parametrize("size", EG.SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_port_equals_verbatim_reference_at_size(oracle_ref, size):
    w, h = size
    for img, nf in ((synth.mono_frame(5, 0, 0, w, h), 1000), (synth.white_noise(6, w, h), 2000)):
        R, P = oracle_ref.RefExtractor(nf), oracle_ref.PortExtractor(nf)
        kr, dr = R(img)
        kp, dp = P(img)
        assert np.array_equal(kr, kp) and np.array_equal(dr, dp)
        for l in range(8):
            assert np.array_equal(R.level(l), P.level(l)), l


@pytest.mark.parametrize("case", DOT_CASES, ids=lambda c: f"{c[0]}-seed{c[3]}")
def test_port_equals_verbatim_reference_at_onchip_boundary(oracle_ref, case):
    _, n, (w, h), seed = case
    img = EG.dot_image(n, w, h, seed)
    kr, dr = oracle_ref.RefExtractor(DOT_NFEATURES)(img)
    kp, dp = oracle_ref.PortExtractor(DOT_NFEATURES)(img)
    assert np.array_equal(kr, kp) and np.array_equal(dr, dp)


@pytest.mark.parametrize("sf,nl,nf", ENVELOPE)
def test_port_equals_verbatim_reference_at_envelope(oracle_ref, sf, nl, nf):
    img = synth.white_noise(7, *synth.KITTI)
    kr, dr = oracle_ref.RefExtractor(nf, sf, nl)(img)
    kp, dp = oracle_ref.PortExtractor(nf, sf, nl)(img)
    assert np.array_equal(kr, kp) and np.array_equal(dr, dp)
