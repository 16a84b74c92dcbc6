"""GPU sweep of the extraction kernels across image geometries and quadtree envelopes, stage by stage against the port.

The sizes (tests/extract_geometry.py SIZES) are chosen so that every tiling edge of the kernels is hit on purpose: every
level-width residue mod 4, a pitch with no slack, blur strips that end full or one pixel wide, single-column and
single-row cell grids, FAST cells at the 4/3/2-cells-per-CTA switches, and the smallest accepted frame.  The quadtree is
driven across its on-chip candidate limit with dot images of exact level-0 candidate counts, and to the largest quota its
shared-memory envelope accepts."""
import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import extract_geometry as EG
from tests.extract_geometry import DOT_CASES, DOT_NFEATURES, ENVELOPE
from tests.test_gpu_extract import assert_kps_equal

pytestmark = pytest.mark.gpu
BORB_ERR_UNSUPPORTED = 4
IDS = lambda s: f"{s[0]}x{s[1]}"


@pytest.fixture(scope="module")
def X():
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor


def images(size):
    w, h = size
    return {"natural": (synth.mono_frame(13, 0, 0, w, h), 1000), "noise": (synth.white_noise(14, w, h), 2000)}


def assert_stages_equal(G, P, kg, dg, kp, dp, nlevels=8, image=0):
    """Pyramid, blur, FAST candidates (multiset), quadtree count and order, then keypoints and descriptors bit for bit."""
    for l in range(nlevels):
        assert np.array_equal(G.pyramid(l, image), P.level(l)), f"pyramid level {l}"
        if P.blurred(l) is not None:
            assert np.array_equal(G.debug_blurred(l, image), P.blurred(l)), f"blur level {l}"
        cg, cp = G.debug_candidates(l, image), P.candidates(l)
        assert sorted(map(tuple, cg.tolist())) == sorted(map(tuple, cp.tolist())), f"FAST candidates level {l}"
        sel = G.debug_selected(l, image)
        m = kp["octave"] == l
        assert len(sel) == int(m.sum()), f"quadtree count level {l}"
        assert np.array_equal(sel[:, 2], kp["response"][m].astype(np.int32)), f"quadtree order level {l}"
    assert_kps_equal(kg, dg, kp, dp)


@pytest.mark.parametrize("kind", ["natural", "noise"])
@pytest.mark.parametrize("size", EG.SIZES, ids=IDS)
def test_sweep_matches_port_all_stages(X, oracle, size, kind):
    img, nf = images(size)[kind]
    G, P = X(nf), oracle.PortExtractor(nf)
    kg, dg = G(img)
    kp, dp = P(img)
    assert_stages_equal(G, P, kg, dg, kp, dp)


@pytest.mark.parametrize("size", EG.SIZES, ids=IDS)
def test_stale_state_equals_fresh_handle(X, size):
    """A handle that just processed another size and content (saturated noise, every candidate buffer full) must give what a
    fresh handle gives, alone and as both images of a batch: stale pitch slack, padding or counts would show here."""
    w, h = size
    a, b = synth.mono_frame(15, 0, 0, w, h), synth.white_noise(16, w, h)
    fresh, want = [], []
    for im in (a, b):
        F = X(1000)
        fresh.append(F(im))
        want.append([(sorted(map(tuple, F.debug_candidates(l).tolist())), F.debug_selected(l).tolist()) for l in range(8)])
    G = X(1000)
    ow, oh = (w + 97, h + 61) if (w + 97, h + 61) not in EG.SIZES else (w + 98, h + 61)
    G(np.where(synth.white_noise(17, ow, oh) > 127, 255, 0).astype(np.uint8))
    kg, dg = G(a)
    assert_kps_equal(kg, dg, *fresh[0])
    G(np.full((oh, ow), 255, np.uint8))
    outs = G.extract_batch([b, a])
    for i, ((kb, db), (kf, df), wn) in enumerate(zip(outs, fresh[::-1], want[::-1])):
        assert_kps_equal(kb, db, kf, df)
        for l in range(8):
            assert sorted(map(tuple, G.debug_candidates(l, i).tolist())) == wn[l][0], (i, l)
            assert G.debug_selected(l, i).tolist() == wn[l][1], (i, l)


def test_size_limits(X, oracle):
    from orb_slam2_b200._lib import BorbError
    G = X(1000)
    for (w, h) in [(221, 221), (221, 300), (640, 221)]:
        img = synth.mono_frame(18, 0, 0, w, h)
        P = oracle.PortExtractor(1000)
        kp, dp = P(img)
        assert_stages_equal(G, P, *G(img), kp, dp)
        for (rw, rh) in [(w - 1, h), (w, h - 1)] if w == h else []:
            with pytest.raises(BorbError) as e:
                G(synth.mono_frame(18, 0, 0, rw, rh))
            assert e.value.status == BORB_ERR_UNSUPPORTED
    for (rw, rh) in [(220, 220), (220, 300), (640, 220), (221, 480)]:
        with pytest.raises(BorbError) as e:
            G(synth.mono_frame(19, 0, 0, rw, rh))
        assert e.value.status == BORB_ERR_UNSUPPORTED
    img = synth.mono_frame(20, 0, 0, 221, 221)         # the handle still works after the refusals
    assert_kps_equal(*G(img), *oracle.PortExtractor(1000)(img))


@pytest.mark.parametrize("case", DOT_CASES, ids=lambda c: f"{c[0]}-seed{c[3]}")
def test_quadtree_onchip_boundary(X, oracle, case):
    """Exactly 5119 / 5120 / 5121 candidates on level 0 (the register path holds 256 x 20 = 5120), and more than twice that."""
    target, n, (w, h), seed = case
    img = EG.dot_image(n, w, h, seed)
    G, P = X(DOT_NFEATURES), oracle.PortExtractor(DOT_NFEATURES)
    kg, dg = G(img)
    kp, dp = P(img)
    got = len(G.debug_candidates(0))
    print(f"dot image {w}x{h} seed {seed}: {got} level-0 candidates, {len(G.debug_selected(0))} selected")
    assert got == target == len(P.candidates(0))
    assert_stages_equal(G, P, kg, dg, kp, dp)
    both = G.extract_batch([img, img[:, ::-1].copy()])
    assert_kps_equal(*both[0], kp, dp)
    assert_kps_equal(*both[1], *P(img[:, ::-1].copy()))


@pytest.mark.parametrize("sf,nl,nf", ENVELOPE)
def test_node_capacity_envelope(X, oracle, sf, nl, nf):
    """The largest nfeatures whose level-0 node capacity fits the quadtree's 200 KB of shared memory, on white noise where
    the large levels fill their quotas, matches the port; one more feature is refused, not run.  ENVELOPE checks it through
    the table-driven resize kernel (1.2 x 8) and through the generic one (3.0 x 2)."""
    from orb_slam2_b200._lib import BorbError
    img = synth.white_noise(21, *synth.KITTI)
    G, P = X(nf, sf, nl), oracle.PortExtractor(nf, sf, nl)
    kg, dg = G(img)
    kp, dp = P(img)
    assert_stages_equal(G, P, kg, dg, kp, dp, nlevels=nl)
    quota = G.mnFeaturesPerLevel
    cands = [len(G.debug_candidates(l)) for l in range(nl)]
    counts = [int((kg["octave"] == l).sum()) for l in range(nl)]
    print(f"scale {sf} x {nl} levels, nfeatures {nf}: quotas {quota.tolist()}, candidates {cands}, kept {counts}")
    assert counts[0] >= quota[0]                       # level 0 runs at the full node capacity
    for l in range(nl):
        # a level with enough candidates keeps its quota to quota + 3; one without keeps every candidate
        assert quota[l] <= counts[l] <= quota[l] + 3 if cands[l] >= quota[l] else counts[l] == cands[l], l
    with pytest.raises(BorbError) as e:
        X(nf + 1, sf, nl)(img)
    assert e.value.status == BORB_ERR_UNSUPPORTED


# the smallest size, a level 0 with no pitch slack (h 240: one cell row at the top levels), two odd widths
@pytest.mark.parametrize("size", [(221, 221), (376, 240), (641, 480), (1195, 240), (1087, 375)], ids=IDS)
def test_stereo_at_edge_sizes(X, oracle, size):
    w, h = size
    bf, fx = 40.0, 525.0
    pairs = [synth.stereo_pair(400 + i, 0, 0, w, h) for i in range(2)]
    outs = X(1000).stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], bf, fx)
    for (L, R, _), out in zip(pairs, outs):
        EL, ER = oracle.PortExtractor(1000), oracle.PortExtractor(1000)
        kl, dl = EL(L)
        kr, dr = ER(R)
        ur, dp, _ = oracle.port_stereo(kl, dl, kr, dr, [EL.level(i) for i in range(8)], [ER.level(i) for i in range(8)],
                                       EL.scale, EL.inv_scale, bf, fx)
        assert_kps_equal(out["mvKeys"], out["mDescriptors"], kl, dl)
        assert_kps_equal(out["mvKeysRight"], out["mDescriptorsRight"], kr, dr)
        assert np.array_equal(out["mvuRight"], ur), int((out["mvuRight"] != ur).sum())
        assert np.array_equal(out["mvDepth"], dp)
