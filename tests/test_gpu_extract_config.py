"""GPU sweep of the extractor's configuration domain, stage by stage against the port (tests/extract_config.py).

FAST thresholds at 0, 1, 7, 20, 126-129, 200, 253-255 on exact-score dot images and white noise: the packed reject's
constant boundaries, the unrejected path above 127 where every domain pixel of a tile is queued, pass B at every cell.
Per-level quotas of 0 and 1 and quadtree N on each branch boundary of DistributeOctTree.  One and BORB_MAX_LEVELS pyramid
levels.  And the configurations borb_extractor_create refuses."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import extract_config as XC
from tests.test_gpu_extract import assert_kps_equal
from tests.test_gpu_extract_geometry import assert_stages_equal

pytestmark = pytest.mark.gpu
BORB_ERR_INVALID_ARG = 1


@pytest.fixture(scope="module")
def X():
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor


def _check(X, oracle, img, nf, sf, nl, ini=20, mn=7):
    """GPU == port at every stage; GPU == the verbatim reference where it is built."""
    G, P = X(nf, sf, nl, ini, mn), oracle.PortExtractor(nf, sf, nl, ini, mn)
    kg, dg = G(img)
    kp, dp = P(img)
    assert np.array_equal(G.mnFeaturesPerLevel, P.per_level)
    assert_stages_equal(G, P, kg, dg, kp, dp, nlevels=nl)
    if oracle.have_ref():
        assert_kps_equal(kg, dg, *oracle.RefExtractor(nf, sf, nl, ini, mn)(img))
    return G, kg, dg


@pytest.mark.parametrize("case", XC.THRESHOLD_CASES, ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}")
def test_thresholds_match_port_all_stages(X, oracle, case):
    ini, mn, kind = case
    img, dots = XC.threshold_image(ini, mn, kind)
    G, _, _ = _check(X, oracle, img, XC.THRESHOLD_NFEATURES, 1.2, 8, ini, mn)
    if dots is not None:                 # every level-0 candidate is a planned dot with its planned score
        planned = {(x, y): s for x, y, s, _ in dots}
        assert all(planned.get((x, y)) == s for x, y, s in G.debug_candidates(0).tolist())


@pytest.mark.parametrize("pair", XC.FULL_QUEUE_PAIRS, ids=lambda p: f"{p[0]}-{p[1]}")
@pytest.mark.parametrize("size", XC.FULL_QUEUE_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_full_queues_at_largest_tiles(X, oracle, size, pair):
    """iniThFAST above 127 queues every domain pixel of every tile: the word and pixel queues fill to their capacity at the
    widest (124 px) and tallest (64 rows) FAST tiles; (255, 0) also redoes every cell at minThFAST."""
    w, h = size
    for img in (synth.white_noise(32, w, h), synth.mono_frame(33, 0, 0, w, h)):
        _check(X, oracle, img, 1000, 1.2, 8, *pair)


@pytest.mark.parametrize("pair", XC.THRESHOLD_PAIRS, ids=lambda p: f"{p[0]}-{p[1]}")
def test_mixed_batch_equals_single_calls(X, pair):
    """One batch of a bright-dot, a dark-dot, a noise and a natural image gives each image what a call of its own gives."""
    ini, mn = pair
    w, h = XC.THRESHOLD_SIZE
    imgs = [XC.threshold_image(ini, mn, k)[0] for k in XC.THRESHOLD_KINDS] + [synth.mono_frame(34, 0, 0, w, h)]
    G = X(XC.THRESHOLD_NFEATURES, 1.2, 8, ini, mn)
    single = []
    for im in imgs:
        k, d = G(im)
        single.append((k, d, [(sorted(map(tuple, G.debug_candidates(l).tolist())), G.debug_selected(l).tolist()) for l in range(8)]))
    outs = G.extract_batch(imgs)
    for i, ((kb, db), (ks, ds, st)) in enumerate(zip(outs, single)):
        assert_kps_equal(kb, db, ks, ds)
        for l in range(8):
            assert sorted(map(tuple, G.debug_candidates(l, i).tolist())) == st[l][0], (i, l)
            assert G.debug_selected(l, i).tolist() == st[l][1], (i, l)


@pytest.mark.parametrize("case", XC.quadtree_cases(), ids=lambda c: f"N{c[0]}-L{c[1]}")
def test_quadtree_quotas_match_port(X, oracle, case):
    """Quadtree N on DistributeOctTree's branch boundaries (one level: N = nfeatures) and quotas of 0 and 1 (8 levels)."""
    nf, nl = case
    img = XC.quadtree_image()
    G, _, _ = _check(X, oracle, img, nf, 1.2, nl)
    P = oracle.PortExtractor(nf, 1.2, nl)
    P(img)
    for l, (xys, w, h, N) in enumerate(XC.level_inputs(P, nl)):
        sel, _ = XC.distribute(xys, w, h, N)
        assert len(G.debug_selected(l)) == len(sel), l


@pytest.mark.parametrize("case", XC.LEVEL_CASES, ids=lambda c: f"{c[0]}-{c[1]}x{c[2]}")
def test_level_counts_match_port(X, oracle, case):
    nf, sf, nl = case
    img = XC.level_image()
    G, kg, dg = _check(X, oracle, img, nf, sf, nl)
    assert set(kg["octave"].tolist()) == set(range(nl))
    both = G.extract_batch([img, img[::-1].copy()])
    assert_kps_equal(*both[0], kg, dg)
    assert_kps_equal(*both[1], *oracle.PortExtractor(nf, sf, nl)(img[::-1].copy()))


REFUSED = [  # (n_features, scale_factor, n_levels, ini_th_fast, min_th_fast, field the error text names)
    (1000, 1.2, 0, 20, 7, "levels"), (1000, 1.2, XC.MAX_LEVELS + 1, 20, 7, "levels"), (0, 1.2, 8, 20, 7, "n_features"),
    (1000, 1.0, 8, 20, 7, "scale"), (1000, float("nan"), 8, 20, 7, "scale"),
    (1000, 1.2, 8, -1, 7, "ini_th_fast"), (1000, 1.2, 8, 256, 7, "ini_th_fast"),
    (1000, 1.2, 8, 20, -1, "min_th_fast"), (1000, 1.2, 8, 20, 256, "min_th_fast"),
]


@pytest.mark.parametrize("cfg", REFUSED, ids=lambda c: "-".join(map(str, c[:5])))
def test_create_refuses_config(X, cfg):
    from orb_slam2_b200 import _lib
    *args, field = cfg
    so = _lib.load()
    h = C.c_void_p(0x1000)
    assert so.borb_extractor_create(C.byref(_lib.ExtractorCfg(*args)), 0, C.byref(h)) == BORB_ERR_INVALID_ARG
    assert h.value is None
    assert field in so.borb_last_error().decode()
    with pytest.raises(_lib.BorbError) as e:
        X(*args)
    assert e.value.status == BORB_ERR_INVALID_ARG


def test_create_accepts_threshold_bounds(X, oracle):
    """0 and 255 are accepted for both thresholds, in either order."""
    img = synth.mono_frame(35, 0, 0, *XC.THRESHOLD_SIZE)
    for ini, mn in [(0, 255), (255, 0)]:
        _check(X, oracle, img, 1000, 1.2, 8, ini, mn)
