"""CPU checks of the configuration sweep (tests/extract_config.py): the Python restatement of DistributeOctTree against the
reference's own and the port's, the coverage of the committed case lists, and the port against the reference's
ORBextractor.cc compiled verbatim on every case: FAST thresholds across 0..255, quotas down to zero, 1 and 16 levels."""
import numpy as np
import pytest

from tests import extract_config as XC

QT_IDS = lambda c: f"N{c[0]}-L{c[1]}"
TH_IDS = lambda c: f"{c[0]}-{c[1]}-{c[2]}"


def _assert_port_equals_reference(oracle_ref, img, nf, sf, nl, ini=20, mn=7):
    R, P = oracle_ref.RefExtractor(nf, sf, nl, ini, mn), oracle_ref.PortExtractor(nf, sf, nl, ini, mn)
    assert np.array_equal(R.per_level, P.per_level)
    kr, dr = R(img)
    kp, dp = P(img)
    assert len(kr) == len(kp), (len(kr), len(kp))
    assert np.array_equal(kr, kp) and np.array_equal(dr, dp)
    for l in range(nl):
        assert np.array_equal(R.level(l), P.level(l)), l
    return kp


@pytest.fixture(scope="module")
def quadtree_inputs(oracle):
    """[(case, level, candidates, width, height, quota)] of every level of every quadtree case (the port's candidates)."""
    img, out = XC.quadtree_image(), []
    for nf, nl in XC.quadtree_cases():
        P = oracle.PortExtractor(nf, 1.2, nl)
        P(img)
        out += [((nf, nl), l) + inp for l, inp in enumerate(XC.level_inputs(P, nl))]
    return out


def _random_sets():
    """Small random candidate sets on narrow and wide boxes, at N from 0 to above the candidate count."""
    rng = np.random.default_rng(3)
    for width, height in [(1210, 343), (608, 448), (147, 102), (315, 73)]:
        for n in (1, 2, 7, 40, 300):
            flat = rng.choice((width - 6) * (height - 6), size=n, replace=False)
            xs, ys = 3 + flat % (width - 6), 3 + flat // (width - 6)
            order = np.lexsort((xs, ys))
            xys = np.stack([xs[order], ys[order], rng.integers(7, 60, n)], 1)
            for N in sorted({0, 1, 2, 3, n // 3, n - 1, n, n + 5}):
                yield xys, width, height, N


def test_distribute_restatement_equals_reference(oracle_ref, quadtree_inputs):
    R = oracle_ref.RefExtractor(1000)
    sets = [(c, w, h, N) for _, _, c, w, h, N in quadtree_inputs if len(c)] + list(_random_sets())
    sets += [(c, w, h, N) for c, w, h, _ in sets[:19] for N in (0, 4, 7)]
    for xys, w, h, N in sets:
        sel, _ = XC.distribute(xys, w, h, N)
        want = R.distribute(np.asarray(xys, np.float32), w, h, N).astype(np.int64)
        assert np.array_equal(np.asarray(xys)[sel].reshape(-1, 3), want), (w, h, len(xys), N)


def test_distribute_restatement_equals_port(oracle, quadtree_inputs):
    """The same pin without the verbatim build: the port's distribute is itself pinned to it in test_oracle_extract.py."""
    for _, _, xys, w, h, N in quadtree_inputs:
        sel, _ = XC.distribute(xys, w, h, N)
        want = oracle.port_distribute(np.asarray(xys, np.int32), w, h, N) if len(xys) else np.zeros((0, 3), np.int32)
        assert np.array_equal(np.asarray(xys)[sel].reshape(-1, 3), want), (w, h, len(xys), N)


def test_quadtree_cases_cover_every_class(quadtree_inputs):
    hit = {c: [] for c in XC.QUADTREE_CLASSES}
    for case, l, xys, w, h, N in quadtree_inputs:
        for c in XC.quadtree_classes(xys, w, h, N):
            hit[c].append((case, l))
    missing = [c for c, where in hit.items() if not where]
    assert not missing, missing
    assert len(set(XC.quadtree_cases())) == len(XC.quadtree_cases())


def test_threshold_cases_cover_every_class(oracle):
    names = XC.threshold_class_names()
    hit = {c: [] for c in names}
    for ini, mn, kind in XC.THRESHOLD_CASES:
        img, _ = XC.threshold_image(ini, mn, kind)
        P = oracle.PortExtractor(XC.THRESHOLD_NFEATURES, 1.2, 8, ini, mn)
        P(img)
        for c in XC.threshold_classes(ini, mn, kind, [tuple(r) for r in P.candidates(0).tolist()]):
            if c in hit:
                hit[c].append((ini, mn, kind))
    missing = [c for c, where in hit.items() if not where]
    assert not missing, missing
    required = [(0, 0), (1, 0), (20, 0), (126, 7), (127, 7), (128, 7), (128, 127), (129, 128), (200, 20), (255, 128),
                (254, 253), (255, 0), (255, 255), (7, 7)]
    assert set(required) <= set(XC.THRESHOLD_PAIRS)


def test_threshold_dots_have_their_scores(oracle):
    """Every dot of a dot image is either absent or a candidate with exactly its planned score; nothing else is."""
    for ini, mn, kind in XC.THRESHOLD_CASES:
        if kind == "noise":
            continue
        img, dots = XC.threshold_image(ini, mn, kind)
        P = oracle.PortExtractor(XC.THRESHOLD_NFEATURES, 1.2, 8, ini, mn)
        P(img)
        planned = {(x, y): s for x, y, s, _ in dots}
        for x, y, s in P.candidates(0).tolist():
            assert planned.get((x, y)) == s, (ini, mn, kind, x, y, s)


def test_fast_tiles_of_the_full_queue_sizes():
    """FULL_QUEUE_SIZES hold the widest (124 px) and the tallest (64 rows) FAST tile, and THRESHOLD_SIZE the largest one."""
    for size in XC.FULL_QUEUE_SIZES + [XC.THRESHOLD_SIZE]:
        assert size == XC.THRESHOLD_SIZE or size in XC.EG.SIZES
        tiles = XC.fast_tiles(*size)
        assert max(t[1] for t in tiles) == 124 and max(t[2] for t in tiles) == XC.FAST_H_BAND, size
    assert (0, 124, XC.FAST_H_BAND) in XC.fast_tiles(*XC.THRESHOLD_SIZE)


def test_level_cases_are_accepted():
    for nf, sf, nl in XC.LEVEL_CASES:
        assert XC.EG.accepted(*XC.LEVEL_SIZE, nfeatures=nf, scale_factor=sf, nlevels=nl), (nf, sf, nl)
    assert {nl for _, _, nl in XC.LEVEL_CASES} == {1, XC.MAX_LEVELS}
    assert {sf for _, sf, nl in XC.LEVEL_CASES if nl == XC.MAX_LEVELS} == {1.2, 1.1}


@pytest.mark.parametrize("case", XC.THRESHOLD_CASES, ids=TH_IDS)
def test_port_equals_verbatim_reference_at_thresholds(oracle_ref, case):
    ini, mn, kind = case
    img, _ = XC.threshold_image(ini, mn, kind)
    _assert_port_equals_reference(oracle_ref, img, XC.THRESHOLD_NFEATURES, 1.2, 8, ini, mn)


@pytest.mark.parametrize("case", XC.quadtree_cases(), ids=QT_IDS)
def test_port_equals_verbatim_reference_at_quota(oracle_ref, case):
    nf, nl = case
    img = XC.quadtree_image()
    kp = _assert_port_equals_reference(oracle_ref, img, nf, 1.2, nl)
    P = oracle_ref.PortExtractor(nf, 1.2, nl)
    P(img)
    for l, (xys, w, h, N) in enumerate(XC.level_inputs(P, nl)):
        sel, _ = XC.distribute(xys, w, h, N)
        assert int((kp["octave"] == l).sum()) == len(sel), l


@pytest.mark.parametrize("case", XC.LEVEL_CASES, ids=lambda c: f"{c[0]}-{c[1]}x{c[2]}")
def test_port_equals_verbatim_reference_at_level_count(oracle_ref, case):
    nf, sf, nl = case
    kp = _assert_port_equals_reference(oracle_ref, XC.level_image(), nf, sf, nl)
    assert set(kp["octave"].tolist()) == set(range(nl))
