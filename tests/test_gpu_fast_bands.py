"""FAST bands: each fast_kernel CTA detects a band of rowsPerBlk = max(1, min(FAST_H_BAND / hCell, nRows)) stacked cell rows.

The CPU tests restate the band table (build_geometry / build_fast_tiles in the library) and check that the benchmark
geometries and the sweep sizes reach every band class.  The GPU tests check that the band changes no result: per-level
FAST candidates, keypoints and descriptors equal the port on natural and white-noise frames, a corner on the last row of a
band's upper cell row survives a stronger corner right below it in the next cell row, and a cell row that falls back to
minThFAST sits in the same band as one that does not."""
import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests import extract_geometry as EG

FAST_H_BAND = 64
EDGE = EG.EDGE
BENCH = {"kitti": ((1242, 375), 2000), "tum": ((640, 480), 1000), "euroc": ((752, 480), 1200)}


def rows_per_blk(lv):
    return max(1, min(FAST_H_BAND // lv["hCell"], lv["nRows"]))


def bands(lv):
    """[(first cell row, cell rows, y0, y1)] of one level: y0..y1 is the band's detection domain (clipped at h - EDGE)."""
    r, out = rows_per_blk(lv), []
    for c in range(0, lv["nRows"], r):
        n = min(r, lv["nRows"] - c)
        y0 = EDGE + c * lv["hCell"]
        y1 = min(y0 + n * lv["hCell"], lv["h"] - EDGE)
        if y0 < y1:
            out.append((c, n, y0, y1))
    return out


BAND_CLASSES = {
    "R==1": lambda lv: rows_per_blk(lv) == 1,
    "R==2": lambda lv: rows_per_blk(lv) == 2,
    "last band shorter than R": lambda lv: bands(lv)[-1][1] < rows_per_blk(lv),
    "one-row cell grid": lambda lv: lv["nRows"] == 1,
}


def test_bench_band_table():
    """Cell rows per band, per level, of the benchmark geometries (the band table the kernel's grid is built from)."""
    want = {"kitti": [2, 2, 1, 2, 1, 1, 2, 1], "tum": [2, 2, 2, 2, 1, 1, 1, 1], "euroc": [2, 2, 2, 2, 1, 1, 1, 1]}
    for name, (size, nf) in BENCH.items():
        levels, refusal = EG.geometry(*size, nfeatures=nf)
        assert refusal is None
        assert [rows_per_blk(lv) for lv in levels] == want[name], name
        for lv in levels:
            b = bands(lv)
            assert b[0][0] == 0 and sum(n for _, n, _, _ in b) == lv["nRows"]
            assert all(y1 - y0 <= max(FAST_H_BAND, lv["hCell"]) for _, _, y0, y1 in b)


def test_band_classes_are_covered():
    sizes = [s for s, _ in BENCH.values()] + EG.SIZES
    hit = {c: [] for c in BAND_CLASSES}
    for s in sizes:
        levels, refusal = EG.geometry(*s)
        assert refusal is None
        for c, pred in BAND_CLASSES.items():
            if any(pred(lv) for lv in levels):
                hit[c].append(s)
    assert all(hit.values()), {c: v for c, v in hit.items() if not v}
    assert (221, 221) in hit["one-row cell grid"] and (221, 221) in hit["R==1"]
    assert all(rows_per_blk(lv) <= 2 for s in sizes for lv in EG.geometry(*s)[0])   # hCell >= 30: no 3-row band at 64


# ---------------------------------------------------------------------------------------------------------------------
# GPU

@pytest.fixture(scope="module")
def X():
    from orb_slam2_b200.extractor import ORBextractor
    return ORBextractor


def _cands(G, l):
    return sorted(map(tuple, G.debug_candidates(l).tolist()))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["natural", "noise"])
@pytest.mark.parametrize("case", ["kitti", "tum", "euroc", "221x221"])
def test_bands_match_port(X, oracle, case, kind):
    from tests.test_gpu_extract_geometry import assert_stages_equal
    (w, h), nf = BENCH.get(case, ((221, 221), 1000))
    img = synth.mono_frame(31, 0, 0, w, h) if kind == "natural" else synth.white_noise(32, w, h)
    G, P = X(nf), oracle.PortExtractor(nf)
    kg, dg = G(img)
    kp, dp = P(img)
    assert_stages_equal(G, P, kg, dg, kp, dp)


def _level0(size, nf):
    levels, refusal = EG.geometry(*size, nfeatures=nf)
    assert refusal is None
    return levels[0]


@pytest.mark.gpu
def test_corner_above_cell_row_border_is_kept(X, oracle):
    """Dots on the last row of each inner cell row of a level-0 band, each with a stronger dot directly below it in the next
    cell row: the cell-local NMS counts a neighbour in another cell row as 0, so both dots are kept."""
    (w, h), nf = BENCH["kitti"]
    lv = _level0((w, h), nf)
    R, hc = rows_per_blk(lv), lv["hCell"]
    assert R == 2
    img = np.full((h, w), EG.DOT_BACKGROUND, np.uint8)
    pairs = []
    for c0, n, _, _ in bands(lv):
        for c in range(c0, c0 + n - 1):                       # borders between two cell rows of the same band
            y = EDGE + (c + 1) * hc - 1
            for x in range(EDGE + 10, w - EDGE - 10, 47):
                img[y, x], img[y + 1, x] = 150, 250
                pairs.append((x, y))
    assert len(pairs) > 50
    G, P = X(nf), oracle.PortExtractor(nf)
    kg, dg = G(img)
    kp, dp = P(img)
    got = _cands(G, 0)
    assert got == sorted(map(tuple, P.candidates(0).tolist()))
    pts = {(x, y) for x, y, _ in got}
    for x, y in pairs:
        assert (x, y) in pts and (x, y + 1) in pts, (x, y)
    from tests.test_gpu_extract import assert_kps_equal
    assert_kps_equal(kg, dg, kp, dp)


@pytest.mark.gpu
def test_pass_b_in_one_cell_row_of_a_band(X, oracle):
    """First level-0 band (2 cell rows): the top cell row has a strong corner (S >= iniThFAST) in every cell, the bottom one
    only weak corners (minThFAST <= S < iniThFAST).  Only the bottom cell row falls back to minThFAST: its weak corners are
    found, the weak corners placed next to strong ones in the top row are not."""
    (w, h), nf = BENCH["kitti"]
    lv = _level0((w, h), nf)
    hc, wc = lv["hCell"], lv["wCell"]
    assert bands(lv)[0][1] == 2
    bg, weak, strong = 90, 105, 200                           # S = 14 (between minTh 7 and iniTh 20) and S = 109
    img = np.full((h, w), bg, np.uint8)
    top_weak, low_weak = [], []
    for cx in range(lv["nCols"]):
        x = EDGE + cx * wc + 8
        if x + 12 >= w - EDGE:
            break
        img[EDGE + 10, x] = strong
        img[EDGE + 20, x + 10] = weak
        top_weak.append((x + 10, EDGE + 20))
        img[EDGE + hc + 12, x + 5] = weak
        low_weak.append((x + 5, EDGE + hc + 12))
    G, P = X(nf), oracle.PortExtractor(nf)
    kg, dg = G(img)
    kp, dp = P(img)
    got = _cands(G, 0)
    assert got == sorted(map(tuple, P.candidates(0).tolist()))
    pts = {(x, y) for x, y, _ in got}
    assert all(p in pts for p in low_weak)
    assert not any(p in pts for p in top_weak)
    from tests.test_gpu_extract import assert_kps_equal
    assert_kps_equal(kg, dg, kp, dp)
