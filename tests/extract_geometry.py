"""Python restatement of the extractor's per-level geometry (build_geometry in orb_slam2_b200/csrc/borb_host.cu), used
only by the tests: which sizes reach which tiling path of the extraction kernels, and which sizes and quotas the library
refuses.  Float arithmetic is done in float32 op by op, as the C++ does it.

Also the fixed list of image sizes the geometry tests sweep (SIZES), chosen offline with coverage() so that every edge
class below is hit by construction rather than by whatever rounding a natural frame size gives, and the synthetic images
that put an exact candidate count on level 0.
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32

MIN_BORDER = 16        # EDGE_THRESHOLD - 3
EDGE = 19              # EDGE_THRESHOLD
FAST_TILE_W = 124      # widest detection domain of one FAST CTA
BLUR_TILE_W = 120      # blur strip width
QT_ONCHIP = 5120       # candidates per level the quadtree kernel keeps in registers
QT_SMEM_LIMIT = 200 * 1024
MAX_DIM = 4095


def _lrintf(v) -> int:
    return int(np.rint(f32(v)))          # cvRound / lrintf: round half to even


def _align_up(v: int, a: int) -> int:
    return (v + a - 1) // a * a


def scale_tables(nfeatures: int, scale_factor: float = 1.2, nlevels: int = 8):
    """(scale, inv_scale, per_level quota) exactly as init_tables derives them (double chain rounded to float per level)."""
    sf = float(f32(scale_factor))
    scale = [f32(1.0)] * nlevels
    for i in range(1, nlevels):
        scale[i] = f32(float(scale[i - 1]) * sf)
    inv_scale = [f32(1.0) / s for s in scale]
    factor = f32(1.0 / sf)
    want = f32(nfeatures) * (f32(1.0) - factor) / (f32(1.0) - f32(math.pow(float(factor), float(nlevels))))
    per_level, total = [], 0
    for _ in range(nlevels - 1):
        q = _lrintf(want)
        per_level.append(q)
        total += q
        want = f32(want * factor)
    per_level.append(max(nfeatures - total, 0))
    return scale, inv_scale, per_level


def quadtree_smem_bytes(node_cap: int) -> int:
    return node_cap * 84 + 4 + 35 * 4


def x_windowed(src: int, dst: int) -> bool:
    """Whether level dst (resized from a level of width src) takes the table-driven pyr_resize_kernel: every group of 4
    destination columns, padding columns included, reads inside one aligned 12-byte source window (resize_table and
    resize_window_table).  False: pyr_resize_generic_kernel."""
    scale = 1.0 / (dst / src)
    ofs = []
    for d in range(dst):
        s = math.floor(f32((d + 0.5) * scale - 0.5))
        ofs.append(min(max(s, 0), src - 1))
    wpad = (dst + 8 + 3) & ~3
    ofs += [ofs[max(dst - 2 - k, 0)] for k in range(wpad - dst)]    # reflect-101 padding columns
    return all(max(ofs[g:g + 4]) + 1 - (min(ofs[g:g + 4]) & ~3) <= 11 for g in range(0, wpad, 4))


def geometry(w: int, h: int, nfeatures: int = 1000, scale_factor: float = 1.2, nlevels: int = 8):
    """-> (levels, refusal).  levels: one dict per level built so far; refusal: None if the library accepts the size and
    quota, else the reason it returns BORB_ERR_UNSUPPORTED."""
    if not (1 <= w <= MAX_DIM and 1 <= h <= MAX_DIM):
        return [], "image size"
    _, inv_scale, quota = scale_tables(nfeatures, scale_factor, nlevels)
    levels, sel = [], 0
    for l in range(nlevels):
        lw, lh = _lrintf(f32(w) * inv_scale[l]), _lrintf(f32(h) * inv_scale[l])
        width, height = f32(lw - 2 * MIN_BORDER), f32(lh - 2 * MIN_BORDER)
        n_cols, n_rows = int(width / f32(30)), int(height / f32(30))
        if n_cols < 1 or n_rows < 1:
            return levels, f"level {l} has no FAST cell"
        w_cell, h_cell = math.ceil(width / f32(n_cols)), math.ceil(height / f32(n_rows))
        n_ini = int(math.floor(float(width / height) + 0.5))      # std::round of a positive float
        if n_ini < 1:
            return levels, f"level {l} has no quadtree root"
        node_cap = _align_up(max(quota[l], 4 * n_ini) + 3 + 1, 4)
        lv = dict(w=lw, h=lh, nCols=n_cols, nRows=n_rows, wCell=w_cell, hCell=h_cell,
                  cellsPerBlk=max(FAST_TILE_W // w_cell, 1), pitch=_align_up(lw + 8, 128), quota=quota[l], nIni=n_ini,
                  node_cap=node_cap, smem=quadtree_smem_bytes(node_cap),
                  x_windowed=None if l == 0 else x_windowed(levels[-1]["w"], lw))
        levels.append(lv)
        sel += node_cap
        if lv["smem"] > QT_SMEM_LIMIT:
            return levels, f"level {l} quota exceeds the quadtree shared-memory envelope"
    if sel >= 65536:
        return levels, "keypoint capacity"
    return levels, None


def accepted(w, h, **kw) -> bool:
    return geometry(w, h, **kw)[1] is None


def level_shapes(w, h, **kw):
    levels, refusal = geometry(w, h, **kw)
    assert refusal is None, refusal
    return [(lv["h"], lv["w"]) for lv in levels]


def largest_nfeatures(w, h, scale_factor=1.2, nlevels=8):
    """Largest nfeatures the library accepts at this size (offline helper; the tests commit the result)."""
    lo, hi = 1, 1
    while accepted(w, h, nfeatures=hi, scale_factor=scale_factor, nlevels=nlevels):
        lo, hi = hi, hi * 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if accepted(w, h, nfeatures=mid, scale_factor=scale_factor, nlevels=nlevels):
            lo = mid
        else:
            hi = mid
    return lo


def smallest_side(scale_factor=1.2, nlevels=8, other=480):
    """Smallest accepted width (with height `other`) at the default quota (offline helper)."""
    return next(v for v in range(1, MAX_DIM + 1) if accepted(v, other, scale_factor=scale_factor, nlevels=nlevels))


# Edge classes of the kernels' tiling, as predicates over one level's geometry.
LEVEL_CLASSES = {
    "w%4==0": lambda lv: lv["w"] % 4 == 0,                       # pyramid / blur rows end on, or inside, an aligned word
    "w%4==1": lambda lv: lv["w"] % 4 == 1,
    "w%4==2": lambda lv: lv["w"] % 4 == 2,
    "w%4==3": lambda lv: lv["w"] % 4 == 3,
    "tight pitch": lambda lv: (lv["w"] + 8) % 128 == 0,            # exactly 8 bytes of padding, no slack
    "w%120==0": lambda lv: lv["w"] % BLUR_TILE_W == 0,             # the last blur strip is full
    "w%120==1": lambda lv: lv["w"] % BLUR_TILE_W == 1,             # the last blur strip holds one pixel
    "w%120==119": lambda lv: lv["w"] % BLUR_TILE_W == 119,
    "nCols==1": lambda lv: lv["nCols"] == 1,
    "nRows==1": lambda lv: lv["nRows"] == 1,
    "wCell==31": lambda lv: lv["wCell"] == 31,                    # 4 cells of 31 fill the FAST tile exactly
    "wCell==41": lambda lv: lv["wCell"] == 41,                    # widest cell at 3 cells per CTA
    "wCell==42": lambda lv: lv["wCell"] == 42,                    # narrowest cell at 2 cells per CTA
    "wCell==59": lambda lv: lv["wCell"] == 59,                    # widest cell there is
    "cellsPerBlk==2": lambda lv: lv["cellsPerBlk"] == 2,
    "cellsPerBlk==3": lambda lv: lv["cellsPerBlk"] == 3,
    "cellsPerBlk==4": lambda lv: lv["cellsPerBlk"] == 4,
}
# "level-0 tight pitch": pad_level0_kernel's 8-byte write ends on the last byte of the row (the other levels' padding
# comes from the resize kernels)
SIZE_CLASSES = ("smallest width", "smallest height", "level-0 tight pitch")


def coverage(sizes, nfeatures=1000, scale_factor=1.2, nlevels=8):
    """{class: [sizes that hit it]} for every class of LEVEL_CLASSES and SIZE_CLASSES (a class no size hits maps to [])."""
    out = {c: [] for c in list(LEVEL_CLASSES) + list(SIZE_CLASSES)}
    kw = dict(nfeatures=nfeatures, scale_factor=scale_factor, nlevels=nlevels)
    for (w, h) in sizes:
        levels, refusal = geometry(w, h, **kw)
        assert refusal is None, ((w, h), refusal)
        for c, pred in LEVEL_CLASSES.items():
            if any(pred(lv) for lv in levels):
                out[c].append((w, h))
        if not accepted(w - 1, h, **kw):
            out["smallest width"].append((w, h))
        if not accepted(w, h - 1, **kw):
            out["smallest height"].append((w, h))
        if levels[0]["pitch"] == levels[0]["w"] + 8:
            out["level-0 tight pitch"].append((w, h))
    return out


# Chosen offline with coverage() (1000 features, scale 1.2, 8 levels); every class above is hit at least once.
SIZES = [
    (221, 221), (221, 300), (327, 240), (376, 240), (390, 480), (410, 240), (417, 480), (431, 240),
    (489, 240), (540, 480), (588, 480), (634, 480), (640, 221), (641, 480), (681, 375), (693, 240),
    (723, 480), (755, 240), (1006, 240), (1087, 375), (1107, 375), (1180, 240), (1195, 240), (1283, 240),
]


# ---------------------------------------------------------------------------------------------------------------------
# Level-0 images with an exact FAST candidate count: isolated single-pixel dots on a flat background, at least 7 px apart
# (a dot is the only corner within its ring, so no two dots interact), in three intensities so that responses tie and
# the quadtree's emission-order tie-break decides.  `n` dots are drawn from a 7-px lattice over the detection domain.
DOT_BACKGROUND = 90
DOT_LEVELS = (150, 200, 250)


def dot_image(n, w, h, seed):
    rng = np.random.default_rng(seed)
    img = np.full((h, w), DOT_BACKGROUND, np.uint8)
    xs = np.arange(EDGE + 2, w - EDGE - 2, 7)
    ys = np.arange(EDGE + 2, h - EDGE - 2, 7)
    assert n <= len(xs) * len(ys), (n, len(xs) * len(ys))
    pick = rng.choice(len(xs) * len(ys), size=n, replace=False)
    img[ys[pick // len(xs)], xs[pick % len(xs)]] = rng.choice(DOT_LEVELS, size=n)
    return img


# Quadtree on-chip boundary images: (target level-0 candidate count, dots, frame size, seed); one dot gives one candidate.
# The register path holds 5120 candidates.  They run at DOT_NFEATURES, whose level-0 quota (2432) is the largest the node
# capacity allows: about two candidates per selected node, so losing any one candidate changes the level-0 selection about
# three times in four.  Eight 5121-candidate layouts make a dropped candidate practically certain to show.
DOT_NFEATURES = 11200
DOT_CASES = ([(5119, 5119, (1242, 375), 1), (5120, 5120, (1242, 375), 1)]
             + [(5121, 5121, (1242, 375), seed) for seed in range(1, 9)]
             + [(10300, 10300, (1280, 720), 3)])

# (scale factor, levels, largest accepted nfeatures) on a KITTI-sized 1242x375 frame; one more feature is refused.  At 1.2 x 8
# every level takes the table-driven pyr_resize_kernel; at 3.0 x 2 level 1 takes pyr_resize_generic_kernel.
ENVELOPE = [(1.2, 8, 11200), (3.0, 2, 3243)]
