"""The extractor's configuration domain as test cases: FAST thresholds across 0..255, per-level quotas down to zero, and 1 to
BORB_MAX_LEVELS pyramid levels.  Test tooling only: tests/test_oracle_extract_config.py pins the port to the verbatim
ORBextractor.cc on every case, tests/test_gpu_extract_config.py pins the CUDA library to the port.

Every case list below was chosen offline with the coverage functions here, from named edge classes of the kernels; the
tests assert that the committed lists still reach every class.  Nothing in this module calls the CUDA library.

Thresholds.  A single pixel of contrast c on a flat background is the only FAST corner within its ring, with score exactly
S = c - 1, so images of such dots put an exact score next to every threshold: at t the dot with S = t is a corner and the
dot with S = t - 1 is not.  fast_kernel's packed reject is only valid for t <= 127 (k_fast.cu gt_flag), so above that
every domain pixel is queued and scored; a cell with no kept corner at iniThFAST is redone at minThFAST (pass B).

Quadtree.  distribute() restates DistributeOctTree's control flow (ORBextractor.cc:539-763) and records which branches a
(candidate set, N) takes; quadtree_kernel implements the same branches (k_quadtree.cu:263, 275, 284).
"""
from __future__ import annotations

import math

import numpy as np

from orb_slam2_b200 import synth
from tests import extract_geometry as EG

f32 = np.float32
EDGE, MIN_BORDER = EG.EDGE, EG.MIN_BORDER
MAX_LEVELS = 16                                         # BORB_MAX_LEVELS (include/borb.h)
FAST_H_BAND = 64                                        # borb_internal.h: detection-domain rows of the tallest FAST tile

# ---------------------------------------------------------------------------------------------------------------------
# FAST thresholds

# (iniThFAST, minThFAST).  0, 127/128 and 255 are the reject's constant boundaries (K = (127 - min(t, 127)) * 0x01010101,
# reject only for t <= 127, tc = max(t, 1)); min >= ini never runs pass B.
THRESHOLD_PAIRS = [(0, 0), (1, 0), (20, 0), (126, 7), (127, 7), (128, 7), (128, 127), (129, 128), (200, 20), (255, 128),
                   (254, 253), (255, 0), (255, 255), (7, 7), (127, 128)]
THRESHOLD_KINDS = ("bright", "dark", "noise")
THRESHOLD_SIZE = (640, 480)           # level 0: 20 x 14 cells of 31 x 32, FAST tiles of 124 x 64 (the largest there are)
THRESHOLD_NFEATURES = 1000


def level0_cells(w, h):
    """[(cell row, cell col, x0, x1, y0, y1)] of level 0: each cell's FAST detection domain (ORBextractor.cc:789-806)."""
    lv = EG.geometry(w, h)[0][0]
    out = []
    for r in range(lv["nRows"]):
        for c in range(lv["nCols"]):
            x0, y0 = EDGE + c * lv["wCell"], EDGE + r * lv["hCell"]
            x1, y1 = min(x0 + lv["wCell"], w - EDGE), min(y0 + lv["hCell"], h - EDGE)
            if x0 < x1 and y0 < y1:
                out.append((r, c, x0, x1, y0, y1))
    return out


def _kept_score(t):
    """Smallest score a threshold t keeps: S >= t, and a kept corner has S > 0 (strict NMS against non-corners' 0)."""
    return max(t, 1)


def threshold_dots(ini, mn, bright, w=THRESHOLD_SIZE[0], h=THRESHOLD_SIZE[1], seed=0):
    """-> (image, dots).  Flat background (0 under bright dots, 255 under dark ones) and single-pixel dots of exact score,
    7 px apart, on a 4 x 4 lattice per level-0 cell.  Cells take three roles in turn:
      "A": a dot of S = max(ini,1) (kept at ini) and one of S = max(ini,1) - 1 (not), one of S = 254, and random scores;
      "B": nothing >= ini, so the cell runs pass B: a dot of S = max(min,1) and one of S = max(min,1) - 1, random scores < ini;
      "-": empty.
    A role that cannot exist for this pair (no S >= 255 for "A" at ini = 255; no pass B unless min < ini) is replaced by
    the other one.  dots: [(x, y, S, cell index)]."""
    rng = np.random.default_rng(seed * 1000 + ini * 7 + mn)
    bg = 0 if bright else 255
    img = np.full((h, w), bg, np.uint8)
    dots = []
    can_a, can_b = _kept_score(ini) <= 254, mn < ini
    for ci, (r, c, x0, x1, y0, y1) in enumerate(level0_cells(w, h)):
        role = "AB-"[(r + 2 * c) % 3]
        if role == "A" and not can_a:
            role = "B" if can_b else "A"
        if role == "B" and not can_b:
            role = "A"
        if role == "-":
            continue
        if role == "A":
            k = _kept_score(ini)
            fixed = ([k] if k <= 254 else []) + [k - 1, 254]
            rand = lambda: int(rng.integers(0, 255))
        else:
            k = _kept_score(mn)
            fixed = [s for s in (k, k - 1) if s < ini]
            rand = lambda: int(rng.integers(0, ini))
        slots = [(x0 + 3 + 7 * i, y0 + 3 + 7 * j) for j in range(4) for i in range(4) if x0 + 3 + 7 * i < x1 and y0 + 3 + 7 * j < y1]
        rng.shuffle(slots)
        for n, (x, y) in enumerate(slots):
            if n < len(fixed):
                s = fixed[n]
            elif rng.random() < 0.5:
                s = rand()
            else:
                continue
            img[y, x] = bg + (s + 1) if bright else bg - (s + 1)
            dots.append((x, y, s, ci))
    return img, dots


def threshold_image(ini, mn, kind, w=THRESHOLD_SIZE[0], h=THRESHOLD_SIZE[1]):
    """-> (image, dots or None) of one threshold case."""
    if kind == "noise":
        return synth.white_noise(31, w, h), None
    return threshold_dots(ini, mn, kind == "bright", w, h)


THRESHOLD_CASES = [(ini, mn, kind) for (ini, mn) in THRESHOLD_PAIRS for kind in THRESHOLD_KINDS]


def threshold_class_names(pairs=THRESHOLD_PAIRS):
    named = ["pass A t=0", "pass B t=0", "pass A t=127", "pass B t=127", "pass A t=128", "pass B t=128",
             "reject off in pass A", "reject off in pass B", "every level-0 cell in pass B", "ini == min", "ini < min",
             "S=254 emitted", "dense: pass A queues every domain pixel"]
    for ini, mn in pairs:
        for p, t in [("A", ini)] + ([("B", mn)] if mn < ini else []):
            k = _kept_score(t)
            if k <= 254 and (p == "A" or k < ini):      # a pass-B cell holds nothing >= ini
                named.append(f"pass {p} t={t}: S={k} kept")
            named.append(f"pass {p} t={t}: S={k - 1} absent")
    return list(dict.fromkeys(named))


def threshold_classes(ini, mn, kind, cands, w=THRESHOLD_SIZE[0], h=THRESHOLD_SIZE[1]):
    """Classes one case reaches, judged from its level-0 candidates [(x, y, S)] (the port's)."""
    cells = level0_cells(w, h)
    lv = EG.geometry(w, h)[0][0]
    cell_of = lambda x, y: ((y - EDGE) // lv["hCell"]) * lv["nCols"] + (x - EDGE) // lv["wCell"]
    index = {(r * lv["nCols"] + c): i for i, (r, c, *_) in enumerate(cells)}
    per_cell = [[] for _ in cells]
    for x, y, s in cands:
        per_cell[index[cell_of(x, y)]].append(s)
    hit = set()
    pass_a = [i for i, ss in enumerate(per_cell) if any(s >= ini for s in ss)]
    pass_b = [i for i, ss in enumerate(per_cell) if mn < ini and not any(s >= ini for s in ss)]
    b_emitted = [i for i in pass_b if per_cell[i]]
    if pass_a:
        hit.add(f"pass A t={ini}")
        if ini > 127:
            hit.add("reject off in pass A")
        if ini > 127 and kind == "noise":
            hit.add("dense: pass A queues every domain pixel")
    if b_emitted:
        hit.add(f"pass B t={mn}")
        if mn > 127:
            hit.add("reject off in pass B")
    if len(b_emitted) == len(cells):
        hit.add("every level-0 cell in pass B")
    if cands:
        if ini == mn:
            hit.add("ini == min")
        if ini < mn:
            hit.add("ini < min")
        if any(s == 254 for _, _, s in cands):
            hit.add("S=254 emitted")
    if kind != "noise":
        _, dots = threshold_dots(ini, mn, kind == "bright", w, h)
        have = {(x, y, s) for x, y, s in cands}
        at = {(x, y) for x, y, _ in cands}
        # a cell ends in pass A if it keeps a corner at ini, or if there is no pass B (min >= ini)
        a_set, b_set = set(pass_a) if mn < ini else set(range(len(cells))), set(pass_b)
        for p, t, cellset in (("A", ini, a_set), ("B", mn, b_set)):
            if p == "B" and not mn < ini:
                continue
            k = _kept_score(t)
            for x, y, s, ci in dots:
                if ci not in cellset:
                    continue
                if s == k and (x, y, s) in have:
                    hit.add(f"pass {p} t={t}: S={k} kept")
                if s == k - 1 and (x, y) not in at:
                    hit.add(f"pass {p} t={t}: S={k - 1} absent")
    return hit


# ---------------------------------------------------------------------------------------------------------------------
# DistributeOctTree

class _Node:
    __slots__ = ("x0", "x1", "y0", "y1", "pts", "no_more", "birth")

    def __init__(self, x0, x1, y0, y1, pts, birth):
        self.x0, self.x1, self.y0, self.y1, self.pts, self.birth = x0, x1, y0, y1, pts, birth
        self.no_more = len(pts) == 1


def _round_half_away(v):
    return int(math.floor(v + 0.5)) if v >= 0 else -int(math.floor(-v + 0.5))


def distribute(xys, width, height, N):
    """DistributeOctTree (ORBextractor.cc:539-763) on candidates xys [(x, y, score)] relative to the minimum border, in
    emission order.  -> (indices of the selected candidates in list order, trace).  trace: one dict per pass with its
    phase, the list size before (n) and after (nn), nToExpand, whether a phase-2 pass stopped before its last expandable
    node (cut), and whether the pass finished the distribution.  The list is a Python list with index 0 at the front;
    `birth` orders nodes by creation, which is the order of their addresses in the reference (its sort key after size)."""
    xys = [tuple(int(v) for v in p) for p in xys]
    trace = []
    if not xys:
        return [], trace
    n_ini = _round_half_away(float(f32(width) / f32(height)))
    hx = f32(width) / f32(n_ini)
    births = iter(range(1 << 30))
    roots = [_Node(int(hx * f32(i)), int(hx * f32(i + 1)), 0, height, [], next(births)) for i in range(n_ini)]
    for i, (x, _, _) in enumerate(xys):
        roots[int(f32(x) / hx)].pts.append(i)
    nodes = [r for r in roots if r.pts]
    for r in nodes:
        r.no_more = len(r.pts) == 1

    def divide(nd):
        half_x = math.ceil(float(f32(nd.x1 - nd.x0) / f32(2)))
        half_y = math.ceil(float(f32(nd.y1 - nd.y0) / f32(2)))
        mx, my = nd.x0 + half_x, nd.y0 + half_y
        q = [[], [], [], []]
        for i in nd.pts:
            x, y, _ = xys[i]
            q[(0 if y < my else 2) if x < mx else (1 if y < my else 3)].append(i)
        boxes = [(nd.x0, mx, nd.y0, my), (mx, nd.x1, nd.y0, my), (nd.x0, mx, my, nd.y1), (mx, nd.x1, my, nd.y1)]
        return [_Node(*boxes[k], q[k], next(births)) for k in range(4) if q[k]]

    finish = False
    while not finish:
        prev = len(nodes)
        created, kept, expand = [], [], []
        for nd in nodes:
            if nd.no_more:
                kept.append(nd)
                continue
            for ch in divide(nd):
                created.append(ch)
                if len(ch.pts) > 1:
                    expand.append(ch)
        nodes = created[::-1] + kept
        rec = dict(phase=1, n=prev, nn=len(nodes), nToExpand=len(expand), cut=False, finish=False)
        trace.append(rec)
        if len(nodes) >= N or len(nodes) == prev:
            rec["finish"] = finish = True
        elif len(nodes) + 3 * len(expand) > N:
            while not finish:
                prev = len(nodes)
                order = sorted(expand, key=lambda nd: (len(nd.pts), nd.birth))[::-1]
                expand, created, done = [], [], set()
                for nd in order:
                    chs = divide(nd)
                    for ch in chs:
                        created.append(ch)
                        if len(ch.pts) > 1:
                            expand.append(ch)
                    done.add(id(nd))
                    if prev - len(done) + len(created) >= N:
                        break
                nodes = created[::-1] + [nd for nd in nodes if id(nd) not in done]
                rec = dict(phase=2, n=prev, nn=len(nodes), nToExpand=len(expand), cut=len(done) < len(order), finish=False)
                trace.append(rec)
                if len(nodes) >= N or len(nodes) == prev:
                    rec["finish"] = finish = True
    sel = []
    for nd in nodes:
        best = nd.pts[0]
        for i in nd.pts[1:]:
            if xys[i][2] > xys[best][2]:
                best = i
        sel.append(best)
    return sel, trace


QUADTREE_CLASSES = ("quota 0", "quota 1", "N below occupied roots", "first pass finishes with nn == N",
                    "first pass finishes with nn > N", "phase 1 finishes on nn == n < N", "two or more phase-1 passes",
                    "phase-1 pass continues with nn + 3 * nToExpand == N", "phase-2 cut with nn == N",
                    "phase-2 cut with nn == N+1", "phase-2 cut with nn == N+2", "phase 2 finishes on nn == n")
# A phase-2 cut overshoots by at most 2: the list holds at most N - 1 nodes before the divide that reaches N, and one divide
# adds at most 3.  Only a first pass overshoots further.


def quadtree_classes(xys, width, height, N):
    """Classes of QUADTREE_CLASSES one (candidate set, N) reaches."""
    if len(xys) == 0:
        return set()
    _, trace = distribute(xys, width, height, N)
    hit = set()
    if N == 0:
        hit.add("quota 0")
    if N == 1:
        hit.add("quota 1")
    hx = f32(width) / f32(_round_half_away(float(f32(width) / f32(height))))
    roots = len({int(f32(int(x)) / hx) for x, _, _ in xys})
    if 1 <= N < roots:
        hit.add("N below occupied roots")
    first = trace[0]
    if first["finish"] and first["nn"] != first["n"]:
        hit.add("first pass finishes with nn == N" if first["nn"] == N else "first pass finishes with nn > N")
    p1 = [r for r in trace if r["phase"] == 1]
    if len(p1) >= 2:
        hit.add("two or more phase-1 passes")
    for r in trace:
        if r["phase"] == 1 and r["finish"] and r["nn"] == r["n"] and r["nn"] < N:
            hit.add("phase 1 finishes on nn == n < N")
        if r["phase"] == 1 and not r["finish"] and r["nn"] + 3 * r["nToExpand"] == N:
            hit.add("phase-1 pass continues with nn + 3 * nToExpand == N")
        if r["phase"] == 2 and r["cut"] and 0 <= r["nn"] - N <= 2:
            hit.add("phase-2 cut with nn == N" + (f"+{r['nn'] - N}" if r["nn"] > N else ""))
        if r["phase"] == 2 and r["finish"] and r["nn"] == r["n"]:
            hit.add("phase 2 finishes on nn == n")
    return hit


def level_inputs(P, nlevels):
    """[(candidates relative to the minimum border, width, height, quota)] of every level of the port's last call."""
    out = []
    for l in range(nlevels):
        lh, lw = P.level(l).shape
        c = P.candidates(l).astype(np.int64)
        rel = np.stack([c[:, 0] - MIN_BORDER, c[:, 1] - MIN_BORDER, c[:, 2]], 1) if len(c) else np.zeros((0, 3), np.int64)
        out.append((rel, lw - 2 * MIN_BORDER, lh - 2 * MIN_BORDER, int(P.per_level[l])))
    return out


# Quadtree cases: (nfeatures, nlevels) on one KITTI-sized dot image (EG.dot_image: one candidate per dot, four quadtree roots
# at level 0).  With one level the level-0 quota is nfeatures itself, so N is swept directly; at 8 levels and nfeatures
# 1-20 the upper levels get quotas of 0 and 1.
QT_SIZE = synth.KITTI
QT_DOTS, QT_SEED = 300, 5
QT_N_SINGLE = [1, 2, 3, 5, 16, 17, 18, 19, 41, 42, 43, 64, 150, 252, 299, 300, 301, 396, 399]
QT_N_EIGHT = list(range(1, 21))


def quadtree_image():
    return EG.dot_image(QT_DOTS, *QT_SIZE, QT_SEED)


def quadtree_cases():
    return [(n, 1) for n in QT_N_SINGLE] + [(n, 8) for n in QT_N_EIGHT]


# ---------------------------------------------------------------------------------------------------------------------
# Level counts: (nfeatures, scale factor, nlevels) on a 2000 x 1500 frame.  One level: the pyramid loop is empty.  Sixteen
# (BORB_MAX_LEVELS): the largest Geometry and TMaps kernel parameters.
LEVEL_SIZE = (2000, 1500)
LEVEL_CASES = [(2000, 1.2, 1), (3000, 1.2, MAX_LEVELS), (2000, 1.1, MAX_LEVELS)]


def level_image():
    return synth.mono_frame(41, 0, 0, *LEVEL_SIZE)


# ---------------------------------------------------------------------------------------------------------------------
# FAST tiles (build_fast_tiles in k_fast.cu): the detection domain of one CTA.

def fast_tiles(w, h, **kw):
    """[(level, width, height)] of every FAST tile of a frame."""
    levels, refusal = EG.geometry(w, h, **kw)
    assert refusal is None, refusal
    out = []
    for l, lv in enumerate(levels):
        rows = max(1, min(FAST_H_BAND // lv["hCell"], lv["nRows"]))
        for r0 in range(0, lv["nRows"], rows):
            for c0 in range(0, lv["nCols"], lv["cellsPerBlk"]):
                x0, y0 = EDGE + c0 * lv["wCell"], EDGE + r0 * lv["hCell"]
                x1 = min(x0 + min(lv["cellsPerBlk"], lv["nCols"] - c0) * lv["wCell"], lv["w"] - EDGE)
                y1 = min(y0 + min(rows, lv["nRows"] - r0) * lv["hCell"], lv["h"] - EDGE)
                if x0 < x1 and y0 < y1:
                    out.append((l, x1 - x0, y1 - y0))
    return out


# Sizes of EG.SIZES whose FAST tiles include the widest (124 px) and the tallest (64 rows) one, run at thresholds where
# every domain pixel is queued (chosen offline with fast_tiles).
FULL_QUEUE_SIZES = [(221, 300), (641, 480), (1107, 375)]
FULL_QUEUE_PAIRS = [(200, 7), (255, 0)]
