"""Stereo association inputs at the edges where k_stereo.cu (Frame::ComputeStereoMatches, reference src/Frame.cc:466-640) takes
its branches, and a coverage report of which branches a case reaches.  Test tooling: tests/test_oracle_stereo_envelope.py pins
the port (oracle/orb_port_stereo.cpp) to the verbatim Frame.cc on every case, tests/test_gpu_stereo_envelope.py pins the CUDA
library to the port through every stereo entry point.

The kernel constants are restated next to the line each comes from, and stage 1 (row band, octave window, u-range, best
Hamming) and the SAD refinement and median cull are restated in plain numpy, only to classify what a case reaches.  Nothing in
this module calls the CUDA library.

A class counts only where its effect reaches mvuRight / mvDepth (see restate): a branch whose result the median cull throws
away is not covered, because no comparison of the outputs could see it go wrong.

Each case is a pair of images, the extractor settings (nfeatures, scaleFactor, nlevels) of the left and the right handle, and
(bf, fx).  The settings and sizes were checked against extract_geometry.geometry, and the crafted images chosen offline, so that
every class of CLASSES is reached by construction.  Classes the code has but real extraction cannot reach are listed in
UNREACHABLE with the reason.
"""
import functools
import math

import numpy as np

from orb_slam2_b200 import synth
from tests import extract_geometry as G

f32 = np.float32

SBIN_SHIFT = 3             # k_stereo.cu:26 — 8 image rows per bin
SBIN_MAX = 512             # k_stereo.cu:27 — bins per pair (images up to 4096 rows)
IR_BITS = 16               # k_stereo.cu:144 — key = dist << 16 | iR: right keypoint indices below 2^16
TH_HIGH, TH_LOW = 100, 50  # ORBmatcher.cc:52-53, k_stereo.cu:129
TH_ORB = (TH_HIGH + TH_LOW) // 2   # k_stereo.cu:152 — thOrbDist = 75 (Frame.cc:471)
W = LH = 5                 # k_stereo.cu:161 — 11x11 SAD window, shifts -5..5 (Frame.cc:565,573)
HIST_BINS = 256            # k_stereo.cu:231-271 — two 256-bin passes: SAD >> 8, then SAD & 255
KITTI_CAM = (386.1448, 718.856)    # Examples/Stereo/KITTI00-02.yaml Camera.bf / Camera.fx
VGA_CAM = (40.0, 525.0)

# coverage classes -> the kernel line each exists for (reference line after "vs")
CLASSES = {
    "hamming_tie": "k_stereo.cu:144-150 min over (dist << 16 | iR): first of tied distances vs Frame.cc:543",
    "band_edge_row": "k_stereo.cu:139 left row equal to a candidate's minr or maxr",
    "band_spans_3_bins": "k_stereo.cu:47,89 a right keypoint registered in three or more 8-row bins",
    "octave_window_edge": "k_stereo.cu:140 best candidate one octave away from the left keypoint",
    "u_at_maxU": "k_stereo.cu:141 candidate exactly at maxU = uL",
    "u_at_minU": "k_stereo.cu:141 candidate exactly at minU = uL - maxD",
    "minU_negative": "k_stereo.cu:125 minU < 0 with candidates in range",
    "best_74_accepted": "k_stereo.cu:153 best distance 74 goes on to the SAD search",
    "best_75_rejected": "k_stereo.cu:153 best distance 75 is rejected",
    "sad_tie": "k_stereo.cu:194 a later shift with the best SAD: first wins",
    "sad_extreme_rejected": "k_stereo.cu:196 best shift at -5 or +5",
    "parabola_half_step": "k_stereo.cu:201-203 |deltaR| = 0.5, the largest step the fit can take",
    # (uL - 0.01 in double, then float, equals uL - 0.01f in float for every float uL in [1, 4096): only the clamp itself shows)
    "disparity_clamp": "k_stereo.cu:208-211 zero disparity clamped to 0.01, uR = uL - 0.01, depth = bf / 0.01f",
    "disparity_ge_maxD": "k_stereo.cu:207 refined disparity at or beyond maxD",
    "sad_window_left_of_level": "k_stereo.cu:164 scaleduR0 - 10 < 0: the window leaves the level (reference: cv::Mat range)",
    "median_odd": "k_stereo.cu:252 odd number of accepted matches",
    "median_even": "k_stereo.cu:252 even number of accepted matches",
    "median_single": "k_stereo.cu:252 one accepted match",
    "median_across_hist_bin": "k_stereo.cu:255,270 median on a multiple of 256, or its neighbours in another coarse bin",
    "cull_boundary": "k_stereo.cu:278 largest kept / smallest culled SAD next to thDist",
    "no_accepted": "k_stereo.cu:251 nothing accepted: no median, no cull",
    "nR_gt_8192": "k_stereo.cu:144 more than 8192 right keypoints in the 16-bit iR",
    "all_bins_last_rows": "k_stereo.cu:39,132 nb == SBIN_MAX (h = 4095): kept matches in the last four bins that hold records",
    "records_exceed_left_stride": "k_stereo.cu:94,134 right records beyond the left handle's record stride",
}
# Branches of the code that no extracted keypoint can take, so no case claims them:
UNREACHABLE = {
    # d2 is the FIRST minimum of the SAD scan, so d1 (the earlier shift) is strictly larger and d3 is not smaller: the
    # denominator 2*(d1+d3-2*d2) > 0 and |deltaR| = |d1-d3| / (2*(d1-d2 + d3-d2)) <= 1/2.  Neither den == 0 nor the |deltaR| > 1
    # reject (k_stereo.cu:204, Frame.cc:600) can happen; parabola_half_step pins the largest step instead.
    "parabola_flat": "den > 0 whenever the best shift is not an extreme",
    # uR0 <= uL (the u-range) and a left keypoint lies at most at W_l - 20 on its own level (FAST in a cell clipped at
    # W_l - 16), so scaleduR0 + 11 <= W_l - 9: endu never reaches the level width, and iniu = scaleduR0 >= 0 always.
    "endu_guard": "uR0 <= uL keeps the window inside the level on the right",
    # Images are at most BORB_MAX_DIM = 4095 rows, so (h >> 3) + 1 <= 512: the min() with SBIN_MAX on nb (k_stereo.cu:39) and on
    # the left row's bin (:141) never changes a value.  all_bins_last_rows runs the largest table there is instead.
    "sbin_max_clamp": "h <= 4095 keeps nb and every bin index below SBIN_MAX without the clamp",
}


# ---------------------------------------------------------------------------------------------------------------------------
# restated host constants
def sel_image_stride(w, h, nfeatures, scale_factor, nlevels):
    levels, refusal = G.geometry(w, h, nfeatures=nfeatures, scale_factor=scale_factor, nlevels=nlevels)
    assert refusal is None, refusal
    return sum(lv["node_cap"] for lv in levels)


def rec_stride(w, h, nfeatures, scale_factor, nlevels):
    """k_stereo.cu stereo_rec_stride: a band spans 2*ceil(2*scale_max)+2 rows, at most (that >> 3) + 2 bins."""
    scale, _, _ = G.scale_tables(nfeatures, scale_factor, nlevels)
    band = 2 * math.ceil(f32(2.0) * scale[nlevels - 1]) + 3
    return sel_image_stride(w, h, nfeatures, scale_factor, nlevels) * ((band >> SBIN_SHIFT) + 2)


def n_bins(h):
    return min((h >> SBIN_SHIFT) + 1, SBIN_MAX)                       # k_stereo.cu:39


def _roundf(v):
    v = float(v)
    return int(math.copysign(math.floor(abs(v) + 0.5), v))             # roundf: halves away from zero


# ---------------------------------------------------------------------------------------------------------------------------
# crafted images
def shifted(img, d):
    """Right = left shifted by an integer disparity d (a left point at x shows up at x - d); the last d columns repeat."""
    R = np.empty_like(img)
    R[:, :-d] = img[:, d:]
    R[:, -d:] = img[:, -1:]
    return R


def periodic(seed, w, h, period):
    """A texture that repeats every `period` columns: keypoints one period apart carry the same descriptor on a row."""
    tile = synth.mono_frame(seed, 0, 0, period, h)
    return np.ascontiguousarray(np.tile(tile, (1, -(-w // period)))[:, :w])


def blobs(seed, w, h, n, d, noise):
    """Flat background with n bright squares; right = left shifted by d plus +-noise gray levels (so SAD > 0)."""
    rng = np.random.default_rng(seed)
    L = np.full((h, w), 90, np.uint8)
    for _ in range(n):
        s = int(rng.integers(8, 20))
        x, y = int(rng.integers(60, w - 60)), int(rng.integers(60, h - 60))
        L[y:y + s, x:x + s] = int(rng.integers(160, 240))
    R = shifted(L, d).astype(np.int16) + rng.integers(-noise, noise + 1, (h, w))
    return L, np.clip(R, 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------------
# cases: name -> dict(w, h, left=(nf, sf, nl), right=(nf, sf, nl), cam=(bf, fx), images=callable() -> (L, R))
def _natural(seed, w, h):
    return lambda: synth.stereo_pair(seed, 0, 0, w, h)[:2]


def _mono_shift(seed, w, h, d):
    def f():
        L = synth.mono_frame(seed, 0, 0, w, h)
        return L, shifted(L, d)
    return f


def _same(seed, w, h):
    def f():
        L = synth.mono_frame(seed, 0, 0, w, h)
        return L, L.copy()
    return f


def _periodic(seed, w, h, period, d):
    def f():
        R = periodic(seed, w, h, period)
        return np.ascontiguousarray(np.roll(R, d, axis=1)), R
    return f


def _blank_right(seed, w, h):
    return lambda: (synth.mono_frame(seed, 0, 0, w, h), np.full((h, w), 90, np.uint8))


def _blobs(seed, w, h, n, d, noise):
    return lambda: blobs(seed, w, h, n, d, noise)


def _half_same(seed, w, h, d, noise):
    """Left half of the right image = left image (zero disparity), right half shifted by d with +-noise gray levels: the
    shifted half keeps the median SAD above zero, so clamped zero-disparity matches of the identical half survive the cull."""
    def f():
        L = synth.mono_frame(seed, 0, 0, w, h)
        rng = np.random.default_rng(seed)
        R = np.clip(shifted(L, d).astype(np.int16) + rng.integers(-noise, noise + 1, (h, w)), 0, 255).astype(np.uint8)
        R[:, :w // 2] = L[:, :w // 2]
        return L, R
    return f


def _case(w, h, images, left, right=None, cam=KITTI_CAM, ref_asserts=False):
    return dict(w=w, h=h, images=images, left=left, right=right or left, cam=cam, ref_asserts=ref_asserts)


KW, KH = synth.KITTI
CASES = {
    # settings
    "kitti_1.2x8": _case(KW, KH, _natural(700, KW, KH), (2000, 1.2, 8)),
    "vga_1.2x12": _case(640, 480, _natural(701, 640, 480), (2000, 1.2, 12), cam=VGA_CAM),    # KITTI: level 10 has no FAST cell
    "kitti_1.5x5": _case(KW, KH, _natural(702, KW, KH), (2000, 1.5, 5)),
    "kitti_2.0x3": _case(KW, KH, _natural(703, KW, KH), (2000, 2.0, 3)),
    "kitti_1.05x6": _case(KW, KH, _natural(704, KW, KH), (2000, 1.05, 6)),
    "kitti_11200": _case(KW, KH, _natural(705, KW, KH), (11200, 1.2, 8)),                       # extract_geometry.ENVELOPE
    # crafted content
    "periodic_48": _case(KW, KH, _periodic(706, KW, KH, 48, 20), (2000, 1.2, 8)),
    "shift_23": _case(KW, KH, _mono_shift(707, KW, KH, 23), (2000, 1.2, 8)),
    "shift_23_maxD_23": _case(KW, KH, _mono_shift(708, KW, KH, 23), (2000, 1.2, 8), cam=(46.0, 23.0)),   # b = 2, maxD = 23
    "half_same_LR": _case(640, 480, _half_same(901, 640, 480, 10, 4), (1000, 1.2, 8), cam=VGA_CAM),
    "same_LR": _case(640, 480, _same(709, 640, 480), (1000, 1.2, 8), cam=VGA_CAM),
    "blank_right": _case(640, 480, _blank_right(710, 640, 480), (1000, 1.2, 8), cam=VGA_CAM),
    "blobs_one_accepted": _case(640, 480, _blobs(205, 640, 480, 2, 10, 3), (1000, 1.2, 8), cam=VGA_CAM),
    "blobs_two_accepted": _case(640, 480, _blobs(46, 640, 480, 1, 10, 3), (1000, 1.2, 8), cam=VGA_CAM),
    "tall_2120x4095": _case(2120, 4095, _natural(711, 2120, 4095), (2000, 1.2, 8)),   # 2100 x 4095: level 7 has no quadtree root
    # scaleFactor > 2: an octave-0 right keypoint at x = 19..23 is the best match of an octave-1 left keypoint, and its window
    # scaleduR0 - 10 = round(x / 2.5) - 10 < 0 leaves level 1 (the reference would index before the row: not comparable)
    "vga_2.5x3": _case(640, 480, _natural(720, 640, 480), (2000, 2.5, 3), cam=VGA_CAM, ref_asserts=True),
    # two handles with differing nfeatures (borb_stereo_match2)
    "kitti_L1000_R4000": _case(KW, KH, _natural(712, KW, KH), (1000, 1.2, 8), (4000, 1.2, 8)),
    "kitti_L4000_R1000": _case(KW, KH, _natural(713, KW, KH), (4000, 1.2, 8), (1000, 1.2, 8)),
}
NAMES = list(CASES)


def geometry_ok(c):
    for nf, sf, nl in (c["left"], c["right"]):
        _, refusal = G.geometry(c["w"], c["h"], nfeatures=nf, scale_factor=sf, nlevels=nl)
        if refusal is not None:
            return refusal
    return None


@functools.lru_cache(maxsize=None)
def images(name):
    L, R = CASES[name]["images"]()
    return np.ascontiguousarray(L, np.uint8), np.ascontiguousarray(R, np.uint8)


@functools.lru_cache(maxsize=None)
def run_port(oracle, name):
    """Port extraction of both images with their own settings, then the port's stereo association.  -> dict"""
    c = CASES[name]
    L, R = images(name)
    EL, ER = oracle.PortExtractor(*c["left"]), oracle.PortExtractor(*c["right"])
    kl, dl = EL(L)
    kr, dr = ER(R)
    pyrL = [EL.level(i) for i in range(EL.nlevels)]
    pyrR = [ER.level(i) for i in range(ER.nlevels)]
    bf, fx = c["cam"]
    ur, dp, sad = oracle.port_stereo(kl, dl, kr, dr, pyrL, pyrR, EL.scale, EL.inv_scale, bf, fx)
    return dict(kl=kl, dl=dl, kr=kr, dr=dr, pyrL=pyrL, pyrR=pyrR, scale=EL.scale.copy(), inv_scale=EL.inv_scale.copy(),
                ur=ur, dp=dp, sad=sad)


_POP = np.array([bin(i).count("1") for i in range(256)], np.int32)


def _hamming(a, B):
    return _POP[np.bitwise_xor(B, a[None, :])].sum(1)


def _refine(p, kp, iR, maxD, bf):
    """SAD search, parabola and disparity gate of one left keypoint against right keypoint iR (k_stereo.cu:153-219).
    -> (status, bestD, uR, depth, tags): status "ok", "window_left", "extreme" or "disparity"."""
    scale, inv_scale = p["scale"], p["inv_scale"]
    oL = int(kp["octave"])
    uL = f32(kp["x"])
    tags = set()
    sf = inv_scale[oL]
    cxL, cy, cxR = _roundf(f32(kp["x"]) * sf), _roundf(f32(kp["y"]) * sf), _roundf(f32(p["kr"]["x"][iR]) * sf)
    IL, IR = p["pyrL"][oL].astype(np.int32), p["pyrR"][oL].astype(np.int32)
    Hl, Wl = IL.shape
    assert cy - W >= 0 and cy + W < Hl and cxL - W >= 0 and cxL + W < Wl       # left windows always fit (see UNREACHABLE)
    assert cxR >= 0 and cxR + LH + W + 1 < Wl
    if cxR - LH - W < 0:
        return "window_left", None, None, None, tags
    pl = IL[cy - W:cy + W + 1, cxL - W:cxL + W + 1]
    pl = pl - pl[W, W]
    d = []
    for inc in range(-LH, LH + 1):
        pr = IR[cy - W:cy + W + 1, cxR + inc - W:cxR + inc + W + 1]
        d.append(int(np.abs(pl - (pr - pr[W, W])).sum()))
    bi = int(np.argmin(d))                        # first of tied minima in shift order
    bestD, binc = d[bi], bi - LH
    if d.count(bestD) > 1:
        tags.add("sad_tie")
    if binc in (-LH, LH):
        return "extreme", bestD, None, None, tags
    d1, d2, d3 = f32(d[bi - 1]), f32(d[bi]), f32(d[bi + 1])
    den = f32(2.0) * (d1 + d3 - f32(2.0) * d2)
    assert den > 0                                # see UNREACHABLE["parabola_flat"]
    deltaR = (d1 - d3) / den
    if abs(deltaR) == f32(0.5):
        tags.add("parabola_half_step")
    bestuR = scale[oL] * ((f32(cxR) + f32(binc)) + deltaR)
    disp = uL - bestuR
    if not (disp >= 0 and disp < maxD):
        if disp >= maxD:
            tags.add("disparity_ge_maxD")
        return "disparity", bestD, None, None, tags
    if disp <= 0:
        tags.add("disparity_clamp")
        disp = f32(0.01)
        bestuR = f32(float(uL) - 0.01)
    return "ok", bestD, bestuR, f32(bf) / disp, tags


@functools.lru_cache(maxsize=None)
def restate(oracle, name):
    """numpy restatement of the whole association on the port's keypoints.  -> (ur, dp, classes hit, records)

    A class counts only where its effect reaches mvuRight / mvDepth, so that a kernel that got the branch wrong would change
    the output: a class of an accepted match counts if the match survives the median cull; a rejection counts if the rejected
    match would have survived the cull had it been accepted (its SAD below thDist; for best distance 75, the SAD search run as
    if it had passed)."""
    c = CASES[name]
    p = run_port(oracle, name)
    kl, dl, kr, dr, scale = p["kl"], p["dl"], p["kr"], p["dr"], p["scale"]
    h = c["h"]
    bf, fx = c["cam"]
    b = f32(bf) / f32(fx)
    maxD = f32(bf) / b
    hit = set()
    nL, nR = len(kl), len(kr)
    ur = np.full(nL, -1.0, f32)
    dp = np.full(nL, -1.0, f32)
    # right keypoints: row bands and bins (k_stereo.cu:43-49)
    r = f32(2.0) * scale[kr["octave"]] if nR else np.zeros(0, f32)
    maxr = np.ceil(kr["y"] + r).astype(np.int64)
    minr = np.floor(kr["y"] - r).astype(np.int64)
    nb = n_bins(h)
    b0 = np.maximum(minr, 0) >> SBIN_SHIFT
    b1 = np.minimum(np.minimum(maxr, h - 1) >> SBIN_SHIFT, nb - 1)
    records = int((b1 - b0 + 1).clip(min=0).sum())
    if records > rec_stride(c["w"], h, *c["left"]):
        hit.add("records_exceed_left_stride")
    rows = [[] for _ in range(h)]
    for i in range(nR):
        for y in range(max(minr[i], 0), min(maxr[i], h - 1) + 1):
            rows[y].append(i)
    rows = [np.array(v, np.int64) for v in rows]
    acc, tags_of, rejected = [], {}, []
    for iL in range(nL):
        kp = kl[iL]
        uL, vL, oL = f32(kp["x"]), f32(kp["y"]), int(kp["octave"])
        row = int(vL)
        cand = rows[row] if 0 <= row < h else np.zeros(0, np.int64)
        minU, maxU = uL - maxD, uL
        if len(cand) == 0 or maxU < 0:
            continue
        oR = kr["octave"][cand]
        uR = kr["x"][cand]
        ok = (oR >= oL - 1) & (oR <= oL + 1) & (uR >= minU) & (uR <= maxU)
        ev = cand[ok]
        if len(ev) == 0:
            continue
        dist = _hamming(dl[iL], dr[ev])
        k = int(np.argmin(dist))                  # first of tied minima in iR order
        best = int(dist[k])
        if best >= TH_HIGH:
            continue
        iR = int(ev[k])
        if best == TH_ORB:                        # would the match have survived had the gate let it through?
            st, bestD, _, _, _ = _refine(p, kp, iR, maxD, bf)
            if st == "ok":
                rejected.append(("best_75_rejected", bestD))
        if best >= TH_ORB:
            continue
        # tags of the winning candidate: each decides which right keypoint the SAD search starts from
        tags = set()
        if best == TH_ORB - 1:
            tags.add("best_74_accepted")
        if (dist == best).sum() > 1:
            tags.add("hamming_tie")
        if abs(int(kr["octave"][iR]) - oL) == 1:
            tags.add("octave_window_edge")
        if row in (minr[iR], maxr[iR]):
            tags.add("band_edge_row")
        if kr["x"][iR] == maxU:
            tags.add("u_at_maxU")
        if kr["x"][iR] == minU:
            tags.add("u_at_minU")
        if minU < 0:
            tags.add("minU_negative")
        if b1[iR] - b0[iR] >= 2:
            tags.add("band_spans_3_bins")
        if iR >= 8192:
            tags.add("nR_gt_8192")
        if nb == SBIN_MAX and (row >> SBIN_SHIFT) >= int(b1.max()) - 3:        # one of the last four bins that hold records
            tags.add("all_bins_last_rows")
        st, bestD, u, dd, t = _refine(p, kp, iR, maxD, bf)
        tags |= t
        if st == "window_left":
            rejected.append(("sad_window_left_of_level", None))
        elif st == "extreme":
            rejected.append(("sad_extreme_rejected", bestD))
        elif st == "disparity" and "disparity_ge_maxD" in t:
            rejected.append(("disparity_ge_maxD", bestD))
        if st != "ok":
            continue
        ur[iL], dp[iL] = u, dd
        acc.append((bestD, iL))
        tags_of[iL] = tags
    n = len(acc)
    if nL and n == 0:
        hit.add("no_accepted")
    if n:
        acc.sort()
        hit.add("median_odd" if n % 2 else "median_even")
        if n == 1:
            hit.add("median_single")
        ds = [a[0] for a in acc]
        k = n // 2
        med = ds[k]
        if med % HIST_BINS == 0 or any(0 <= j < n and ds[j] >> 8 != med >> 8 for j in (k - 1, k + 1)):
            hit.add("median_across_hist_bin")
        th = f32(f32(1.5) * f32(1.4)) * f32(med)
        kept = [x for x in ds if f32(x) < th]
        culled = [x for x in ds if not f32(x) < th]
        lo, hi = math.ceil(float(th)) - 1, math.ceil(float(th))       # largest integer below thDist, smallest at or above it
        if (kept and kept[-1] == lo) or (culled and culled[0] == hi):
            hit.add("cull_boundary")
        for x, i in acc:
            if not f32(x) < th:
                ur[i] = dp[i] = f32(-1.0)
            else:
                hit |= tags_of[i]
        for cls, bestD in rejected:
            if kept and (bestD is None or f32(bestD) < th):
                hit.add(cls)
    return ur, dp, frozenset(hit), records


def coverage(oracle, name):
    return restate(oracle, name)[2]


def record_count(oracle, name):
    """Right-keypoint records stereo_bin_kernel writes for the case (k_stereo.cu:85-95), before the stride clamp."""
    return restate(oracle, name)[3]


def ref_eligible(oracle, name):
    """Cases the verbatim Frame.cc can run: not reference-asserting, and something accepted (Frame.cc:627 is UB on an empty
    vDistIdx)."""
    return not CASES[name]["ref_asserts"] and bool((run_port(oracle, name)["sad"] >= 0).any())
