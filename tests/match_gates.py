"""Matcher inputs placed on the descriptor-distance gates every matcher kernel applies after its Hamming distances: the TH_HIGH /
TH_LOW / ORBdist thresholds, the nnratio products, the second best taken under claims, and the order in which
SearchForTriangulation keeps its candidate.  Test tooling: tests/test_oracle_match_gates.py pins the port to the verbatim
ORBmatcher.cc on every case and checks that both members of every pair are decided differently by the verbatim build;
tests/test_gpu_match_gates.py pins the CUDA library to the port.

The geometry is deliberately boring (tests/proj_geometry.py's poses, points well inside the frustum, one grid cell, one
FeatureVector node, level 0 unless a class needs another), so that the descriptors decide.  Descriptors sit at exact Hamming
distances from a query: each candidate flips its own bits of the query, drawn from one pool without replacement, so that two
candidates' distances to the query are independent and their distance to each other is the sum.  A pair is two cases that
differ in one descriptor bit, one nnratio step or one claim; each gate is restated here in numpy, in integers and with the
float32 product in the reference's order, next to the kernel line it exists for.  Nothing in this module calls the CUDA library.

The resident-keyframe-database BoW searches (tests/bow_envelope.py), the stereo match (tests/stereo_envelope.py) and the rotation
histogram (proj_geometry rot_*, match_envelope hist_boundary) are pinned at their gates elsewhere."""
import dataclasses
import functools
import operator
import zlib

import numpy as np

from orb_slam2_b200.matcher import FeatureVector, FrameView, KeyFrameView, MapPointsView
from tests import proj_geometry as G

f32, f64 = np.float32, np.float64
TH_LOW, TH_HIGH = 50, 100                  # ORBmatcher.cc:15-16
BOW_JCAP = 1024                            # k_match.cu:332 — wider target buckets are evaluated directly (k_match.cu:424-434)
INIT_K = 8                                 # borb_match.h:96 — window entries per F1 feature in init_prefix_kernel's prefix
INT_MAX_F = f32(2147483648.0)              # (float)INT_MAX, SearchForInitialization's bestDist2 without a second entry

# coverage classes -> the kernel line each exists for
CLASSES = {
    # thresholds, one pair each (world-point cases, run through every world-point method; the decider is named in DECIDER)
    "th_local_100": "k_proj.cu:333 bestDist <= TH_HIGH in SearchLocalPoints' SearchByProjection(F, vpMapPoints)",
    "th_last_100": "k_proj.cu:332 bestDist <= th_dist = TH_HIGH in SearchByProjection(CurrentFrame, LastFrame) (borb_match_host.cu:938)",
    "th_kf_orbdist_64": "k_proj.cu:332 bestDist <= ORBdist = 64 in SearchByProjection(CurrentFrame, KeyFrame) (borb_match_host.cu:947)",
    "th_kf_orbdist_100": "k_proj.cu:332 bestDist <= ORBdist = 100 in SearchByProjection(CurrentFrame, KeyFrame)",
    "th_sim3proj_50": "k_proj.cu:332 bestDist <= th_dist = TH_LOW in SearchByProjection(pKF, Scw) (borb_match_host.cu:956)",
    "th_fuse_kf_50": "k_proj.cu:215 best >> 16 <= TH_LOW in Fuse(pKF, vpMapPoints) (borb_match_host.cu:1096)",
    "th_fuse_scw_50": "k_proj.cu:215 best >> 16 <= TH_LOW in Fuse(pKF, Scw)",
    "th_sim3_12": "k_proj.cu:215 best >> 16 <= TH_HIGH in SearchBySim3's direction 1 -> 2 (borb_match_host.cu:1186)",
    "th_sim3_21": "k_proj.cu:215,237 direction 2 -> 1 at 101 refuses a point 1 -> 2 accepts at 100; the agreement test drops it",
    # SearchByProjection(F, vpMapPoints): ratio only at bestLevel == bestLevel2, `>` against the float product
    "proj_no_second": "k_proj.cu:333-337 no second entry: bestDist2 = 256, bestLevel2 = -1, so no ratio even at nnratio 0.25",
    "proj_ratio_07": "k_proj.cu:337 (float)bestDist > __fmul_rn(0.7f, bestDist2) at (7, 10), where the float product is 7.0",
    "proj_ratio_09": "k_proj.cu:337 (float)bestDist > __fmul_rn(0.9f, bestDist2) at (9, 10), where the float product is 9.0",
    "proj_ratio_075": "k_proj.cu:337 bestDist == 0.75 * bestDist2 exactly: `>` keeps the match",
    "proj_ratio_levels": "k_proj.cu:337 bestLevel != bestLevel2: the same distances never apply the ratio",
    "proj_claim_held": "k_proj.cu:313 a second held by a MapPoint with observations is skipped for the ratio",
    "proj_claim_wave": "k_proj.cu:313 a second claimed by an earlier query of the wave is skipped for the ratio",
    # SearchByBoW(KF, F) (mode 0) and SearchByBoW(KF1, KF2) (mode 1)
    "bow0_th": "k_match.cu:440 mode 0 bestDist1 <= TH_LOW",
    "bow0_ratio_06": "k_match.cu:441 (float)bestDist1 < __fmul_rn(0.6f, bestDist2) at (3, 5), where the float product is 3.0",
    "bow0_ratio_08": "k_match.cu:441 (float)bestDist1 < __fmul_rn(0.8f, bestDist2) at (4, 5), where the float product is 4.0",
    "bow0_ratio_075": "k_match.cu:441 bestDist1 == 0.75 * bestDist2 exactly: `<` drops the match",
    "bow0_one_col": "k_match.cu:439 a one-column bucket: bestDist2 = 256, at nnratio 50/256",
    "bow0_claim": "k_match.cu:420 a column claimed by an earlier row is skipped for best and second",
    "bow0_wide_ratio_06": "k_match.cu:424-434,441 the 0.6 product in a bucket wider than BOW_JCAP (direct evaluation)",
    "bow0_wide_claim": "k_match.cu:428 the claimed second in a bucket wider than BOW_JCAP",
    "bow1_th": "k_match.cu:440 mode 1 bestDist1 < TH_LOW (strict)",
    "bow1_ratio_06": "k_match.cu:441 mode 1 at (3, 5) and 0.6f",
    "bow1_ratio_08": "k_match.cu:441 mode 1 at (4, 5) and 0.8f",
    "bow1_ratio_075": "k_match.cu:441 mode 1 at bestDist1 == 0.75 * bestDist2",
    "bow1_one_col": "k_match.cu:439 mode 1 one-column bucket at nnratio 49/256",
    "bow1_claim": "k_match.cu:420 mode 1: a column an earlier row matched (vbMatched2) is skipped for best and second",
    "bow1_no_mp": "k_match.cu:383 mode 1: a column without a MapPoint is skipped for best and second",
    "bow1_wide_no_mp": "k_match.cu:429 mode 1: the column without a MapPoint in a bucket wider than BOW_JCAP",
    "bow1_wide_claim": "k_match.cu:428 mode 1: the claimed second in a bucket wider than BOW_JCAP",
    # SearchForInitialization
    "init_th": "k_proj.cu:572 bestDist <= TH_LOW",
    "init_ratio_06": "k_proj.cu:572 (float)bestDist < __fmul_rn((float)bestDist2, 0.6f) at (3, 5)",
    "init_ratio_08": "k_proj.cu:572 (float)bestDist < __fmul_rn((float)bestDist2, 0.8f) at (4, 5)",
    "init_ratio_075": "k_proj.cu:572 bestDist == 0.75 * bestDist2 exactly: `<` drops the match",
    "init_no_second_09": "k_proj.cu:571 a single-candidate window at nnratio 0.9: bestDist2 = INT_MAX",
    "init_no_second_10": "k_proj.cu:571 a single-candidate window at nnratio 1.0",
    "init_no_second_int_max": "k_proj.cu:571 2147483648.f * nnratio == 50 exactly at nnratio 25 * 2^-30, where 256 * nnratio is 6e-6",
    "init_excl_prefix": "k_proj.cu:548 vMatchedDistance[i2] <= dist excludes an equal distance; a smaller one displaces the owner",
    "init_excl_walk": "k_proj.cu:560 the same exclusion in the window walk, after eight excluded prefix entries",
    # SearchForTriangulation
    "tri_th": "k_match.cu:525 dist > TH_LOW rejects, so 50 matches",
    "tri_order_epipole": "k_match.cu:527-536 a closer candidate near the epipole does not shadow a later one that passes",
    "tri_order_epiline": "k_match.cu:531-536 a closer candidate off the epipolar line does not shadow a later one that passes",
    "tri_equal_later": "k_match.cu:536 dist <= bestDist: of two equal distances the later candidate wins",
}

# rows of the gate table these cases do not reach, each with the reason; test_every_class_is_reached keeps CLASSES and this
# table together
NOT_COVERED = {
    "proj_ratio_06_08": "k_proj.cu:337 at 0.6f and 0.8f: both round above the decimal, so a float product that lands on an integer "
                        "d1 has an exact product above d1 as well, and `d1 > product` is false either way: no pair can separate them",
    "lt_ratio_07_09": "k_match.cu:441 and k_proj.cu:572 at 0.7f and 0.9f: both round below the decimal, so `d1 < product` is false "
                      "in float and in exact arithmetic alike wherever the float product lands on d1",
    "ratio_10": "nnratio 1.0: every product is exact, float and double agree everywhere",
    "fuse_sim3_ratio": "Fuse, SearchBySim3 and the LAST-mode projection searches apply no ratio test (k_proj.cu:215,332)",
}

# ---------------------------------------------------------------------------------------------------------------------------
# the gates, restated: integers, and the float32 product in the reference's operation order


def proj_gate(d1, l1, d2, l2, r, prod=lambda r, d2: f32(f32(r) * f32(d2))):
    """SearchByProjection(F, vpMapPoints) (ORBmatcher.cc:118-120, k_proj.cu:333-337): d2 None means no second entry."""
    if d2 is None:
        d2, l2 = 256, -1
    return bool(d1 <= TH_HIGH and not (l1 == l2 and f32(d1) > prod(r, d2)))


def bow_gate(mode, d1, d2, r, prod=lambda r, d2: f32(f32(r) * f32(d2))):
    """SearchByBoW (ORBmatcher.cc:228-230, 598-600, k_match.cu:439-441): mode 0 `<=`, mode 1 `<`; d2 None is a one-column bucket."""
    d2 = 256 if d2 is None else d2
    return bool((d1 <= TH_LOW if mode == 0 else d1 < TH_LOW) and f32(d1) < prod(r, d2))


def init_gate(d1, d2, r, prod=lambda r, d2: f32(f32(d2) * f32(r))):
    """SearchForInitialization (ORBmatcher.cc:459-461, k_proj.cu:570-572): bestDist < (float)bestDist2*mfNNratio, d2 None is
    INT_MAX."""
    return bool(d1 <= TH_LOW and f32(d1) < prod(r, INT_MAX_F if d2 is None else d2))


def double_product(r, d2):
    """What a restatement that multiplied in double would compare against."""
    return f64(f32(r)) * f64(d2)


def separating(r, op):
    """The (d1, d2), d2 in 1..256, that `d1 op r*d2` decides differently with the float32 product and the exact one."""
    out = []
    for d2 in range(1, 257):
        p32, p64 = f32(f32(r) * f32(d2)), f64(f32(r)) * f64(d2)
        out += [(d1, d2) for d1 in range(0, 257) if op(f64(d1), f64(p32)) != op(f64(d1), p64)]
    return out


def first_separating(r, op):
    return separating(r, op)[0]


# ---------------------------------------------------------------------------------------------------------------------------
# descriptors at exact distances
class Bits:
    """Descriptors at exact Hamming distances from `base`: each call flips bits drawn from one pool without replacement, so two
    results are at the sum of their distances from each other."""

    def __init__(self, seed, base=None):
        self.rng = np.random.default_rng(seed)
        self.base = self.rng.integers(0, 256, 32, dtype=np.uint8) if base is None else np.asarray(base, np.uint8)
        self.pool = list(self.rng.permutation(256))

    def at(self, d, base=None):
        bits = np.unpackbits(self.base if base is None else base).copy()
        bits[[self.pool.pop() for _ in range(d)]] ^= 1
        return np.packbits(bits)


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(np.asarray(a, np.uint8), np.asarray(b, np.uint8))).sum())


def _seed(cls):
    return zlib.crc32(cls.encode()) % 100000


def fillers(seed, base, n):
    """n descriptors at least 200 bits from base (and so from every descriptor a few bits from it)."""
    rng = np.random.default_rng(seed)
    out = np.repeat(~np.asarray(base, np.uint8)[None], n, 0)
    bits = np.unpackbits(out, axis=1)
    for i in range(n):
        bits[i, rng.choice(256, 20, replace=False)] ^= 1
    return np.packbits(bits, axis=1)


def _ratio_pair(r, op):
    """(nnratio of member 0, nnratio of member 1) on the float product's boundary: for `<` the product equal to d1 drops the
    match and one step up keeps it; for `>` the product equal to d1 keeps it and one step down drops it."""
    r = f32(r)
    return (G.step(r, 1), r) if op is operator.lt else (r, G.step(r, -1))


# ---------------------------------------------------------------------------------------------------------------------------
# world-point cases: point 0 at U0_CAM seen by keypoint 0 half a pixel from its projection, and proj_geometry's ordinary points;
# point 0's descriptor sits d12 bits from keypoint 0's (d21 for KF2's points in SearchBySim3)
DECIDER = {"th_local_100": "local_match", "th_last_100": "last", "th_kf_orbdist_64": "kf", "th_kf_orbdist_100": "kf",
           "th_sim3proj_50": "sim3proj", "th_fuse_kf_50": "fuse_kf", "th_fuse_scw_50": "fuse", "th_sim3_12": "sim3",
           "th_sim3_21": "sim3"}
WORLD_METHODS = ("local", "last", "kf", "sim3proj", "fuse", "fuse_kf", "sim3")


def _world(cls, member, d12, d21=None, orb_dist=100):
    c = G._world_case(cls, member, G.U0_CAM, (G.U0 + 0.5, G.V0))
    kd = c["F"].mDescriptors
    P1 = dataclasses.replace(c["P"], descriptors=c["P"].descriptors.copy())
    P1.descriptors[0] = Bits(_seed(cls) + 1, kd[0]).at(d12)
    P2 = dataclasses.replace(c["P"], descriptors=c["P"].descriptors.copy())
    P2.descriptors[0] = Bits(_seed(cls) + 2, kd[0]).at(d12 if d21 is None else d21)
    return dict(c, P=P1, P2=P2, orb_dist=orb_dist, focus=(0, 0), dists=(d12, d21))


def _pairs_world():
    out = []
    for cls, th, orb in (("th_local_100", TH_HIGH, 100), ("th_last_100", TH_HIGH, 100), ("th_kf_orbdist_64", 64, 64),
                         ("th_kf_orbdist_100", 100, 100), ("th_sim3proj_50", TH_LOW, 100), ("th_fuse_kf_50", TH_LOW, 100),
                         ("th_fuse_scw_50", TH_LOW, 100)):
        for m, d in enumerate((th, th + 1)):
            out.append(_world(cls, m, d, orb_dist=orb))
    for m, d in enumerate((TH_HIGH, TH_HIGH + 1)):
        out.append(_world("th_sim3_12", m, d, TH_HIGH))
        out.append(_world("th_sim3_21", m, TH_HIGH, d))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchByProjection(F, vpMapPoints, th = 1): every query projects to (100, 100) at level `level` (radius 4 * scale), its
# candidates are keypoints k = 0, 1, ... at (100 + 0.25 * (k + 1), 100), one grid cell, in index (= GetFeaturesInArea) order
def _proj(cls, member, ratio, qdesc, kdesc, octaves=None, occupied=None, has_obs=None, level=0, focus=(0, 0)):
    nk, nq = len(kdesc), len(qdesc)
    keys = G._keys([(100.0 + 0.25 * (k + 1), 100.0) for k in range(nk)])
    keys["octave"] = octaves if octaves is not None else 0
    F = FrameView(mvKeysUn=keys, mDescriptors=np.stack(kdesc), mvScaleFactors=G.SCALE, bounds=G.BOUNDS,
                  mvuRight=np.full(nk, -1.0, np.float32), occupied=None if occupied is None else np.asarray(occupied, np.uint8))
    mps = MapPointsView(mTrackProjX=np.full(nq, 100.0, np.float32), mTrackProjY=np.full(nq, 100.0, np.float32),
                        mTrackProjXR=np.full(nq, -1.0, np.float32), mnTrackScaleLevel=np.full(nq, level, np.int32),
                        mTrackViewCos=np.full(nq, 0.9, np.float32), descriptors=np.stack(qdesc), valid=np.ones(nq, np.uint8),
                        has_obs=np.ones(nq, np.uint8) if has_obs is None else np.asarray(has_obs, np.uint8))
    return dict(cls=cls, member=member, kind="proj", F=F, mps=mps, th=1.0, ratio=float(ratio), focus=focus)


def _pairs_proj():
    out = []
    b = Bits(_seed("proj_no_second"))
    k0 = {d: b.at(d) for d in (TH_HIGH, TH_HIGH + 1)}
    for m, d in enumerate((TH_HIGH, TH_HIGH + 1)):
        out.append(_proj("proj_no_second", m, 0.25, [b.base], [k0[d]]))
    for cls, r in (("proj_ratio_07", 0.7), ("proj_ratio_09", 0.9), ("proj_ratio_075", 0.75)):
        d1, d2 = (3, 4) if r == 0.75 else first_separating(r, operator.gt)
        b = Bits(_seed(cls))
        ks = [b.at(d1), b.at(d2)]
        for m, rr in enumerate(_ratio_pair(r, operator.gt)):
            out.append(dict(_proj(cls, m, rr, [b.base], ks), dists=(d1, d2)))
    # the 0.7 pair at the rejecting nnratio: the second at octave 1 (levels differ: kept) against octave 0 (ratio: dropped)
    d1, d2 = first_separating(0.7, operator.gt)
    b = Bits(_seed("proj_ratio_levels"))
    ks = [b.at(d1), b.at(d2)]
    r = _ratio_pair(0.7, operator.gt)[1]
    for m, o2 in enumerate((1, 0)):
        out.append(dict(_proj("proj_ratio_levels", m, r, [b.base], ks, octaves=[0, o2], level=1), dists=(d1, d2)))
    # held second: k1 ties the best and is held by a MapPoint with observations; the ratio is decided by k2 at 0.75 exactly
    b = Bits(_seed("proj_claim_held"))
    ks = [b.at(3), b.at(3), b.at(4)]
    for m, rr in enumerate(_ratio_pair(0.75, operator.gt)):
        out.append(_proj("proj_claim_held", m, rr, [b.base], ks, occupied=[0, 1, 0]))
    # claimed in the wave: query 0 takes ka (distance 0, with observations); query 1 sees ka at 3 (a tie with kb), kb at 3, kc at 4
    b = Bits(_seed("proj_claim_wave"))
    ka, kb, kc = b.at(3), b.at(3), b.at(4)
    for m, rr in enumerate(_ratio_pair(0.75, operator.gt)):
        out.append(_proj("proj_claim_wave", m, rr, [ka, b.base], [ka, kb, kc], focus=(1, 1)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchByBoW: every feature of both sides in FeatureVector node 0.  Mode 0: rows are the keyframe's features with a MapPoint,
# columns the frame's; mode 1: rows are KF1's features with a MapPoint, columns KF2's (those without one are skipped)
def _kfview(desc, has_mp=None, y0=20.0):
    n = len(desc)
    keys = G._keys([(20.0 + 0.5 * (i % 1200), y0 + 0.5 * (i // 1200)) for i in range(n)])
    return KeyFrameView(mvKeysUn=keys, mDescriptors=np.ascontiguousarray(np.stack(desc), np.uint8),
                        mFeatVec=FeatureVector.from_nodes(np.zeros(n, np.int64)),
                        has_mp=None if has_mp is None else np.asarray(has_mp, np.uint8))


def _bow(cls, member, mode, ratio, rows, cols, cols_mp=None, n_fill=0, focus=(0, 0)):
    """rows / cols: descriptors; the filler columns (n_fill, far from every row) come first, so that the gate columns sit at
    positions above BOW_JCAP of a bucket the direct path evaluates."""
    cols = list(cols)
    cmp_ = [1] * len(cols) if cols_mp is None else list(cols_mp)
    if n_fill:
        cols = list(fillers(_seed(cls) + 3, rows[0], n_fill)) + cols
        cmp_ = [1] * n_fill + cmp_
        focus = (focus[0], focus[1] + n_fill)
    kf = _kfview(rows, np.ones(len(rows), np.uint8))
    other = _kfview(cols, None if mode == 0 else cmp_, y0=300.0)
    return dict(cls=cls, member=member, kind=f"bow{mode}", kf=kf, F=other, ratio=float(ratio), focus=focus, n_fill=n_fill)


def _pairs_bow():
    out = []
    wide = BOW_JCAP + 76
    for mode in (0, 1):
        p = f"bow{mode}"
        th = TH_LOW if mode == 0 else TH_LOW - 1                 # the last distance each mode keeps
        b = Bits(_seed(p + "_th"))
        far = b.at(200)
        for m, d in enumerate((th, th + 1)):
            out.append(_bow(p + "_th", m, mode, 0.75, [b.base], [Bits(_seed(p) + d, b.base).at(d), far]))
        for suffix, r in (("_ratio_06", 0.6), ("_ratio_08", 0.8), ("_ratio_075", 0.75)):
            d1, d2 = (3, 4) if r == 0.75 else first_separating(r, operator.lt)
            b = Bits(_seed(p + suffix))
            cs = [b.at(d1), b.at(d2)]
            for m, rr in enumerate(_ratio_pair(r, operator.lt)):
                out.append(dict(_bow(p + suffix, m, mode, rr, [b.base], cs), dists=(d1, d2)))
                if suffix == "_ratio_06" and mode == 0:
                    out.append(dict(_bow(p + "_wide" + suffix, m, mode, rr, [b.base], cs, n_fill=wide), dists=(d1, d2)))
        # one column: bestDist2 = 256, so d1 < r*256 turns at r = d1/256 (exact)
        b = Bits(_seed(p + "_one_col"))
        c0 = b.at(th)
        r0 = f32(th / 256.0)
        for m, rr in enumerate((G.step(r0, 1), r0)):
            out.append(dict(_bow(p + "_one_col", m, mode, rr, [b.base], [c0]), dists=(th, None)))
        # claims: row 0 takes ca (distance 0); row 1 sees ca at 3 (a tie with cb), cb at 3, cc at 4, at the 0.75 product
        b = Bits(_seed(p + "_claim"))
        ca, cb, cc = b.at(3), b.at(3), b.at(4)
        for m, rr in enumerate(_ratio_pair(0.75, operator.lt)):
            out.append(_bow(p + "_claim", m, mode, rr, [ca, b.base], [ca, cb, cc], focus=(1, 1)))
            out.append(_bow(p + "_wide_claim", m, mode, rr, [ca, b.base], [ca, cb, cc], n_fill=wide, focus=(1, 1)))
    # mode 1: the tie at 3 is a column without a MapPoint
    b = Bits(_seed("bow1_no_mp"))
    cs = [b.at(3), b.at(3), b.at(4)]
    for m, rr in enumerate(_ratio_pair(0.75, operator.lt)):
        out.append(_bow("bow1_no_mp", m, 1, rr, [b.base], cs, cols_mp=[1, 0, 1]))
        out.append(_bow("bow1_wide_no_mp", m, 1, rr, [b.base], cs, cols_mp=[1, 0, 1], n_fill=wide))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchForInitialization: every F1 feature at octave 0 with its window (size 10) centred on (100, 100); F2's keypoints at
# (100 + 0.25 * (k + 1), 100), all in the window, in index order
INIT_WINDOW = 10


def _init(cls, member, ratio, qdesc, kdesc, focus):
    n1, n2 = len(qdesc), len(kdesc)
    F1 = FrameView(mvKeysUn=G._keys([(20.0 + 3.0 * i, 400.0) for i in range(n1)]), mDescriptors=np.stack(qdesc),
                   mvScaleFactors=G.SCALE, bounds=G.BOUNDS)
    F2 = FrameView(mvKeysUn=G._keys([(100.0 + 0.25 * (k + 1), 100.0) for k in range(n2)]), mDescriptors=np.stack(kdesc),
                   mvScaleFactors=G.SCALE, bounds=G.BOUNDS)
    prev = np.tile(np.array([[100.0, 100.0]], np.float32), (n1, 1))
    return dict(cls=cls, member=member, kind="init", F1=F1, F2=F2, prev=prev, window=INIT_WINDOW, ratio=float(ratio), focus=focus)


def _pairs_init():
    out = []
    b = Bits(_seed("init_th"))
    far = b.at(200)
    for m, d in enumerate((TH_LOW, TH_LOW + 1)):
        out.append(_init("init_th", m, 0.9, [b.base], [Bits(_seed("init_th") + d, b.base).at(d), far], (0, 0)))
    for cls, r in (("init_ratio_06", 0.6), ("init_ratio_08", 0.8), ("init_ratio_075", 0.75)):
        d1, d2 = (3, 4) if r == 0.75 else first_separating(r, operator.lt)
        b = Bits(_seed(cls))
        ks = [b.at(d1), b.at(d2)]
        for m, rr in enumerate(_ratio_pair(r, operator.lt)):
            out.append(dict(_init(cls, m, rr, [b.base], ks, (0, 0)), dists=(d1, d2)))
    # a single-candidate window: bestDist2 = INT_MAX
    for cls, r in (("init_no_second_09", 0.9), ("init_no_second_10", 1.0)):
        b = Bits(_seed(cls))
        for m, d in enumerate((TH_LOW, TH_LOW + 1)):
            out.append(dict(_init(cls, m, r, [b.base], [Bits(_seed(cls) + d, b.base).at(d)], (0, 0)), dists=(d, None)))
    b = Bits(_seed("init_no_second_int_max"))
    r0 = f32(25.0 * 2.0 ** -30)                                  # 2^31 * r0 == 50
    c0 = b.at(TH_LOW)
    for m, rr in enumerate((G.step(r0, 1), r0)):
        out.append(dict(_init("init_no_second_int_max", m, rr, [b.base], [c0], (0, 0)), dists=(TH_LOW, None)))
    # exclusion served by the prefix: query A (F1 0) takes fa at 5; query B (F1 1) sees fa at 5 (equal: excluded, B takes fb at
    # 12 against fc at 20) or at 4 (smaller: B takes fa, A loses it)
    for m, da in enumerate((5, 4)):
        b = Bits(_seed("init_excl_prefix"))
        fa = b.at(da)
        A = b.at(5, base=fa)
        fb, fc = b.at(12), b.at(20)
        out.append(_init("init_excl_prefix", m, 0.75, [A, b.base], [fa, fb, fc], (1, 1)))
    # exclusion in the window walk: queries A_0..A_7 take f_0..f_7 at 5; B's window holds those eight (B's INIT_K nearest) and fb,
    # fc: with all eight excluded (equal distances) the prefix yields nothing and the walk takes fb; with f_0 at 4, f_0
    for m, d0 in enumerate((5, 4)):
        b = Bits(_seed("init_excl_walk"))
        fs = [b.at(d0 if k == 0 else 5) for k in range(INIT_K)]
        As = [b.at(5, base=f) for f in fs]
        fb, fc = b.at(12), b.at(20)
        out.append(_init("init_excl_walk", m, 0.75, As + [b.base], fs + [fb, fc], (INIT_K, INIT_K)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# SearchForTriangulation with proj_geometry's F12 (the epipolar line of kp1 is its row) and epipole (445, 302.5); kp1 at
# (200, 50), both keyframes monocular, no MapPoints
TRI_GOOD = [(300.0, 50.0), (320.0, 50.0)]                # on the line, far from the epipole
TRI_NEAR_EPIPOLE = (445.0, 305.0)                         # (ex - x)^2 + (ey - y)^2 = 6.25 < 100
TRI_OFF_LINE = (300.0, 80.0)                              # dsqr = 900


def _tri(cls, member, q, cdesc, cxy, focus):
    n2 = len(cdesc)
    mk = lambda xy, d: KeyFrameView(mvKeysUn=G._keys(xy), mDescriptors=np.stack(d), mFeatVec=FeatureVector.from_nodes(np.zeros(len(d), np.int64)),
                                    has_mp=np.zeros(len(d), np.uint8), mvuRight=np.full(len(d), -1.0, np.float32),
                                    mvScaleFactors=G.SCALE, mvLevelSigma2=G.SIGMA2)
    return dict(cls=cls, member=member, kind="tri", kf1=mk([(200.0, 50.0)], [q]), kf2=mk(cxy, cdesc), F12=G.TRI_F12, Ow1=G.TRI_OW1,
                T2w=G.TRI_T2W, ep=G.epipole(), focus=focus)


def _pairs_tri():
    out = []
    for m, d in enumerate((TH_LOW, TH_LOW + 1)):
        b = Bits(_seed("tri_th"))
        out.append(_tri("tri_th", m, b.base, [b.at(d)], TRI_GOOD[:1], (0, 0)))
    for cls, bad in (("tri_order_epipole", TRI_NEAR_EPIPOLE), ("tri_order_epiline", TRI_OFF_LINE)):
        for m, d in enumerate((TH_LOW, TH_LOW + 1)):
            b = Bits(_seed(cls))
            out.append(_tri(cls, m, b.base, [b.at(10), b.at(d)], [bad, TRI_GOOD[0]], (0, 1)))
    for m, d in enumerate((20, 21)):
        b = Bits(_seed("tri_equal_later"))
        out.append(_tri("tri_equal_later", m, b.base, [b.at(20), b.at(d)], TRI_GOOD, (0, 1)))
    return out


@functools.lru_cache(maxsize=None)
def cases():
    """Every case; world-point cases (no 'kind') are run through every world-point method."""
    return tuple(_pairs_world() + _pairs_proj() + _pairs_bow() + _pairs_init() + _pairs_tri())


def methods(c):
    return (c["kind"],) if "kind" in c else WORLD_METHODS


# ---------------------------------------------------------------------------------------------------------------------------
# the port and the verbatim reference, in comparable form
S12_ID, S21_ID = G.S12_ID, G.S21_ID


def run_port(O, c, method):
    if method in ("local", "last", "sim3proj", "fuse", "fuse_kf", "proj", "tri"):
        if method == "tri":
            return O.port_search_for_triangulation(c["kf1"], c["kf2"], c["F12"], c["ep"], False, False)
        return G.run_port(O, c, method)
    if method == "kf":
        return O.port_search_by_projection_kf(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], c["th"], c["orb_dist"], False)
    if method == "sim3":
        return O.port_search_by_sim3(c["F"], c["F"], c["P"], c["P2"], c["Tcw"], c["Tcw"], S12_ID, S21_ID, c["K"], c["th"])
    if method == "bow0":
        return O.port_search_by_bow(c["kf"], c["F"], c["ratio"], False)
    if method == "bow1":
        return O.port_search_by_bow_kf(c["kf"], c["F"], c["ratio"], False)
    if method == "init":
        return O.port_search_for_initialization(c["F1"], c["F2"], c["prev"], c["window"], c["ratio"], False)
    raise ValueError(method)


def run_ref(O, c, method):
    if method in ("local", "last", "sim3proj", "fuse", "fuse_kf", "proj"):
        return G.run_ref(O, c, method)
    if method == "tri":
        return O.ref_search_for_triangulation(c["kf1"], c["kf2"], c["F12"], c["Ow1"], c["T2w"], G.K_CAM, False, False)
    if method == "kf":
        return O.ref_search_by_projection_kf(c["F"], c["P"], c["Tcw"], c["K"], c["th"], c["orb_dist"], False)
    if method == "sim3":
        return O.ref_search_by_sim3(c["F"], c["F"], c["P"], c["P2"], c["Tcw"], c["Tcw"], 1.0, np.eye(3, dtype=np.float32),
                                    np.zeros(3, np.float32), c["K"], c["th"])
    if method == "bow0":
        return O.ref_search_by_bow(c["kf"], c["F"], c["ratio"], False)
    if method == "bow1":
        return O.ref_search_by_bow_kf(c["kf"], c["F"], c["ratio"], False)
    if method == "init":
        return O.ref_search_for_initialization(c["F1"], c["F2"], c["prev"], c["window"], c["ratio"], False)
    raise ValueError(method)


def ref_pairs(O, c, method):
    """The verbatim build's matches as a set of (query, feature): (MapPoint, keypoint) for the projection searches and Fuse,
    (KF1, KF2 feature) for SearchBySim3, (row, column) for SearchByBoW, (F1, F2) / (KF1, KF2) feature for the rest."""
    r = run_ref(O, c, "local" if method == "local_match" else method)
    if method in ("local", "local_match"):
        owner = r[1][1]
    elif method in ("last", "kf", "sim3proj", "proj"):
        owner = r[1]
    elif method in ("fuse", "fuse_kf", "sim3", "init", "bow1"):
        return {(i, int(f)) for i, f in enumerate(r[1]) if f >= 0}
    elif method == "bow0":
        return {(int(k), j) for j, k in enumerate(r[1]) if k >= 0}
    elif method == "tri":
        return {(int(a), int(b)) for a, b in r}
    else:
        raise ValueError(method)
    return {(int(q), k) for k, q in enumerate(owner) if q >= 0}


def decided(O, c):
    """The reference's decision on case c: does the class's focus pair (query, feature) match?"""
    method = c.get("kind") or DECIDER[c["cls"]]
    return tuple(c["focus"]) in ref_pairs(O, c, method)
