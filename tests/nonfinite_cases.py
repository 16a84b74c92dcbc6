"""Matcher inputs on the values where the reference's bits come from x86's float-to-int conversion rather than from arithmetic.
Test tooling: tests/test_oracle_nonfinite.py pins the port to the verbatim Frame.cc / ORBmatcher.cc on every case and checks that
the verbatim build decides the two members of every pair differently; tests/test_gpu_nonfinite.py pins the CUDA library to the
port.  Nothing in this module calls the CUDA library.

On x86, (int)f of NaN, +-inf or |f| >= 2^31 is cvttss2si's INT_MIN.  The device's cvt.rzi.s32.f32 saturates instead (+inf and
large values INT_MAX, -inf INT_MIN, NaN 0); the kernels restate the x86 result with x86_int (match_rules.cuh) where it decides
something.  A pair is two cases that differ in one input:

  grid_*      a keypoint coordinate NaN against the finite value that puts the key into grid column / row 0, which is where the
              device conversion of NaN would put it (Frame::PosInGrid: the reference drops the NaN key)
  radius_*    a window edge (x - mnMinX + r)*invW on 2^31 against one float step below it, reached through th, windowSize against
              narrow frame bounds, a host view's mvScaleFactors, and the Fuse / SearchBySim3 radii (GetFeaturesInArea: the
              reference's nMaxCellX is INT_MIN there, so the window is empty; one step below it is the whole frame)
  nan_centre_*  a query centre NaN against a finite one (GetFeaturesInArea: the reference's window is empty)

An infinite input against the largest finite float decides no gate differently: both are past 2^31 after the scaling by invW
(a key or a centre at FLT_MAX is as far outside every window as one at +inf, and a radius of FLT_MAX empties the window as
+inf does), so such pairs are not listed.  A NaN centre or a NaN key can never pass GetFeaturesInArea's |dx| < r, so which cells
the window walks decides no match: the nan_centre_* classes pin the result, and the grid is compared cell by cell through
borb_debug_frame_read, where a NaN key in the wrong cell shows.

The other float inputs of the searches reach no conversion of their own.  A NaN in mvuRight, in a MapPoint's normal or distance
bounds, in mvLevelSigma2 / mvInvLevelSigma2 or in a keyframe keypoint of SearchForTriangulation only enters IEEE comparisons
(ur > 0, viewCos < limit, dist < 0.8f*min, e2*invSigma2 > 5.99, dsqr < 3.84*sigma2, ...), which x86 and the device decide alike;
a NaN or infinite pose or world position becomes a NaN / infinite projection, i.e. a window centre (nan_centre_*, or a far edge
as in radius_*) and the same comparisons, plus PredictScale's ratio, whose conversion k_match.cu restates for every value; a NaN
mvScaleFactors entry makes the radius NaN, whose window edges are NaN like a NaN centre's.  A NaN keypoint angle reaches only the
rotation histogram, where the reference is undefined (NOT_COVERED).

INVENTORY lists every float-to-int conversion of the device code with the domain of its input and the class that covers it,
or the reason no NaN, infinite or int-overflowing value reaches it."""
import functools
import os
import re

import numpy as np

from orb_slam2_b200.matcher import FrameView
from tests import proj_geometry as G

f32 = np.float32
INT_MIN = -2 ** 31
TWO31 = f32(2.0 ** 31)
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "orb_slam2_b200", "csrc")


def x86_int(v):
    """(int)v as cvttss2si computes it: truncation, and INT_MIN for NaN, +-inf and every value outside [-2^31, 2^31)."""
    v = f32(v)
    return int(v) if (v >= -TWO31 and v < TWO31) else INT_MIN


def grid_cell(bounds, x, y):
    """Frame::PosInGrid (Frame.cc:384-395) with the x86 conversion: (col, row), or None when the key is in no cell."""
    minX, minY, maxX, maxY = [f32(b) for b in bounds]
    invW, invH = f32(f32(64) / f32(maxX - minX)), f32(f32(48) / f32(maxY - minY))
    rnd = lambda t: np.copysign(np.floor(abs(np.float64(t)) + 0.5), t) if np.isfinite(t) else t      # std::round of a float
    with np.errstate(invalid="ignore"):
        cx = x86_int(rnd(f32(f32(f32(x) - minX) * invW)))
        cy = x86_int(rnd(f32(f32(f32(y) - minY) * invH)))
    return (cx, cy) if 0 <= cx < 64 and 0 <= cy < 48 else None


def area_window(bounds, x, y, r):
    """GetFeaturesInArea's cell window (Frame.cc:332-344) with the x86 conversion: (c0x, c1x, c0y, c1y), or None when empty."""
    minX, minY, maxX, maxY = [f32(b) for b in bounds]
    invW, invH = f32(f32(64) / f32(maxX - minX)), f32(f32(48) / f32(maxY - minY))
    x, y, r = f32(x), f32(y), f32(r)
    with np.errstate(invalid="ignore", over="ignore"):
        c0x = max(0, x86_int(np.floor(f32(f32(f32(x - minX) - r) * invW))))
        c1x = min(63, x86_int(np.ceil(f32(f32(f32(x - minX) + r) * invW))))
        c0y = max(0, x86_int(np.floor(f32(f32(f32(y - minY) - r) * invH))))
        c1y = min(47, x86_int(np.ceil(f32(f32(f32(y - minY) + r) * invH))))
    return None if (c0x >= 64 or c1x < 0 or c0y >= 48 or c1y < 0) else (c0x, c1x, c0y, c1y)


# coverage classes -> the kernel line each exists for
CLASSES = {
    "grid_nan_x": "k_frame.cu:94 PosInGrid's round((x - mnMinX)*invW): NaN is INT_MIN, the key is in no cell (device: column 0)",
    "grid_nan_y": "k_frame.cu:95 PosInGrid's round((y - mnMinY)*invH): NaN is INT_MIN, the key is in no cell (device: row 0)",
    "radius_th_proj": "k_proj.cu:42 ceil((x - minX + r)*invW) on 2^31, r = 4*th in SearchByProjection(F, vpMapPoints, th)",
    "radius_scale_proj": "k_proj.cu:42 the same edge through a host view's mvScaleFactors[level] (th 1)",
    "radius_window_init": "k_proj.cu:42 the same edge in SearchForInitialization: windowSize 100 against mnMaxX - mnMinX of ~3e-6",
    "radius_th_fuse": "k_proj.cu:42 the same edge through th*mvScaleFactors[level] in Fuse(pKF, Scw)",
    "radius_th_fuse_kf": "k_proj.cu:42 the same edge through th*mvScaleFactors[level] in Fuse(pKF, vpMapPoints)",
    "radius_th_sim3": "k_proj.cu:42 the same edge through th*mvScaleFactors[level] in both directions of SearchBySim3",
    "radius_th_kf": "k_proj.cu:42 the same edge through th*mvScaleFactors[level] in SearchByProjection(CurrentFrame, KeyFrame)",
    "radius_th_last": "k_proj.cu:42 the same edge through th*mvScaleFactors[nLastOctave] in SearchByProjection(CurrentFrame, LastFrame)",
    # A NaN centre fails area_passes' |dx| < r (k_proj.cu:57) for every key, so these pin the search's RESULT (no match), not the
    # window: a saturating conversion in area_window walks column / row 0 instead of nothing and finds the same nothing
    "nan_centre_proj_x": "k_proj.cu:41-42,57 a NaN mTrackProjX finds no match (the result only; see above)",
    "nan_centre_proj_y": "k_proj.cu:43-44,57 a NaN mTrackProjY finds no match (the result only; see above)",
    "nan_centre_init": "k_proj.cu:41-44,57 a NaN vbPrevMatched[i] in SearchForInitialization finds no match (the result only)",
}

# gates where the reference itself is undefined on a non-finite input, each with its argument
NOT_COVERED = {
    "rot_bin_nan": "match_rules.cuh:38 rot_bin of a NaN or infinite angle difference: the reference's round(NaN) is INT_MIN, "
                   "and rotHist[INT_MIN].push_back (ORBmatcher.cc:246) writes outside the histogram; no result is defined",
}


# ---------------------------------------------------------------------------------------------------------------------------
# pairs
def bisect_window(window_of, lo, hi):
    """(kept, dropped): adjacent float32 values of the free input between lo and hi, the first giving a window and the second
    none (window_of is monotone on [lo, hi])."""
    a, b = G.bisect(lambda p: window_of(p) is None, f32(lo), f32(hi))
    assert window_of(a) is not None and window_of(b) is None
    return a, b


def _grid_case(cls, member, v):
    k = G._keys([(300.0, 200.0), (0.0, 100.0), (500.0, 400.0), (10.0, 0.0)])
    k["x"][1] = v if cls == "grid_nan_x" else 0.0
    k["y"][3] = v if cls == "grid_nan_y" else 0.0
    desc = G._desc(len(cls) + 5, len(k))
    F = FrameView(mvKeysUn=k, mDescriptors=desc, mvScaleFactors=G.SCALE, bounds=G.BOUNDS)
    return dict(cls=cls, member=member, kind="grid", F=F, key=1 if cls == "grid_nan_x" else 3)


def _pairs_grid():
    return [_grid_case(cls, m, v) for cls in ("grid_nan_x", "grid_nan_y") for m, v in enumerate((f32(0.0), f32(np.nan)))]


Q0 = (100.0, 100.0)                   # the query of the proj_* cases; its key 0 lies at (101, 100)


def _pairs_proj():
    out = []
    # rs = 4*th (mTrackViewCos 0.9, level 0, scale 1)
    a, b = bisect_window(lambda th: area_window(G.BOUNDS, *Q0, f32(f32(4.0) * th)), 1e8, 1e11)
    for m, th in enumerate((a, b)):
        out.append(G._proj_case("radius_th_proj", m, (101.0, 100.0), th=float(th)))
    # th 1: rs = 4*mvScaleFactors[0]
    a, b = bisect_window(lambda s: area_window(G.BOUNDS, *Q0, f32(f32(4.0) * s)), 1e8, 1e11)
    for m, s in enumerate((a, b)):
        c = G._proj_case("radius_scale_proj", m, (101.0, 100.0), th=1.0)
        sf = G.SCALE.copy(); sf[0] = s
        c["F"] = FrameView(c["F"].mvKeysUn, c["F"].mDescriptors, sf, c["F"].bounds, c["F"].mvuRight)
        out.append(c)
    for cls, q in (("nan_centre_proj_x", (np.nan, 100.0)), ("nan_centre_proj_y", (100.0, np.nan))):
        for m, q0 in enumerate((Q0, q)):
            out.append(G._proj_case(cls, m, (101.0, 100.0), q0=q0))
    return out


INIT_WINDOW = 100


def _init_case(cls, member, max_x, prev0):
    """SearchForInitialization: F1 feature 0 (octave 0) searches around prev0 in F2, whose feature 0 has its descriptor at
    (0, 100); F2's bounds are (0, 0, max_x, 480)."""
    d = G._desc(len(cls) + 29, 2)
    k1 = G._keys([(5.0, 100.0), (9.0, 300.0)])
    k2 = G._keys([(0.0, 100.0)])
    F1 = FrameView(mvKeysUn=k1, mDescriptors=d, mvScaleFactors=G.SCALE, bounds=G.BOUNDS)
    F2 = FrameView(mvKeysUn=k2, mDescriptors=d[:1].copy(), mvScaleFactors=G.SCALE, bounds=(0.0, 0.0, float(max_x), 480.0))
    prev = np.array([prev0, (9.0, 300.0)], np.float32)
    return dict(cls=cls, member=member, kind="init", F1=F1, F2=F2, prev=prev, window=INIT_WINDOW)


def _pairs_init():
    out = []
    # invW = 64/max_x: the window edge (0 + 100)*invW crosses 2^31 at max_x ~ 3e-6; a larger max_x gives a finite edge
    b, a = G.bisect(lambda mx: area_window((0.0, 0.0, mx, 480.0), 0.0, 100.0, INIT_WINDOW) is None, f32(1e-6), f32(1e-5))
    assert area_window((0.0, 0.0, a, 480.0), 0.0, 100.0, INIT_WINDOW) is not None
    for m, mx in enumerate((a, b)):
        out.append(_init_case("radius_window_init", m, mx, (0.0, 100.0)))
    for m, p in enumerate(((1.0, 100.0), (np.nan, 100.0))):
        out.append(_init_case("nan_centre_init", m, 640.0, p))
    return out


def _pairs_world_th():
    """Fuse, SearchBySim3 and the KeyFrame / LastFrame overloads of SearchByProjection on proj_geometry's world-point case: the
    boundary point projects to (445, 302.5) at level 0 (scale 1), so its radius is th itself and the x edge crosses 2^31 first."""
    out = []
    a, b = bisect_window(lambda th: area_window(G.BOUNDS, G.U0, G.V0, th), 1e8, 1e11)
    for cls, kind in (("radius_th_fuse", "fuse"), ("radius_th_fuse_kf", "fuse_kf"), ("radius_th_sim3", "sim3"), ("radius_th_kf", "kf"),
                      ("radius_th_last", "last")):
        for m, th in enumerate((a, b)):
            out.append(dict(G._world_case(cls, m, G.U0_CAM, (G.U0 - 0.5, G.V0)), th=float(th), world_method=kind))
    return out


# borb_frames_from_extractor under a calibration with fx == 0 (or fy == 0): 1/fx is +inf, so UndistortKeyPoints' normalised
# coordinates are +-inf, the distortion factor 1/(1 + k1*r^2) is 0 and inf*0 makes every key NaN (the image bounds too).  The
# reference's PosInGrid then drops every key; the device conversion would put all of them into cell (0, 0).
NAN_CALIBRATIONS = (((0.0, 500.0, 320.0, 240.0), (0.1, 0.0, 0.0, 0.0, 0.0)), ((500.0, 0.0, 320.0, 240.0), (0.1, 0.0, 0.0, 0.0, 0.0)))
UNDISTORT_IMAGE = (3, 640, 480)                 # synth.mono_frame seed, width, height


def undistort_image():
    from orb_slam2_b200 import synth
    seed, w, h = UNDISTORT_IMAGE
    return synth.mono_frame(seed, 0, 0, w, h)


@functools.lru_cache(maxsize=None)
def cases():
    return tuple(_pairs_grid() + _pairs_proj() + _pairs_init() + _pairs_world_th())


def methods(c):
    if "world_method" in c:
        return (c["world_method"],)
    return (c["kind"],)


# ---------------------------------------------------------------------------------------------------------------------------
# the port and the verbatim reference
def run_port(O, c, method):
    if method == "grid":
        return O.port_assign_grid(c["F"].mvKeysUn, c["F"].bounds)
    if method == "init":
        return O.port_search_for_initialization(c["F1"], c["F2"], c["prev"], c["window"], 0.9, False)
    return G.run_port(O, c, method)


def run_ref(O, c, method):
    if method == "grid":
        return O.ref_assign_grid(c["F"].mvKeysUn, c["F"].bounds)
    if method == "init":
        return O.ref_search_for_initialization(c["F1"], c["F2"], c["prev"], c["window"], 0.9, False)
    return G.run_ref(O, c, method)


def decided(O, c):
    """The reference's decision on the pair's input: True when key 0 / query 0 gets through (the grid: the key is in a cell)."""
    method = methods(c)[0]
    r = run_ref(O, c, method)
    if method == "grid":
        return bool(c["key"] in r[1][:r[0][-1]].tolist())
    if method == "init":
        return bool(r[1][0] == 0)
    if method in ("fuse", "fuse_kf", "sim3"):
        return bool(r[1][0] == 0)                     # point 0's best feature is keypoint 0
    return bool((r[1] == 0).any())                    # some feature went to query 0


# ---------------------------------------------------------------------------------------------------------------------------
# inventory of the device's float-to-int conversions
# A conversion is a call of x86_int, a __float2int / __float2uint intrinsic, or an explicit integer cast of a float operand: a float
# rounding function, a float intrinsic, an identifier declared float somewhere in the same file, or a keypoint's float field.  The
# identifier rule is by name, so an integer that shares its name with a float of the same file is listed too, as an integer.  Rows are keyed by (file, the source line without its comment and surrounding blanks).
_CAST = r"\((?:int|int32_t|short|unsigned|uint32_t|uint16_t|uint8_t|long|int64_t)\)\s*"
_FLOAT_CALL = r"(?:floorf|ceilf|roundf|rintf|truncf|__f(?:add|sub|mul|div|sqrt|rcp)_r[nzud])\s*\("


def _float_names(src):
    names = set()
    for decl in re.finditer(r"\bfloat\s+([^;{)]*)", src):
        for part in re.split(r",(?![^(]*\))", decl.group(1)):
            m = re.match(r"\s*&?\s*(\w+)", part)
            if m:
                names.add(m.group(1))
    return names


def _paren(code, i):
    """The text inside the parentheses that open at code[i], or None when they do not close on the line."""
    depth = 0
    for j in range(i, len(code)):
        depth += {"(": 1, ")": -1}.get(code[j], 0)
        if depth == 0:
            return code[i + 1:j]
    return None


def scan_conversions():
    """{(file, line text): [line numbers]} of every float-to-int conversion in csrc/k_*.cu and match_rules.cuh."""
    found = {}
    files = sorted(f for f in os.listdir(CSRC) if (f.startswith("k_") and f.endswith(".cu")) or f == "match_rules.cuh")
    for fn in files:
        src = open(os.path.join(CSRC, fn)).read()
        floats = _float_names(src)
        keypoints = set(re.findall(r"borb_keypoint&?\s+(\w+)\s*=", src))
        var = "|".join(sorted(floats)) or "(?!)"
        kp = "|".join(sorted(keypoints)) or "(?!)"
        float_operand = rf"{_FLOAT_CALL}|(?:{var})\b(?!\s*[\(\[.])|(?:{kp})\.(?:x|y|angle|size|response)\b"
        pat = re.compile(rf"\bx86_int\s*\(|__float2u?(?:int|ll)_r[nzud]\s*\(|{_CAST}(?:{float_operand})"
                         rf"|\b(?:int|int32_t|short|unsigned|uint32_t)\s+\w+\s*=\s*{_FLOAT_CALL}")
        # a cast of a parenthesised operand: a conversion when the operand holds a float literal, a float or double cast, a float
        # call or a keypoint's float field (identifiers are left out here: packed integer keys share names with floats)
        inner_float = re.compile(rf"\d\.\d*|\.\d|\((?:float|double)\)|{_FLOAT_CALL}|(?:{kp})\.(?:x|y|angle|size|response)\b")
        cast_paren = re.compile(rf"{_CAST}(?=\()")
        for i, line in enumerate(src.splitlines(), 1):
            code = line.split("//")[0].strip()
            hit = bool(code and pat.search(code))
            for m in cast_paren.finditer(code) if code and not hit else ():
                inner = _paren(code, m.end())
                if inner is not None and inner_float.search(inner):
                    hit = True
                    break
            if hit:
                found.setdefault((fn, code), []).append(i)
    return found


INVENTORY = [
    # (file, line text, input domain, class or reason no non-finite / overflowing value reaches it)
    ("k_describe.cu", "const int r = __float2int_rn(__fadd_rn(__fmul_rn(x, b), __fmul_rn(y, a)));",
     "a pattern tap rotated by the keypoint's cos / sin", "finite: taps are small integers and cos / sin come from the finite IC_Angle moments"),
    ("k_describe.cu", "const int q = __float2int_rn(__fsub_rn(__fmul_rn(x, a), __fmul_rn(y, b)));",
     "the other coordinate of the same tap", "finite, as above"),
    ("k_describe.cu", "const int bin = min((int)(angle * (float)(BRIEF_BINS / 360.0)), BRIEF_BINS - 1);",
     "the keypoint's orientation in degrees, scaled to the rBRIEF bin", "finite: IC_Angle's fastAtan2 of finite moments lies in [0, 360]"),
    ("k_frame.cu", "const int v = (int)kp.y, u = (int)kp.x;",
     "the DISTORTED extractor keypoint of ComputeStereoFromRGBD", "finite: extractor keys lie inside the image"),
    ("k_frame.cu", "const int px = x86_int(roundf(__fmul_rn(__fsub_rn(J.keys[i].x, J.min_x), J.inv_w)));",
     "undistorted / host-view key x", "grid_nan_x"),
    ("k_frame.cu", "const int py = x86_int(roundf(__fmul_rn(__fsub_rn(J.keys[i].y, J.min_y), J.inv_h)));",
     "undistorted / host-view key y", "grid_nan_y"),
    ("k_match.cu", "bestKey = min(bestKey, ((unsigned)dist << 16) | (unsigned)(0xFFFF - (p - ts0)));",
     "int Hamming distance and list position", "integer operands (names shared with floats of the file)"),
    ("k_match.cu", "const unsigned key = ((unsigned)dist << 16) | (unsigned)p;",
     "int Hamming distance and list position", "integer operands (names shared with floats of the file)"),
    ("k_match.cu", "const int k = (int)(0.5 * (double)(N - 1));",
     "half the observation count minus one, in double", "finite: N is a positive int count"),
    ("k_match.cu", "nScale = q >= 2147483648.f || !(q == q) ? 0 : (q <= -2147483648.f ? 0 : (int)q);",
     "PredictScale's ceil(log(ratio)/log(sf))", "restated for every value (proj_geometry predict_scale_ratio_inf, camera_centre)"),
    ("k_proj.cu", "c0x = max(0, x86_int(floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, A.minX), rs), A.invW))));",
     "query x, radius, frame bounds", "nan_centre_proj_x; radius_* (the near edge clamps to 0 on both sides)"),
    ("k_proj.cu", "c1x = min(GRID_COLS - 1, x86_int(ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, A.minX), rs), A.invW))));",
     "query x, radius, frame bounds", "radius_*; nan_centre_proj_x"),
    ("k_proj.cu", "c0y = max(0, x86_int(floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, A.minY), rs), A.invH))));",
     "query y, radius, frame bounds", "nan_centre_proj_y"),
    ("k_proj.cu", "c1y = min(GRID_ROWS - 1, x86_int(ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, A.minY), rs), A.invH))));",
     "query y, radius, frame bounds", "nan_centre_proj_y; radius_* (the y edge is below 2^31 where the x edge crosses it)"),
    ("k_pyramid.cu", "const int sx = mx == mx ? __float2int_rn(mx) : INT_MIN, sy = my == my ? __float2int_rn(my) : INT_MIN;",
     "rectification map entries", "NaN guarded in place (cvRound's INT_MIN); tests/test_gpu_frame_input.py"),
    ("k_quadtree.cu", "const int r = (int)__fdiv_rn((float)(xys_x(x) - MIN_BORDER), hX);",
     "a FAST corner's column over the cell width", "finite: integer pixel coordinates over a positive width"),
    ("k_quadtree.cu", "v.box[0][j] = make_short4((short)(int)__fmul_rn(hX, (float)i), (short)(int)__fmul_rn(hX, (float)(i + 1)), 0,",
     "node edges of the initial quadtree split", "finite: cell width times a small integer"),
    ("k_stereo.cu", "const int maxr = (int)ceilf(__fadd_rn(kr.y, r)), minr = (int)floorf(__fsub_rn(kr.y, r));",
     "right extractor key y +- 2*scale", "finite: takes only extractor keys"),
    ("k_stereo.cu", "const int row = (int)vL;", "left extractor key y", "finite: takes only extractor keys"),
    ("k_stereo.cu", "const int scaleduL = (int)roundf(__fmul_rn(kp.x, sf));", "left extractor key x at its level", "finite: extractor keys"),
    ("k_stereo.cu", "const int scaledvL = (int)roundf(__fmul_rn(kp.y, sf));", "left extractor key y at its level", "finite: extractor keys"),
    ("k_stereo.cu", "const int scaleduR0 = (int)roundf(__fmul_rn(uR0, sf));", "matched right key x at its level", "finite: extractor keys"),
    ("k_stereo.cu", "const int band = 2 * (int)ceilf(2.0f * g.lv[g.nlevels - 1].scale) + 3;",
     "the top level's scale factor", "finite: the extractor refuses scale factors that are not finite and above 1"),
    ("match_rules.cuh", "int bin = (int)roundf(__fmul_rn(rot, 1.0f / HISTO_LENGTH));", "angle difference in degrees",
     "finite for every defined input; see NOT_COVERED rot_bin_nan"),
    ("match_rules.cuh", "__device__ __forceinline__ int x86_int(float v) { return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }",
     "any float", "the x86 restatement itself: the cast runs only inside [-2^31, 2^31)"),
]
