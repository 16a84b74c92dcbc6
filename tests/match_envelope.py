"""Matcher inputs at the sizes where the CUDA kernels change behaviour, and a coverage report of which of those size-dependent
paths a case reaches.  Test tooling: tests/test_oracle_match_envelope.py pins the port to the verbatim ORBmatcher.cc on every
case, tests/test_gpu_match_envelope.py pins the CUDA library to the port.

The kernel constants are restated here (as tests/extract_geometry.py restates the extractor's), each next to the line it
exists for.  Nothing in this module calls the CUDA library."""
import functools

import numpy as np

from orb_slam2_b200.matcher import FrameView, LastFrameView, MapPointsView
from orb_slam2_b200._lib import KP_DTYPE
from tests import match_fixtures as mf

MATCH_MAX_FEATURES = 8192          # borb_match.h:45 — 16-bit feature indices in candidate entries, grid keys and claim arrays
WAVE = 1024                        # k_proj.cu:414,427 — queries per wave of proj_resolve_kernel at n_mp > 512
RES_K = 4                          # k_proj.cu:34 — list entries per query staged in shared memory; later ones come from global
SORT_CAP = 128                     # k_proj.cu:33 — longer candidate lists are resolved by a full scan in position order
BOW_JCAP = 1024                    # k_match.cu:332 — wider target nodes are evaluated directly (k_match.cu:424-434)
BOW_DCAP = 1024                    # k_match.cu:331 — distance-matrix entries per warp: nodes wider than BOW_DCAP / 2 take row chunks
GRID_COLS, GRID_ROWS = 64, 48      # borb_match.h:41
TH_HIGH, TH_LOW = 100, 50
KITTI, EUROC = (1242, 375), (752, 480)
K_CAM = (500.0, 500.0, 621.0, 187.5)

# coverage classes -> the kernel line each exists for
CLASSES = {
    "wave_after_first": "k_proj.cu:350 held bits committed by an earlier wave",
    "chain_depth_gt_32": "k_proj.cu:11-19 fixpoint of more than a warp's depth",
    "chain_depth_1024": "k_proj.cu:304-348 fixpoint of a full 1024-query chain",
    "pick_beyond_res_k": "k_proj.cu:311 sorted list read from global memory under contention",
    "pick_unsorted": "k_proj.cu:317-328 list longer than SORT_CAP resolved under contention",
    "last_two_events": "k_proj.cu:357,368-374 one feature with two LAST match events",
    "n8192_all_in_grid": "k_frame.cu:117-118 grid-sort tail writes cell_start[GRID_CELLS], reached through a host view or borb_frame_create",
    "n8192_all_in_grid_jobs": "k_frame.cu:117-118 the same tail, reached through frames_from_extractor",
    "init_8192": "k_proj.cu:524-526 16-bit matchedDist / owner / took arrays of init_replay at 8192 features",
    "keys_outside_grid": "k_frame.cu:94 keys outside the grid never enter it",
    "bow_node_gt_jcap": "k_match.cu:424-434 direct evaluation of a node wider than BOW_JCAP",
    "bow_row_chunks": "k_match.cu:386 a node split into several row chunks",
    "tie_min_proj": "k_proj.cu:131-157 (distance, position) order of tied minima",
    "tie_min_bow": "k_match.cu:435-436 warp_min over tied (distance, position) keys",
    "tie_min_tri": "k_match.cu:536 later-wins among tied distances",
    "tie_min_last": "k_proj.cu:131-157,314 first of tied minima in the LAST resolve",
    "tie_min_init": "k_proj.cu:495,561 prefix key (dist << 16) | e of init_prefix / init_replay, e the cell_idx position",
    "tie_min_argmin": "k_proj.cu:207 fuse_batch_kernel's first minimum behind Fuse and SearchBySim3",
    "tie_min_local": "k_proj.cu:131-157 tied minima of SearchLocalPoints' projection search",
    "tie_level_ratio": "k_proj.cu:337 bestLevel == bestLevel2 clause at a tie",
    "hist_boundary": "match_rules.cuh:47-48 max2 or max3 exactly 0.1 * max1",
}


def _f32(x):
    return np.float32(x)


def in_grid(keys, bounds):
    """Frame::PosInGrid (src/Frame.cc:382-393) in float32: True where the key lands in the 64 x 48 grid."""
    min_x, min_y, max_x, max_y = [_f32(b) for b in bounds]
    inv_w = _f32(GRID_COLS) / (max_x - min_x)
    inv_h = _f32(GRID_ROWS) / (max_y - min_y)
    px = np.float32(keys["x"] - min_x) * inv_w
    py = np.float32(keys["y"] - min_y) * inv_h
    px = np.where(px >= 0, np.floor(px + 0.5), np.ceil(px - 0.5))      # roundf: halves away from zero
    py = np.where(py >= 0, np.floor(py + 0.5), np.ceil(py - 0.5))
    return (px >= 0) & (px < GRID_COLS) & (py >= 0) & (py < GRID_ROWS)


# ---------------------------------------------------------------------------------------------------------------------------
# envelope frames: the natural extraction at 8192 features overshoots the quota by a few keypoints; host views keep exactly
# MATCH_MAX_FEATURES (or one more, for the refusals)
@functools.lru_cache(maxsize=None)
def _raw_views(oracle, shape, seed):
    return mf.two_views(oracle, seed, shape, nf=MATCH_MAX_FEATURES)


def envelope_views(oracle, shape=KITTI, seed=7, n=MATCH_MAX_FEATURES):
    v = dict(_raw_views(oracle, shape, seed))
    assert len(v["kl"]) >= n and len(v["kr"]) >= n, (len(v["kl"]), len(v["kr"]))
    for k in ("kl", "dl", "kr", "dr", "ur"):
        v[k] = v[k][:n]
    return v


def self_query(v, bounds=None, occupied_every=0):
    """Every feature of the left view queried at its own position, level and descriptor: each query's best candidate is its own
    feature, so a feature that the grid loses (or a 16-bit index that wraps) changes the result."""
    k = v["kl"]
    n = len(k)
    b = bounds if bounds is not None else (0.0, 0.0, float(v["w"]), float(v["h"]))
    occ = None
    if occupied_every:
        occ = np.zeros(n, np.uint8); occ[::occupied_every] = 1
    F = FrameView(mvKeysUn=k, mDescriptors=v["dl"], mvScaleFactors=v["scale"], bounds=b, mvuRight=v["ur"], occupied=occ)
    mps = MapPointsView(mTrackProjX=k["x"].astype(np.float32), mTrackProjY=k["y"].astype(np.float32),
                        mTrackProjXR=np.where(v["ur"] >= 0, v["ur"], k["x"] - 5.0).astype(np.float32), mnTrackScaleLevel=k["octave"].astype(np.int32),
                        mTrackViewCos=np.full(n, 0.9, np.float32), descriptors=v["dl"],
                        valid=np.ones(n, np.uint8), has_obs=(np.arange(n) % 9 != 0).astype(np.uint8))
    return F, mps


# ---------------------------------------------------------------------------------------------------------------------------
# contested query sets
def _ramp(rng, base, dists):
    bits = np.repeat(np.unpackbits(base)[None], len(dists), 0)
    for i, d in enumerate(dists):
        bits[i, rng.choice(256, int(d), replace=False)] ^= 1
    return np.packbits(bits, axis=1)


def _cell_centre(cx, cy, bounds):
    min_x, min_y, max_x, max_y = bounds
    return min_x + cx * (max_x - min_x) / GRID_COLS, min_y + cy * (max_y - min_y) / GRID_ROWS


def contested(seed, clusters, per_cluster, n_q, max_dist, no_obs_every=0, occ_frac=0.0, shape=KITTI):
    """A frame whose features sit in `clusters` small windows, each inside one grid cell (so list order = feature order).  In a
    cluster the descriptors are a distance ramp from the cluster's base descriptor, with ties inside every step and alternating
    octaves, so that the (distance, position) order is the feature order and the ratio test never meets two equal levels.
    Query q asks cluster q % clusters with the base descriptor: each claiming query takes the next free feature, and the claim
    chain is as deep as the number of claiming queries of a cluster in one wave.  Queries without observations match without
    claiming (the next query re-takes their feature); occupied features are held from the start."""
    rng = np.random.default_rng(seed)
    w, h = shape
    bounds = (0.0, 0.0, float(w), float(h))
    cw, ch = w / GRID_COLS, h / GRID_ROWS
    centres = [(cx, cy) for cy in range(4, GRID_ROWS - 4, 5) for cx in range(4, GRID_COLS - 4, 4)][:clusters]
    assert len(centres) == clusters
    n = clusters * per_cluster
    keys = np.zeros(n, KP_DTYPE)
    desc = np.zeros((n, 32), np.uint8)
    bases = rng.integers(0, 256, (clusters, 32), dtype=np.uint8)
    for c, (gx, gy) in enumerate(centres):
        x0, y0 = _cell_centre(gx, gy, bounds)
        s = slice(c * per_cluster, (c + 1) * per_cluster)
        keys["x"][s] = x0 + rng.uniform(-min(3.0, 0.4 * cw), min(3.0, 0.4 * cw), per_cluster)
        keys["y"][s] = y0 + rng.uniform(-min(3.0, 0.4 * ch), min(3.0, 0.4 * ch), per_cluster)
        desc[s] = _ramp(rng, bases[c], (np.arange(per_cluster) * max_dist) // per_cluster)
    keys["octave"] = np.arange(n) % 2
    keys["size"] = 31.0
    keys["response"] = 1.0
    keys["angle"] = rng.uniform(0, 360, n).astype(np.float32)
    scale = (np.float32(1.2) ** np.arange(8)).astype(np.float32)
    occ = (rng.random(n) < occ_frac).astype(np.uint8) if occ_frac else None
    F = FrameView(mvKeysUn=keys, mDescriptors=desc, mvScaleFactors=scale, bounds=bounds, occupied=occ)
    cl = np.arange(n_q) % clusters
    cx = np.array([_cell_centre(*centres[c], bounds)[0] for c in cl], np.float32)
    cy = np.array([_cell_centre(*centres[c], bounds)[1] for c in cl], np.float32)
    has_obs = np.ones(n_q, np.uint8)
    if no_obs_every:
        has_obs[no_obs_every - 1::no_obs_every] = 0
    mps = MapPointsView(mTrackProjX=cx, mTrackProjY=cy, mTrackProjXR=cx - 10.0, mnTrackScaleLevel=np.ones(n_q, np.int32),
                        mTrackViewCos=np.full(n_q, 0.9, np.float32), descriptors=bases[cl], valid=np.ones(n_q, np.uint8), has_obs=has_obs)
    # the LastFrame form of the same queries: identity pose, points at depth 10 on the rays through the cluster centres
    fx, fy, ccx, ccy = K_CAM
    z = np.float32(10.0)
    wp = np.stack([(cx - ccx) * z / fx, (cy - ccy) * z / fy, np.full(n_q, z)], 1).astype(np.float32)
    lk = np.zeros(n_q, KP_DTYPE)
    lk["x"], lk["y"], lk["octave"], lk["size"] = cx, cy, 1, 31.0
    lk["angle"] = rng.uniform(0, 360, n_q).astype(np.float32)
    Last = LastFrameView(mvKeysUn=lk, world_pos=wp, descriptors=bases[cl], valid=np.ones(n_q, np.uint8), has_obs=has_obs)
    return dict(F=F, mps=mps, Last=Last, cluster=cl, per_cluster=per_cluster)


def histogram_case(counts, seed=3, shape=KITTI):
    """SearchByProjection(CurrentFrame, LastFrame) with one isolated feature per query, identical descriptors, and rotations
    chosen per pair so that the rotation histogram has exactly the bin counts `counts` ({bin: count})."""
    rng = np.random.default_rng(seed)
    w, h = shape
    bounds = (0.0, 0.0, float(w), float(h))
    bins = np.concatenate([np.full(c, b) for b, c in counts.items()])
    n = len(bins)
    slots = [(gx, gy) for gy in range(3, GRID_ROWS - 3, 6) for gx in range(3, GRID_COLS - 3, 3)]
    assert n <= len(slots)
    keys = np.zeros(n, KP_DTYPE)
    keys["x"] = [_cell_centre(*slots[i], bounds)[0] for i in range(n)]
    keys["y"] = [_cell_centre(*slots[i], bounds)[1] for i in range(n)]
    keys["octave"], keys["size"], keys["response"] = 0, 31.0, 1.0
    keys["angle"] = rng.uniform(0, 360, n).astype(np.float32)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    scale = (np.float32(1.2) ** np.arange(8)).astype(np.float32)
    Cur = FrameView(mvKeysUn=keys, mDescriptors=desc, mvScaleFactors=scale, bounds=bounds)
    order = rng.permutation(n)                              # queries in an order unrelated to the features
    lk = keys[order].copy()
    lk["angle"] = np.mod(keys["angle"][order] + 30.0 * bins[order] + 5.0, 360.0).astype(np.float32)
    fx, fy, ccx, ccy = K_CAM
    z = np.float32(8.0)
    wp = np.stack([(lk["x"] - ccx) * z / fx, (lk["y"] - ccy) * z / fy, np.full(n, z)], 1).astype(np.float32)
    Last = LastFrameView(mvKeysUn=lk, world_pos=wp, descriptors=desc[order], valid=np.ones(n, np.uint8), has_obs=np.ones(n, np.uint8))
    return dict(F=Cur, Last=Last)


# ---------------------------------------------------------------------------------------------------------------------------
# tied descriptors
def tied_views(v, seed, frac=0.3):
    """Copies of the two views where a fraction of the keypoints hand their descriptor to their nearest neighbour, at the same
    octave for half of them and at another octave for the rest: ties at the minimum become common in every method."""
    rng = np.random.default_rng(seed)
    out = dict(v)
    for kk, dd in (("kl", "dl"), ("kr", "dr")):
        k = v[kk].copy(); d = v[dd].copy()
        xy = np.stack([k["x"], k["y"]], 1)
        for i in np.nonzero(rng.random(len(k)) < frac)[0]:
            d2 = ((xy - xy[i]) ** 2).sum(1); d2[i] = np.inf
            j = int(np.argmin(d2))
            d[j] = d[i]
            k["octave"][j] = k["octave"][i] if i % 2 == 0 else (k["octave"][i] + 1) % 8
        out[kk], out[dd] = k, d
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# the cases: name -> builder(oracle) -> dict(method=..., args...)
TRI_K2 = (525.0, 525.0, 319.5, 239.5)


def _proj(F, mps, th=3.0, ratio=0.8):
    return dict(method="proj", F=F, mps=mps, th=th, ratio=ratio)


def _last(Cur, Last, th=15.0, ori=True, Tcw=None, K=K_CAM):
    T = np.eye(4, dtype=np.float32)[:3] if Tcw is None else Tcw
    return dict(method="last", F=Cur, Last=Last, Tcw=T, K=K, th=th, ori=ori)


def _bow(voc, v, seed, levelsup, mp_frac=0.7, ratio=0.8):
    kf1, kf2 = mf.keyframe_views(v, voc, seed, levelsup=levelsup, mp_frac=mp_frac)
    return dict(method="bow", kf1=kf1, kf2=kf2, ratio=ratio, ori=True)


def _tri(O, voc, v, seed, levelsup, only_stereo=False):
    kf1, kf2 = mf.keyframe_views(v, voc, seed, levelsup=levelsup, mp_frac=0.3)
    Ow1, T2w = np.array([0.3, -0.05, -2.0], np.float32), np.eye(4, dtype=np.float32)[:3]
    # the epipole as the reference evaluates it where its build exists; the same float arithmetic restated otherwise
    ep = O.ref_epipole(Ow1, T2w, TRI_K2) if O.have_matchref() else _epipole(Ow1)
    return dict(method="tri", kf1=kf1, kf2=kf2, F12=mf.rectified_F12(seed), Ow1=Ow1, T2w=T2w, ep=ep, only_stereo=only_stereo, ori=True)


def _init(v, window=100, ratio=0.9):
    b = (0.0, 0.0, float(v["w"]), float(v["h"]))
    F1, F2 = FrameView(v["kl"], v["dl"], v["scale"], b), FrameView(v["kr"], v["dr"], v["scale"], b)
    prev = np.stack([v["kl"]["x"], v["kl"]["y"]], 1).astype(np.float32)
    return dict(method="init", F1=F1, F2=F2, prev=prev, window=window, ratio=ratio, ori=True)


def _fuse(O, v, seed, th=3.0):
    KF, P, Tcw, Ow, K, bf = mf.fuse_case(v, seed)
    Scw = (np.float32(1.4) * np.asarray(Tcw, np.float32)).astype(np.float32)         # the Sim3 overload: [s*R | s*t]
    if O.have_matchref():
        Ow = O.ref_camera_center(Tcw)
        Ts, Ows = O.ref_decompose_scw(Scw)
    else:
        Ts = (Scw / np.float32(1.4)).astype(np.float32)
        Ows = (-(Ts[:, :3].T @ Ts[:, 3])).astype(np.float32)
    return dict(method="fuse", KF=KF, P=P, Tcw=Tcw, Ow=Ow, Scw=Scw, Ts=Ts, Ows=Ows, K=K, bf=bf, th=th)


def _sim3(O, v, seed, th=7.5):
    KF1, KF2, P1, P2, T1w, T2w, S12, S21, K = mf.sim3_case(v, seed)
    a = 0.004
    s12, R12 = np.float32(1.03), np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], np.float32)
    t12 = np.array([0.4, 0.01, -0.02], np.float32)                  # the transform mf.sim3_case builds S12 / S21 from
    if O.have_matchref():
        S12, S21 = O.ref_sim3_mats(s12, R12, t12)
    return dict(method="sim3", KF1=KF1, KF2=KF2, P1=P1, P2=P2, T1w=T1w, T2w=T2w, S12=S12, S21=S21, s12=s12, R12=R12, t12=t12, K=K, th=th)


def _local(v, seed, th=3.0, ratio=0.8):
    F, P, Tcw, Ow, K = mf.world_points_case(v, seed)
    F = FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds, mvuRight=v["ur"], occupied=F.occupied)
    has_obs = (np.random.default_rng(seed).random(len(P.world_pos)) < 0.9).astype(np.uint8)
    return dict(method="local", F=F, P=P, Tcw=Tcw, Ow=Ow, K=K, has_obs=has_obs, th=th, ratio=ratio)


def _contest(ct, last, ori=True):
    c = _last(ct["F"], ct["Last"], ori=ori) if last else _proj(ct["F"], ct["mps"])
    c.update(cluster=ct["cluster"], per_cluster=ct["per_cluster"])
    return c


def _hist(counts):
    h = histogram_case(counts)
    return dict(_last(h["F"], h["Last"], th=3.0), hist=True)


@functools.lru_cache(maxsize=None)
def _contested_unsorted():
    return contested(11, 1, 3000, 2500, 90)


@functools.lru_cache(maxsize=None)
def _contested_unsorted_mixed():
    return contested(12, 1, 3000, 2500, 90, no_obs_every=7, occ_frac=0.05)


@functools.lru_cache(maxsize=None)
def _contested_sorted_mixed():
    return contested(13, 20, 120, 2500, 40, no_obs_every=5, occ_frac=0.05)


@functools.lru_cache(maxsize=None)
def _wide_voc(O):
    return O.PortVocabulary.random(10, 3, 9)


BUILDERS = {
    # 8192 x 8192: every feature queried at itself; all keys in the grid, so the grid sort's last slot holds a real key
    "self_kitti_8192": lambda O: _proj(*self_query(envelope_views(O, KITTI)), th=1.0),
    "self_euroc_8192_occ": lambda O: _proj(*self_query(envelope_views(O, EUROC), occupied_every=5), th=3.0),
    # natural projections of the right view into the left one, 8192 queries
    "proj_kitti_8192": lambda O: _proj(*mf.projection_case(envelope_views(O, KITTI), 3, n_mp=MATCH_MAX_FEATURES), th=3.0),
    # distorted bounds (min_x < 0, max_x inside the image): undistorted keypoints beyond the bounds fall outside the grid
    "self_kitti_8192_distorted": lambda O: _proj(*self_query(envelope_views(O, KITTI), bounds=(-14.5, -6.25, 1180.0, 360.0)), th=3.0),
    "contested_unsorted": lambda O: _contest(_contested_unsorted(), False),
    "contested_unsorted_mixed": lambda O: _contest(_contested_unsorted_mixed(), False),
    "contested_sorted_mixed": lambda O: _contest(_contested_sorted_mixed(), False),
    "contested_unsorted_last": lambda O: _contest(_contested_unsorted_mixed(), True, ori=False),
    "contested_sorted_last": lambda O: _contest(_contested_sorted_mixed(), True),
    # rotation histograms with tied bin counts and max2 (max3) exactly a tenth of max1: kept, the next smaller bin culled
    "hist_max2_tenth": lambda O: _hist({1: 40, 3: 4, 5: 4, 7: 3, 9: 4}),
    "hist_max3_tenth": lambda O: _hist({2: 20, 4: 20, 6: 2, 8: 2, 11: 1}),
    "tied_proj": lambda O: _proj(*mf.projection_case(tied_views(mf.two_views(O, 7), 1), 17, n_mp=600), th=3.0),
    "tied_bow": lambda O: _bow(O.PortVocabulary.random(10, 4, 5), tied_views(mf.two_views(O, 7), 2), 3, 2),
    "tied_tri": lambda O: _tri(O, O.PortVocabulary.random(10, 4, 5), tied_views(mf.two_views(O, 8), 3), 4, 2),
    "tied_last": lambda O: _last(*(lambda Cur, Last, Tcw, K: (Cur, Last, 15.0, True, Tcw, K))(*mf.last_frame_case(tied_views(mf.two_views(O, 8), 5), 28))),
    "tied_init": lambda O: _init(tied_views(mf.two_views(O, 7), 6)),
    "tied_fuse": lambda O: _fuse(O, tied_views(mf.two_views(O, 8), 7), 57),
    "tied_sim3": lambda O: _sim3(O, tied_views(mf.two_views(O, 7), 8), 67),
    "tied_local": lambda O: _local(tied_views(mf.two_views(O, 8), 9), 78),
    "init_kitti_8192": lambda O: _init(envelope_views(O, KITTI)),
    "local_kitti_8192": lambda O: _local(envelope_views(O, KITTI), 79),
    # the frame that frames_from_extractor builds from the extractor's 8192 first keypoints without distortion: its grid comes
    # from grid_sort_jobs_kernel (k_frame.cu), whose tail is then the only writer of cell_start[GRID_CELLS]
    "extract_kitti_8192": lambda O: dict(_proj(*self_query(envelope_views(O, KITTI, seed=9)), th=3.0), grid="jobs"),
    # wide FeatureVector nodes on envelope keyframes: levelsup = L puts every feature in one node (> BOW_JCAP), L - 1 gives
    # ten nodes of a few hundred to over a thousand features (one to a few rows per chunk, or direct evaluation)
    "bow_one_node_8192": lambda O: _bow(_wide_voc(O), envelope_views(O, KITTI), 5, 3, mp_frac=0.5),
    "bow_row_chunks_8192": lambda O: _bow(_wide_voc(O), envelope_views(O, EUROC), 6, 2),
    "tri_one_node_8192": lambda O: _tri(O, _wide_voc(O), tied_views(envelope_views(O, KITTI), 4, frac=0.1), 7, 3),
}
NAMES = sorted(BUILDERS)

_cache = {}


def case(O, name):
    if name not in _cache:
        _cache[name] = BUILDERS[name](O)
    return _cache[name]


# ---------------------------------------------------------------------------------------------------------------------------
# the port and the verbatim reference on a case, in comparable form
def run_port(O, c):
    m = c["method"]
    if m == "proj":
        return O.port_search_by_projection(c["F"], c["mps"], c["th"], c["ratio"])
    if m == "last":
        return O.port_search_by_projection_last(c["F"], c["Last"], c["Tcw"], c["K"], 40.0, c["th"], False, False, c["ori"])
    if m == "bow":
        return O.port_search_by_bow(c["kf1"], c["kf2"], c["ratio"], c["ori"]), O.port_search_by_bow_kf(c["kf1"], c["kf2"], c["ratio"], c["ori"])
    if m == "tri":
        return O.port_search_for_triangulation(c["kf1"], c["kf2"], c["F12"], c["ep"], c["only_stereo"], c["ori"])
    if m == "init":
        return O.port_search_for_initialization(c["F1"], c["F2"], c["prev"], c["window"], c["ratio"], c["ori"])
    if m == "fuse":
        return (O.port_fuse(c["KF"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], False),
                O.port_fuse(c["KF"], c["P"], c["Ts"], c["Ows"], c["K"], c["bf"], c["th"], True))
    if m == "sim3":
        return O.port_search_by_sim3(c["KF1"], c["KF2"], c["P1"], c["P2"], c["T1w"], c["T2w"], c["S12"], c["S21"], c["K"], c["th"])
    if m == "local":
        mps = local_mappoints(O, c)
        return O.port_search_by_projection(c["F"], mps, c["th"], c["ratio"])
    raise ValueError(m)


def local_mappoints(O, c):
    """Frame::isInFrustum of every point (port), as the MapPoints SearchByProjection(F, vpMapPoints) then reads."""
    fr = O.port_is_in_frustum(c["F"], c["P"], c["Tcw"], c["Ow"], c["K"], 40.0, 0.5)
    return MapPointsView(fr["proj_x"], fr["proj_y"], fr["proj_xr"], fr["level"], fr["view_cos"], c["P"].descriptors, valid=fr["in_view"],
                         has_obs=c["has_obs"])


def _epipole(Ow1):
    """C2 = R2w * Ow1 + t2w with T2w = I, projected with TRI_K2 (src/ORBmatcher.cc:663-670)."""
    fx, fy, cx, cy = [np.float32(x) for x in TRI_K2]
    C2 = np.asarray(Ow1, np.float32)
    inv = np.float32(1.0) / C2[2]
    return float(fx * C2[0] * inv + cx), float(fy * C2[1] * inv + cy)


def match_count(c, res):
    """The number of matches in a result of run_port (the first search of a two-search case)."""
    if c["method"] in ("bow", "fuse"):
        return res[0][0]
    return len(res) if c["method"] == "tri" else res[0]


def port_equals_reference(O, c):
    """Asserts that the port and the verbatim ORBmatcher.cc agree on case c; returns the port's result."""
    m = c["method"]
    res = run_port(O, c)
    if m == "proj":
        n_r, owner = O.ref_search_by_projection(c["F"], c["mps"], c["th"], c["ratio"])
        assert n_r == res[0] and np.array_equal(owner, O.owner_from_matches(c["F"], c["mps"], res[1]))
    elif m == "last":
        n_r, owner = O.ref_search_by_projection_last(c["F"], c["Last"], c["Tcw"], c["Tcw"], c["K"], 40.0, 40.0, c["th"], True, c["ori"])
        assert n_r == res[0] and np.array_equal(owner, O.owner_from_state(c["F"].occupied, res[1]))
    elif m == "bow":
        (n_p, m_p), (n_p2, m_p2) = res
        n_r, m_r = O.ref_search_by_bow(c["kf1"], c["kf2"], c["ratio"], c["ori"])
        assert n_r == n_p and np.array_equal(m_r, m_p)
        n_r, m_r = O.ref_search_by_bow_kf(c["kf1"], c["kf2"], c["ratio"], c["ori"])
        assert n_r == n_p2 and np.array_equal(m_r, m_p2)
    elif m == "tri":
        pairs_r = O.ref_search_for_triangulation(c["kf1"], c["kf2"], c["F12"], c["Ow1"], c["T2w"], TRI_K2, c["only_stereo"], c["ori"])
        assert np.array_equal(pairs_r, res)
    elif m == "init":
        n_r, m_r, p_r = O.ref_search_for_initialization(c["F1"], c["F2"], c["prev"], c["window"], c["ratio"], c["ori"])
        assert n_r == res[0] and np.array_equal(m_r, res[1]) and np.array_equal(p_r, res[2])
    elif m == "fuse":
        n_r, b_r = O.ref_fuse(c["KF"], c["P"], c["Tcw"], c["Ow"], c["K"], c["bf"], c["th"], False)
        assert n_r == res[0][0] and np.array_equal(b_r, res[0][1])
        n_r, b_r = O.ref_fuse(c["KF"], c["P"], c["Scw"], c["Ows"], c["K"], c["bf"], c["th"], True)
        assert n_r == res[1][0] and np.array_equal(b_r, res[1][1])
    elif m == "sim3":
        n_r, m_r = O.ref_search_by_sim3(c["KF1"], c["KF2"], c["P1"], c["P2"], c["T1w"], c["T2w"], c["s12"], c["R12"], c["t12"], c["K"], c["th"])
        assert n_r == res[0] and np.array_equal(m_r, res[1])
    elif m == "local":                              # isInFrustum is pinned by tests/test_oracle_frame_ref.py; here the search
        mps = local_mappoints(O, c)
        n_r, owner = O.ref_search_by_projection(c["F"], mps, c["th"], c["ratio"])
        assert n_r == res[0] and np.array_equal(owner, O.owner_from_matches(c["F"], mps, res[1]))
    return res


# ---------------------------------------------------------------------------------------------------------------------------
# coverage
def _hamming(a, b):
    return np.unpackbits(np.bitwise_xor(a, b), axis=-1).sum(-1)


def _claim_replay(c, last):
    """Sequential replay of a contested case, where every query's candidate list is its cluster in feature order.  Returns
    (match per query, wave of each claim, chain depth per query, pick position per query, events per feature)."""
    F = c["F"]
    q = c["Last"] if last else c["mps"]
    d = np.asarray(q.descriptors)
    n_q = len(d)
    held = np.asarray(F.occupied, bool).copy() if F.occupied is not None else np.zeros(len(F.mvKeysUn), bool)
    octv = F.mvKeysUn["octave"]
    cl, pc = c["cluster"], c["per_cluster"]
    dist_rows = {}
    match = np.full(n_q, -1); depth = np.zeros(n_q, int); pick = np.full(n_q, -1)
    events = np.zeros(len(F.mvKeysUn), int)
    claimer = {}                          # feature -> query claiming it in the current wave
    for i in range(n_q):
        if i % WAVE == 0:
            claimer = {}
        k = int(cl[i])
        if k not in dist_rows:
            dist_rows[k] = _hamming(F.mDescriptors[k * pc:(k + 1) * pc], d[i])
        dist = dist_rows[k]
        free = [p for p in range(pc) if not held[k * pc + p]]
        free.sort(key=lambda p: (dist[p], p))
        if not free:
            continue
        picks = free[:1] if last else free[:2]
        e1 = picks[0]
        dep = 0
        for p in range(pc):                       # entries ranked ahead of the last pick and claimed earlier in this wave
            f = k * pc + p
            if f in claimer and (dist[p], p) < (dist[picks[-1]], picks[-1]):
                dep = max(dep, depth[claimer[f]])
        depth[i] = dep + 1
        b1 = dist[e1]
        ok = b1 <= TH_HIGH
        if not last and ok and len(picks) > 1:
            e2 = picks[1]
            ok = not (octv[k * pc + e1] == octv[k * pc + e2] and np.float32(b1) > np.float32(0.8) * np.float32(dist[e2]))
        if ok:
            f = k * pc + e1
            match[i] = f
            pick[i] = e1
            events[f] += 1
            if q.has_obs[i]:
                held[f] = True
                claimer[f] = i
    return match, depth, pick, events


def _has_twin(F, f, radius=8.0):
    """Another feature of F within `radius` px with the same descriptor (tied_views makes such pairs): a matched feature with a
    twin is a tie at the minimum that the tie-break decided."""
    k, d = F.mvKeysUn, F.mDescriptors
    near = (np.abs(k["x"] - k["x"][f]) < radius) & (np.abs(k["y"] - k["y"][f]) < radius)
    near[f] = False
    return bool((near & (d == d[f]).all(1)).any())


def three_maxima(hist):
    """ORBmatcher::ComputeThreeMaxima (src/ORBmatcher.cc:1601-1642) -> (indices kept, counts)."""
    m1 = m2 = m3 = 0; i1 = i2 = i3 = -1
    for i, s in enumerate(hist):
        if s > m1: m3, m2, m1, i3, i2, i1 = m2, m1, s, i2, i1, i
        elif s > m2: m3, m2, i3, i2 = m2, s, i2, i
        elif s > m3: m3, i3 = s, i
    return (m1, m2, m3), (i1, i2, i3)


def _rot_bin(a1, a2):
    rot = np.float32(a1) - np.float32(a2)
    if rot < 0:
        rot = np.float32(rot + np.float32(360.0))
    b = int(np.floor(np.float32(rot * np.float32(1.0 / 30)) + 0.5))
    return 0 if b == 30 else b


def coverage(c, port_result):
    """The coverage classes (CLASSES) that case c reaches, judged from its inputs and the port's result on it."""
    hit = set()
    m = c["method"]
    if m in ("proj", "last"):
        F = c["F"]
        n = len(F.mvKeysUn)
        inside = in_grid(F.mvKeysUn, F.bounds)
        if n == MATCH_MAX_FEATURES and inside.all():
            hit.add("n8192_all_in_grid_jobs" if c.get("grid") == "jobs" else "n8192_all_in_grid")
        if not inside.all():
            hit.add("keys_outside_grid")
    if m in ("proj", "last") and "cluster" in c:
        last = m == "last"
        match, depth, pick, events = _claim_replay(c, last)
        got = port_result[1]
        if last:                                   # the replay's final owners equal the port's state (no culling here)
            want = np.full(len(c["F"].mvKeysUn), -1)
            for i, f in enumerate(match):
                if f >= 0:
                    want[f] = max(want[f], i)
            assert c["ori"] or np.array_equal(np.where(got >= 0, got, -1), want)
        else:
            assert np.array_equal(got, match)
        committed = np.nonzero(match >= 0)[0]
        if (committed >= WAVE).any() and len(match) > WAVE:
            hit.add("wave_after_first")
        if depth.max() > 32:
            hit.add("chain_depth_gt_32")
        if depth.max() >= WAVE:
            hit.add("chain_depth_1024")
        if c["per_cluster"] > SORT_CAP:
            if (pick > 0).any():
                hit.add("pick_unsorted")
        elif (pick >= RES_K).any():
            hit.add("pick_beyond_res_k")
        if last and (events >= 2).any():
            hit.add("last_two_events")
    if m == "last" and c.get("hist"):
        Cur, Last, state = c["F"], c["Last"], port_result[1]
        hist = np.zeros(30, int)
        for f in np.nonzero(state != -1)[0]:
            q = state[f] if state[f] >= 0 else None
            if q is None:                          # culled: recover the query from the construction (one feature per query)
                q = int(np.nonzero((Last.mvKeysUn["x"] == Cur.mvKeysUn["x"][f]) & (Last.mvKeysUn["y"] == Cur.mvKeysUn["y"][f]))[0][0])
            hist[_rot_bin(Last.mvKeysUn["angle"][q], Cur.mvKeysUn["angle"][f])] += 1
        (m1, m2, m3), _ = three_maxima(hist)
        tenth = np.float32(0.1) * np.float32(m1)
        if m1 and (np.float32(m2) == tenth or np.float32(m3) == tenth):
            hit.add("hist_boundary")
    if m == "proj" and "cluster" not in c and len(c["mps"].descriptors) <= 1000:
        F, mps = c["F"], c["mps"]
        for i, f in enumerate(port_result[1]):
            if f < 0:
                continue
            dd = _hamming(F.mDescriptors, mps.descriptors[i])
            near = (np.abs(F.mvKeysUn["x"] - F.mvKeysUn["x"][f]) < 8) & (np.abs(F.mvKeysUn["y"] - F.mvKeysUn["y"][f]) < 8)
            twins = np.nonzero(near & (dd == dd[f]))[0]
            if len(twins) > 1:
                hit.add("tie_min_proj")
                if len(set(F.mvKeysUn["octave"][twins].tolist())) > 1:
                    hit.add("tie_level_ratio")
    if m == "last" and "cluster" not in c and not c.get("hist"):
        if any(_has_twin(c["F"], f) for f in np.nonzero(port_result[1] >= 0)[0]):
            hit.add("tie_min_last")
    if m == "init":
        if len(c["F1"].mvKeysUn) == MATCH_MAX_FEATURES and port_result[0] > 0:
            hit.add("init_8192")
        if any(_has_twin(c["F2"], j) for j in port_result[1][port_result[1] >= 0]):
            hit.add("tie_min_init")
    if m == "fuse":
        if any(_has_twin(c["KF"], f) for r in port_result for f in r[1][r[1] >= 0]):
            hit.add("tie_min_argmin")
    if m == "sim3":
        if any(_has_twin(c["KF2"], j) for j in port_result[1][port_result[1] >= 0]):
            hit.add("tie_min_argmin")
    if m == "local":
        if len(c["P"].world_pos) <= 2000 and any(_has_twin(c["F"], f) for f in port_result[1][port_result[1] >= 0]):
            hit.add("tie_min_local")
    if m == "bow":
        kf1, kf2 = c["kf1"], c["kf2"]
        widths = np.diff(kf2.mFeatVec.start)
        if widths.max() > BOW_JCAP:
            hit.add("bow_node_gt_jcap")
        w1 = dict(zip(kf1.mFeatVec.node_id.tolist(), np.diff(kf1.mFeatVec.start).tolist()))
        for nd, nt in zip(kf2.mFeatVec.node_id.tolist(), widths.tolist()):
            rows = min(256, max(1, BOW_DCAP // nt)) if nt <= BOW_JCAP else 256
            if w1.get(nd, 0) > rows:
                hit.add("bow_row_chunks")
        fv1, fv2 = kf1.mFeatVec.as_dict(), kf2.mFeatVec.as_dict()
        for nd, rows in fv1.items():                    # a keyframe row whose nearest frame features tie: the ratio test meets d == d
            cands = fv2.get(nd, [])
            if len(cands) < 2:
                continue
            for i in rows[:8]:
                dd = _hamming(kf2.mDescriptors[cands], kf1.mDescriptors[i])
                if kf1.has_mp[i] and dd.min() < TH_LOW and (dd == dd.min()).sum() > 1:
                    hit.add("tie_min_bow")
    if m == "tri":
        kf1, kf2 = c["kf1"], c["kf2"]
        fv2 = kf2.mFeatVec.as_dict()
        node2 = {f: nd for nd, fs in fv2.items() for f in fs}
        for i1, i2 in port_result[:400]:
            cands = [f for f in fv2[node2[int(i2)]] if not kf2.has_mp[f] and f != i2]
            if cands and (_hamming(kf2.mDescriptors[cands], kf1.mDescriptors[i1]) == _hamming(kf2.mDescriptors[i2], kf1.mDescriptors[i1])).any():
                hit.add("tie_min_tri")
                break
    return hit
