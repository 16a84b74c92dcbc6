"""GPU: the CUDA library equals the port on the non-finite and int-overflowing cases of tests/nonfinite_cases.py — match arrays
and counts exactly, feature grids cell by cell through borb_debug_frame_read — on host views, on resident frames from
borb_frame_create and borb_frames_from_extractor, and with every case of a method in one batched call next to an empty job.  A host
view whose keypoint octave lies outside [0, n_levels) is refused by every entry point that takes one, before any launch."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from orb_slam2_b200._lib import STATUS_NAMES, BorbError
from tests import nonfinite_cases as N
from tests import proj_geometry as G
from tests import test_gpu_featvec_checks as FC
from tests.test_gpu_proj_geometry import _equal, _set, run_gpu

pytestmark = pytest.mark.gpu

BORB_ERR_INVALID_ARG = next(k for k, v in STATUS_NAMES.items() if v == "BORB_ERR_INVALID_ARG")

CASES = N.cases()


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def mt(M):
    m = M.ORBmatcher(0.8, False)
    yield m
    m.close()


def _grid_equal(read, want):
    cs, ci = want
    return np.array_equal(read["cell_start"], cs) and np.array_equal(read["cell_idx"], ci[:cs[-1]])


def _gpu(mt, c, method, resident):
    if method == "init":
        _set(mt, 0.9)
        if resident:
            F1, F2 = c["F1"].make_resident(mt), c["F2"].make_resident(mt)
            return mt.SearchForInitializationBatch([F1], [F2], [c["prev"]], c["window"])[0]
        return mt.SearchForInitialization(c["F1"], c["F2"], c["prev"], c["window"])
    return run_gpu(mt, c, method, resident)


def _same(method, got, want):
    if method == "init":
        return got[0] == want[0] and np.array_equal(got[1], want[1]) and G.same_float(got[2], want[2])
    return _equal(method, got, want)


SINGLE = [(i, m, r) for i, c in enumerate(CASES) for m in N.methods(c) if m != "grid" for r in (False, True)]


@pytest.mark.parametrize("i,method,resident", SINGLE,
                         ids=[f"{CASES[i]['cls']}-{CASES[i]['member']}-{m}-{'res' if r else 'host'}" for i, m, r in SINGLE])
def test_single_call_equals_port(mt, oracle, i, method, resident):
    c = CASES[i]
    want = N.run_port(oracle, c, method)
    got = _gpu(mt, c, method, resident)
    assert _same(method, got, want), (c["cls"], c["member"], method, got, want)


@pytest.mark.parametrize("cls", ["grid_nan_x", "grid_nan_y"])
def test_frame_create_grid_equals_port(mt, oracle, cls):
    """borb_frame_create's AssignFeaturesToGrid on a NaN key: in no cell, while its finite twin sits in column / row 0."""
    for c in CASES:
        if c["cls"] == cls:
            F = c["F"].make_resident(mt)
            assert _grid_equal(F.resident.read(stereo=False), N.run_port(oracle, c, "grid")), (cls, c["member"])
            F.resident.close()


def test_frames_from_extractor_nan_keys_grid(M, oracle):
    """borb_frames_from_extractor under calibrations whose UndistortKeyPoints gives NaN keys (and NaN bounds): the keys read back
    bit for bit as the port's (NaN as NaN), and the grid holds no key, as Frame.cc's has none."""
    from orb_slam2_b200.extractor import ORBextractor
    X = ORBextractor(1000)
    img = N.undistort_image()
    keys, _ = X.extract_batch([img])[0]
    mt = M.ORBmatcher(0.8, False)
    h, w = img.shape
    for K, dist in N.NAN_CALIBRATIONS:
        frames, host = M.frames_from_extractor(mt, X, [0, 0], [len(keys), len(keys) // 2], K, dist)
        for j, n in enumerate((len(keys), len(keys) // 2)):
            p = oracle.port_rgbd_frame(keys[:n], np.array(K, np.float32), np.array(dist, np.float32), 40.0, np.zeros((h, w), np.float32))
            got = frames[j].resident.read(stereo=False)
            assert np.isnan(p["keys_un"]["x"]).all()
            for f in ("x", "y"):
                assert G.same_float(got["keys_un"][f], p["keys_un"][f]), (K, n, f)
            assert _grid_equal(got, oracle.port_assign_grid(p["keys_un"], p["bounds"])), (K, n)
            frames[j].resident.close()
    mt.close()


def _by(method):
    return [c for c in CASES if method in N.methods(c)]


def _empty_points(P):
    return dataclasses.replace(P, **{f: getattr(P, f)[:0] for f in ("world_pos", "descriptors", "max_distance", "min_distance", "normal",
                                                                      "angle", "valid")})


def test_projection_batch(M, mt, oracle):
    """borb_search_by_projection_batch: the proj cases of one th in one call, next to a job without map points."""
    _set(mt)
    groups = {}
    for c in _by("proj"):
        groups.setdefault(c["th"], []).append(c)
    for th, cs in groups.items():
        frames = [c["F"].make_resident(mt) for c in cs + cs[:1]]
        m0 = cs[0]["mps"]
        empty = M.MapPointsView(*[getattr(m0, f.name)[:0] for f in dataclasses.fields(m0)])
        got = mt.SearchByProjectionBatch(frames, [c["mps"] for c in cs] + [empty], th)
        for j, c in enumerate(cs):
            assert _equal("proj", got[j], N.run_port(oracle, c, "proj")), (c["cls"], c["member"])
        assert got[-1][0] == 0 and len(got[-1][1]) == 0


def test_init_batch(mt, oracle):
    """borb_search_for_initialization_batch: every SearchForInitialization case in one call, next to a job without F1 features."""
    _set(mt, 0.9)
    cs = _by("init")
    F1s = [c["F1"].make_resident(mt) for c in cs]
    F2s = [c["F2"].make_resident(mt) for c in cs]
    e = cs[0]
    empty = dataclasses.replace(e["F1"], mvKeysUn=e["F1"].mvKeysUn[:0], mDescriptors=e["F1"].mDescriptors[:0])
    got = mt.SearchForInitializationBatch(F1s + [empty.make_resident(mt)], F2s + [F2s[0]], [c["prev"] for c in cs] + [np.zeros((0, 2), np.float32)],
                                          N.INIT_WINDOW)
    for j, c in enumerate(cs):
        assert _same("init", got[j], N.run_port(oracle, c, "init")), (c["cls"], c["member"])
    assert got[-1][0] == 0


@pytest.mark.parametrize("method", ["fuse", "fuse_kf"])
def test_fuse_batch(mt, oracle, method):
    """borb_fuse_batch: the Fuse cases of one overload, each with its own th, next to a job without points."""
    cs = _by(method)
    kfs = [c["F"].make_resident(mt) for c in cs + cs[:1]]
    points = [c["P"] for c in cs] + [_empty_points(cs[0]["P"])]
    poses = [(G.scw(c) if method == "fuse" else c["Tcw"], c["Ow"]) for c in cs + cs[:1]]
    got = mt.FuseBatch(kfs, points, poses, G.K_CAM, G.BF, [c["th"] for c in cs + cs[:1]], Scw=method == "fuse")
    for j, c in enumerate(cs):
        assert _equal(method, got[j], N.run_port(oracle, c, method)), (c["cls"], c["member"])
    assert got[-1][0] == 0 and len(got[-1][1]) == 0


def test_sim3_batch(mt, oracle):
    """borb_search_by_sim3_batch: both SearchBySim3 cases, each with its own th, next to a keyframe pair without MapPoints."""
    _set(mt)
    cs = _by("sim3")
    jobs = [G.sim3_args(c) for c in cs]
    none = lambda P: dataclasses.replace(P, valid=np.zeros(len(P.world_pos), np.uint8))
    e = jobs[0]
    jobs.append((e[0], e[1], none(e[2]), none(e[3])) + e[4:])
    got = mt.SearchBySim3Batch([j[0].make_resident(mt) for j in jobs], [j[1].make_resident(mt) for j in jobs], [j[2] for j in jobs],
                               [j[3] for j in jobs], [(j[4], j[5]) for j in jobs], [(j[6], j[7]) for j in jobs], G.K_CAM, [j[9] for j in jobs])
    for j, c in enumerate(cs):
        assert _equal("sim3", got[j], N.run_port(oracle, c, "sim3")), (c["cls"], c["member"])
    assert got[-1][0] == 0 and (got[-1][1] == -1).all()


def test_keyframe_and_last_frame_batches(M, mt, oracle):
    """borb_search_by_projection_kf_batch and _last_batch: their cases, each with its own th, next to a job without points."""
    _set(mt)
    cs = _by("kf")
    got = mt.SearchByProjectionKFBatch([c["F"].make_resident(mt) for c in cs + cs[:1]], [c["P"] for c in cs] + [_empty_points(cs[0]["P"])],
                                       [(c["Tcw"], c["Ow"]) for c in cs + cs[:1]], G.K_CAM, [c["th"] for c in cs + cs[:1]], 100)
    for j, c in enumerate(cs):
        assert _equal("kf", got[j], N.run_port(oracle, c, "kf")), (c["cls"], c["member"])
    assert got[-1][0] == 0
    cs = _by("last")
    L0 = G.last_view(cs[0])
    empty = M.LastFrameView(L0.mvKeysUn[:0], L0.world_pos[:0], L0.descriptors[:0], L0.valid[:0], L0.has_obs[:0])
    cur = lambda c: G.FrameView(c["F"].mvKeysUn, c["F"].mDescriptors, c["F"].mvScaleFactors, c["F"].bounds).make_resident(mt)
    got = mt.SearchByProjectionLastBatch([cur(c) for c in cs + cs[:1]], [G.last_view(c) for c in cs] + [empty], [c["Tcw"] for c in cs + cs[:1]],
                                         G.K_CAM, G.BF, [c["th"] for c in cs + cs[:1]], forward=[False] * (len(cs) + 1),
                                         backward=[False] * (len(cs) + 1))
    for j, c in enumerate(cs):
        assert _equal("last", got[j], N.run_port(oracle, c, "last")), (c["cls"], c["member"])
    assert got[-1][0] == 0


# ---------------------------------------------------------------------------------------------------------------------------
# octave refusals
BAD_FEATURE = 1


def _bad(keys, octave):
    k = np.array(keys, copy=True)
    k["octave"][BAD_FEATURE] = octave
    return k


def _launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def _world():
    return next(c for c in CASES if c["cls"] == "radius_th_fuse" and c["member"] == 0)


def _calls(M, mt, octave):
    """(entry point, call) of every entry point taking a host view, with keypoint BAD_FEATURE of that view at `octave`."""
    w = _world()
    Fb = dataclasses.replace(w["F"], mvKeysUn=_bad(w["F"].mvKeysUn, octave))
    p = next(c for c in CASES if c["cls"] == "radius_th_proj" and c["member"] == 0)
    Fp = dataclasses.replace(p["F"], mvKeysUn=_bad(p["F"].mvKeysUn, octave))
    i = next(c for c in CASES if c["cls"] == "nan_centre_init" and c["member"] == 0)
    t = next(c for c in G.cases() if c["cls"] == "tri_epipole" and c["member"] == 0)
    kf1 = dataclasses.replace(t["kf1"], mvKeysUn=_bad(t["kf1"].mvKeysUn, octave), _keep=[])
    kf2 = dataclasses.replace(t["kf2"], mvKeysUn=_bad(t["kf2"].mvKeysUn, octave), _keep=[])
    Cur = G.FrameView(Fb.mvKeysUn, Fb.mDescriptors, Fb.mvScaleFactors, Fb.bounds)
    K, T, Ow = G.K_CAM, w["Tcw"], w["Ow"]
    return [
        ("borb_search_by_projection", lambda: mt.SearchByProjection(Fp, p["mps"], 3.0)),
        ("borb_search_by_projection_last", lambda: mt.SearchByProjectionLast(Cur, G.last_view(w), T, K, G.BF, 3.0, False, False)),
        ("borb_search_by_projection_kf", lambda: mt.SearchByProjectionKF(Fb, w["P"], T, Ow, K, 3.0, 100)),
        ("borb_search_by_projection_sim3", lambda: mt.SearchByProjectionSim3(Fb, w["P"], T, Ow, K, 3)),
        ("borb_search_local_points", lambda: mt.SearchLocalPoints(Fb, w["P"], T, Ow, K, G.BF, 3.0, has_obs=w["has_obs"])),
        ("borb_fuse(Scw)", lambda: mt.Fuse(Fb, w["P"], T, Ow, K, G.BF, 3.0, Scw=True)),
        ("borb_fuse", lambda: mt.Fuse(Fb, w["P"], T, Ow, K, G.BF, 3.0, Scw=False)),
        ("borb_search_by_sim3(kf1)", lambda: mt.SearchBySim3(Fb, w["F"], w["P"], w["P"], T, T, G.S12_ID, G.S21_ID, K, 7.5)),
        ("borb_search_by_sim3(kf2)", lambda: mt.SearchBySim3(w["F"], Fb, w["P"], w["P"], T, T, G.S12_ID, G.S21_ID, K, 7.5)),
        ("borb_search_for_initialization(F1)",
         lambda: mt.SearchForInitialization(dataclasses.replace(i["F1"], mvKeysUn=_bad(i["F1"].mvKeysUn, octave)), i["F2"], i["prev"], 100)),
        ("borb_search_for_initialization(F2)",
         lambda: mt.SearchForInitialization(i["F1"], dataclasses.replace(i["F2"], mvKeysUn=_bad(np.concatenate([i["F2"].mvKeysUn] * 2), octave),
                                                                          mDescriptors=np.concatenate([i["F2"].mDescriptors] * 2)), i["prev"], 100)),
        ("borb_search_for_triangulation(kf1)", lambda: mt.SearchForTriangulation(kf1, t["kf2"], t["F12"], t["ep"], False)),
        ("borb_search_for_triangulation(kf2)", lambda: mt.SearchForTriangulation(t["kf1"], kf2, t["F12"], t["ep"], False)),
        ("borb_search_for_triangulation_batch", lambda: mt.SearchForTriangulationBatch([t["kf1"], kf1], [t["kf2"], t["kf2"]], [t["F12"]] * 2,
                                                                                       [t["ep"]] * 2)),
        ("borb_search_by_bow_kf", lambda: mt.SearchByBoW_KF(kf1, t["kf2"])),
        ("borb_frame_create", lambda: Fb.make_resident(mt)),
    ]


@pytest.fixture(scope="module")
def bow_world(M, oracle):
    """test_gpu_featvec_checks' keyframe views and database, on which its entry_points() drives every BoW-guided entry point."""
    pv = oracle.PortVocabulary.random(10, 4, 5)
    e = pv.export()
    voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
    mt = M.ORBmatcher(0.7, True)
    good = FC.keyframe(M, 1, flip=0.02)
    frames = [M.FrameView(good.mvKeysUn, good.mDescriptors, FC.SCALE, (0.0, 0.0, 640.0, 480.0)).make_resident(mt) for _ in range(2)]
    good = dataclasses.replace(good, mFeatVec=mt.ComputeBoWBatch(voc, frames, 2)[0][1])
    db = M.KeyFrameDatabase(mt)
    db.add(good, {1: 0.5, 3: 0.25})
    yield mt, db, good, frames
    mt.close()


def _all_calls(M, mt, bow_world, octave):
    """(entry point, call, matcher, job index of a batch or None) of every entry point taking a host view."""
    out = [(name, call, mt, 1 if name.endswith("_batch") else None) for name, call in _calls(M, mt, octave)]
    good = bow_world[2]
    bad = dataclasses.replace(good, mvKeysUn=_bad(good.mvKeysUn, octave), _keep=[])
    return out + [(name, call, bow_world[0], job) for name, call, job in FC.entry_points(M, bow_world, bad)]


@pytest.mark.parametrize("octave", [-1, G.N_LEVELS, 128])
def test_out_of_range_octave_is_refused(M, mt, bow_world, octave):
    """Every entry point that takes a host view refuses an octave outside [0, n_levels) — the reference would index
    mvInvLevelSigma2 / mvScaleFactors outside the pyramid, and the candidate lists pack octaves 0 and 128 alike — with
    BORB_ERR_INVALID_ARG, the feature (and for a batch the job) in the error text, and no launch; a refused borb_kfdb_add takes
    no slot."""
    slots = bow_world[1].size()[0]
    for name, call, m, job in _all_calls(M, mt, bow_world, octave):
        before = _launches(m)
        with pytest.raises(BorbError) as e:
            call()
        msg = str(e.value)
        assert e.value.status == BORB_ERR_INVALID_ARG, (name, msg)
        assert f"keypoint {BAD_FEATURE}: octave {octave} outside" in msg, (name, msg)
        if job is not None:
            assert f"job {job}:" in msg, (name, msg)
        assert _launches(m) == before, name
    assert bow_world[1].size()[0] == slots


def test_in_range_octaves_are_accepted(M, mt, bow_world):
    """The same calls with the octave at the pyramid's last level run."""
    for name, call, m, job in _all_calls(M, mt, bow_world, G.N_LEVELS - 1):
        call()


SENTINEL = 0xA5


class _Sentinels:
    """Stands in for orb_slam2_b200.matcher's numpy (np) or ctypes (C) module during one call: every array a wrapper allocates with
    np.full / np.zeros and every count it allocates with C.c_int32 is its output, and starts filled with SENTINEL bytes instead."""

    def __init__(self, mod, made):
        self._mod, self._made = mod, made

    def __getattr__(self, name):
        return getattr(self._mod, name)

    def _array(self, shape, dtype=float, *args, **kw):
        a = np.empty(shape, dtype)
        a.reshape(-1).view(np.uint8)[:] = SENTINEL
        self._made.append(a)
        return a

    def full(self, shape, fill_value, dtype=None, *args, **kw):
        return self._array(shape, dtype if dtype is not None else np.asarray(fill_value).dtype)

    def zeros(self, shape, dtype=float, *args, **kw):
        return self._array(shape, dtype)

    def c_int32(self, value=0):
        v = self._mod.c_int32(int(np.array(SENTINEL * 0x01010101, np.uint32).view(np.int32)))
        self._made.append(v)
        return v


def test_refusal_leaves_outputs_untouched(M, mt, bow_world, monkeypatch):
    """A refused call writes none of its outputs — not the counts, not the -1 fills, and in a batch not those of the jobs before
    the refused one: every output array and count the wrapper hands over still holds its sentinel bytes."""
    from orb_slam2_b200 import matcher as MM
    calls = [c for c in _all_calls(M, mt, bow_world, -1) if c[0] != "search_by_bow_db_pairs"]
    db, good = bow_world[1], bow_world[2]
    bad = dataclasses.replace(good, mvKeysUn=_bad(good.mvKeysUn, -1), _keep=[])
    # with explicit slots: the wrapper's slot count for None comes from borb_kfdb_size, an output of a call that succeeds
    calls.append(("search_by_bow_db_pairs", lambda: db.SearchByBoWPairs([0], bad), bow_world[0], None))
    for name, call, m, job in calls:
        made = []
        with monkeypatch.context() as mp:
            mp.setattr(MM, "np", _Sentinels(np, made))
            mp.setattr(MM, "C", _Sentinels(C, made))
            with pytest.raises(BorbError):
                call()
        if name != "borb_frame_create":                              # the only output is the handle, which stays unset
            assert made, name
        for o in made:
            raw = np.ascontiguousarray(o).reshape(-1).view(np.uint8) if isinstance(o, np.ndarray) else np.frombuffer(bytes(o), np.uint8)
            assert (raw == SENTINEL).all(), name
    # the sentinels do see writes: an accepted call overwrites its count
    made = []
    name, call = _calls(M, mt, G.N_LEVELS - 1)[2]
    with monkeypatch.context() as mp:
        mp.setattr(MM, "np", _Sentinels(np, made))
        mp.setattr(MM, "C", _Sentinels(C, made))
        call()
    assert any(not (np.frombuffer(bytes(o), np.uint8) == SENTINEL).all() for o in made if not isinstance(o, np.ndarray)), name
