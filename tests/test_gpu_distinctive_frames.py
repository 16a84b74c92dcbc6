"""GPU parity of borb_distinctive_descriptors_frames, MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307) read from
resident keyframes: for every point, best_idx and the chosen descriptor must equal borb_distinctive_descriptors on the same rows
gathered on the host (ResidentFrame.read), the oracle port, and the verbatim MapPoint.cc fed the full observation list with its bad
keyframes.  Frames come from the extractor (mono, stereo, RGB-D) and from borb_frame_create; one launch per call with observations,
none without; argument errors refused before anything is launched, with the outputs untouched."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_b200 import synth

pytestmark = pytest.mark.gpu

SCALE = (1.2 ** np.arange(8)).astype(np.float32)
SHAPES = (0, 1, 2, 3, 4, 5, 8, 13, 33, 64, 100, 300)
CRAFTED = 6                       # index of the crafted frame in the world fixture


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def random_keys(rng, n):
    from orb_slam2_b200._lib import KP_DTYPE
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(20, 600, n).astype(np.float32); k["y"] = rng.uniform(20, 440, n).astype(np.float32)
    k["angle"] = rng.uniform(0, 360, n).astype(np.float32); k["size"] = 31.0; k["octave"] = rng.integers(0, 8, n); k["class_id"] = -1
    return k


def flip_bits(rng, row, n_bits):
    out = row.copy()
    for b in rng.choice(256, n_bits, replace=False):
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def resident(M, mt, desc, rng):
    desc = np.ascontiguousarray(desc, np.uint8)
    return M.FrameView(random_keys(rng, len(desc)), desc, SCALE, (0.0, 0.0, 800.0, 600.0)).make_resident(mt)


def crafted_rows(rng):
    """400 rows: 20 clusters of 20 noisy copies of a base (0-40 flipped bits), then rows 400-409 identical, then a median tie at
    410-412: x = ~a and b = a with 5 bits flipped, so that x, a, b have medians 251, 5, 5 and a (index 1) wins."""
    rows = []
    for _ in range(20):
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        rows += [flip_bits(rng, base, int(rng.integers(0, 41))) for _ in range(20)]
    same = rng.integers(0, 256, 32, dtype=np.uint8)
    rows += [same] * 10
    a = rng.integers(0, 256, 32, dtype=np.uint8)
    rows += [~a, a, flip_bits(rng, a, 5)]
    return np.stack(rows)


@pytest.fixture(scope="module")
def world(M):
    """(matcher, [(name, FrameView)], host rows per frame): extractor frames of the TUM (640x480) shape, monocular and RGB-D, and of
    the EuRoC stereo (752x480) shape, then borb_frame_create frames: the crafted rows, 1000 random rows and 8192 random rows."""
    from orb_slam2_b200.extractor import ORBextractor
    mt = M.ORBmatcher()
    rng = np.random.default_rng(71)
    frames, names = [], []
    X = ORBextractor(1000)
    outs = X.extract_batch([synth.mono_frame(310 + i, 0, 0, 640, 480) for i in range(3)])
    K = (517.3, 516.5, 318.6, 255.3)
    fr, _ = M.frames_from_extractor(mt, X, [0, 1], [len(o[0]) for o in outs[:2]], K, (0.26, -0.95, -0.005, 0.002, 1.16))
    frames += fr; names += ["tum_mono_0", "tum_mono_1"]
    depth = [(1.0 + 2.0 * rng.random((480, 640))).astype(np.float32) for _ in range(2)]
    fr, _ = M.frames_from_extractor(mt, X, [1, 2], [len(o[0]) for o in outs[1:3]], K, bf=40.0, mode=2, depth=depth)
    frames += fr; names += ["tum_rgbd_1", "tum_rgbd_2"]
    XE = ORBextractor(1200)
    pairs = [synth.stereo_pair(95 + i, 0, 0, 752, 480) for i in range(2)]
    res = XE.stereo_frames([p[0] for p in pairs], [p[1] for p in pairs], 47.9, 435.2)
    fr, _ = M.frames_from_extractor(mt, XE, [0, 2], [len(r["mvKeys"]) for r in res], (435.2, 435.2, 376.0, 240.0), bf=47.9, mode=1)
    frames += fr; names += ["euroc_stereo_0", "euroc_stereo_1"]
    frames.append(resident(M, mt, crafted_rows(rng), rng)); names.append("crafted")
    for n in (1000, 8192):
        frames.append(resident(M, mt, rng.integers(0, 256, (n, 32), dtype=np.uint8), rng)); names.append(f"random_{n}")
    rows = [F.resident.read(stereo=False)["desc"] for F in frames]
    assert all(len(r) > 100 for r in rows) and len(rows[-1]) == 8192 and names[CRAFTED] == "crafted"
    return mt, list(zip(names, frames)), rows


def gather(rows, group):
    f, k = group
    return np.stack([rows[a][b] for a, b in zip(f, k)]) if len(f) else np.zeros((0, 32), np.uint8)


def check_points(mt, oracle, frames, rows, groups):
    """The new call against the single call on the gathered rows and against the oracle port, point by point; one launch."""
    c0 = launches(mt)
    best, desc = mt.ComputeDistinctiveDescriptorsFrames(frames, groups)
    assert launches(mt) - c0 == (1 if any(len(g[0]) for g in groups) else 0)
    gathered = [gather(rows, g) for g in groups]
    want = mt.ComputeDistinctiveDescriptors(gathered)
    assert np.array_equal(best, want), np.nonzero(best != want)[0][:10]
    for p, g in enumerate(gathered):
        assert best[p] == oracle.port_distinctive_descriptor(g), p
        assert np.array_equal(desc[p], g[best[p]] if best[p] >= 0 else np.zeros(32, np.uint8)), p
    return best, desc


def shape_points(rng, rows, n_crafted):
    """Points of every N in SHAPES over all frames, drawn at random (repeats included), then the same N inside one crafted cluster
    with rows from other frames mixed in beyond 20."""
    groups = []
    for N in SHAPES:
        f = rng.integers(0, len(rows), N)
        groups.append((f, np.array([rng.integers(0, len(rows[a])) for a in f], np.int64)))
        c = int(rng.integers(0, 20))
        f = np.full(N, n_crafted)
        k = 20 * c + rng.integers(0, 20, N)
        mix = np.arange(N) >= 20
        f[mix] = rng.integers(0, len(rows) - 1, int(mix.sum()))
        k[mix] = [rng.integers(0, len(rows[a])) for a in f[mix]]
        groups.append((f, k))
    return groups


def test_frame_sources_and_point_shapes(M, oracle, world):
    """Points over the extractor frames (mono, stereo, RGB-D) and the borb_frame_create frames, N in SHAPES; all rows identical
    (index 0 wins); an exact median tie (the first minimal median wins); the same (frame, feature) observed twice; one frame
    observed by many points; the 8192-feature frame read at index 8191.  Every point equals the single call on the rows
    ResidentFrame.read() gives and the oracle port."""
    mt, named, rows = world
    frames = [F for _, F in named]
    rng = np.random.default_rng(72)
    groups = shape_points(rng, rows, CRAFTED)
    special = len(groups)
    groups.append((np.full(6, CRAFTED), np.arange(400, 406)))                     # all rows identical
    groups.append((np.full(3, CRAFTED), np.arange(410, 413)))                     # median tie: x, a, b
    groups.append((np.full(5, CRAFTED), np.array([412, 410, 411, 411, 410])))     # b, x, a, a, x: repeats, a tie between b and a
    groups.append((np.array([0, 0, 3, 3]), np.array([5, 5, 7, 7])))             # each pair observed twice
    groups.append((np.array([len(rows) - 1]), np.array([8191])))                 # the last row of the 8192-feature frame
    groups.append((np.array([len(rows) - 1, 0, len(rows) - 1]), np.array([8191, 1, 8190])))
    for _ in range(500):                                                          # one frame observed by many points
        N = int(rng.integers(1, 12))
        groups.append((np.full(N, CRAFTED), rng.integers(0, 400, N)))
    best, desc = check_points(mt, oracle, frames, rows, groups)
    assert best[0] == -1 and best[1] == -1
    assert best[special] == 0 and best[special + 1] == 1
    assert np.array_equal(desc[special + 4], rows[-1][8191])


def test_frames_as_resident_frames_or_views(M, oracle, world):
    """The frame table takes ResidentFrames or FrameViews carrying one, and a frame may appear in it several times."""
    mt, named, rows = world
    rng = np.random.default_rng(73)
    groups = shape_points(rng, rows, CRAFTED)
    mixed = [F.resident if i % 2 else F for i, (_, F) in enumerate(named)]
    b1, d1 = check_points(mt, oracle, mixed, rows, groups)
    twice = mixed + mixed                                                          # the second copy of every frame
    shifted = [(np.asarray(f) + len(mixed), k) for f, k in groups]
    b2, d2 = mt.ComputeDistinctiveDescriptorsFrames(twice, shifted)
    assert np.array_equal(b1, b2) and np.array_equal(d1, d2)


def test_verbatim_reference_with_bad_keyframes(M, oracle_ref, world):
    """The verbatim MapPoint.cc gets each point's full observation list with a bad mask; the new call gets the list with the bad
    keyframes dropped.  The chosen descriptor must be the same (None from the reference where best_idx is -1)."""
    mt, named, rows = world
    frames = [F for _, F in named]
    rng = np.random.default_rng(74)
    full = shape_points(rng, rows, CRAFTED)
    full.append((np.full(4, CRAFTED), np.arange(400, 404)))
    bads, kept = [], []
    for f, k in full:
        bad = (rng.random(len(f)) < 0.25).astype(np.uint8)
        if len(f) == 3:
            bad[:] = 1                                                             # every keyframe bad: no descriptor
        bads.append(bad)
        kept.append((np.asarray(f)[bad == 0], np.asarray(k)[bad == 0]))
    best, desc = mt.ComputeDistinctiveDescriptorsFrames(frames, kept)
    for p, ((f, k), bad) in enumerate(zip(full, bads)):
        ref = oracle_ref.ref_distinctive_descriptor(gather(rows, (f, k)), bad)
        if ref is None:
            assert best[p] == -1, p
        else:
            assert best[p] >= 0 and np.array_equal(desc[p], ref), p


def test_realistic_tick_of_32_streams(M, oracle):
    """32 streams, each ~1500 MapPoints of 2-30 observations over its 20 resident keyframes of 1000 features (the SearchInNeighbors
    refresh), in one call: every point equals the single call run per stream on the host rows.  Each observation takes a row of
    its own (a feature holds one MapPoint); a point with more than 20 observations sees some keyframe at two features."""
    mt = M.ORBmatcher()
    rng = np.random.default_rng(75)
    frames, stream_rows, groups, spans = [], [], [], []
    for s in range(32):
        R = rng.integers(0, 256, (20, 1000, 32), dtype=np.uint8)
        free = [list(rng.permutation(1000)) for _ in range(20)]
        n_pts = int(rng.integers(1400, 1601))
        f0 = len(frames)
        for _ in range(n_pts):
            N = int(min(2 + rng.geometric(1 / 7), 30))
            kfs = rng.choice(20, N, replace=N > 20)
            ks = np.array([free[kf].pop() for kf in kfs])
            noise = rng.random((N, 256)) < rng.uniform(0, 0.2, (N, 1))
            R[kfs, ks] = rng.integers(0, 256, 32, dtype=np.uint8) ^ np.packbits(noise, axis=1)
            groups.append((kfs + f0, ks))
        spans.append((len(groups) - n_pts, len(groups), f0))
        frames += [resident(M, mt, R[i], rng) for i in range(20)]
        stream_rows.append(R)
    c0 = launches(mt)
    best, desc = mt.ComputeDistinctiveDescriptorsFrames(frames, groups)
    assert launches(mt) - c0 == 1
    for s, (p0, p1, f0) in enumerate(spans):
        gathered = [stream_rows[s][f - f0, k] for f, k in groups[p0:p1]]
        want = mt.ComputeDistinctiveDescriptors(gathered)
        assert np.array_equal(best[p0:p1], want), s
        assert np.array_equal(desc[p0:p1], np.stack([g[b] for g, b in zip(gathered, want)])), s
        if s == 0:
            assert all(best[p0 + i] == oracle.port_distinctive_descriptor(g) for i, g in enumerate(gathered[:300]))


def test_frames_of_other_handles(M, oracle, world):
    """Frames created by another matcher handle, on its own stream, are read once they are complete (the call waits on their
    ready events), including frames the other handle created just before the call."""
    mt, named, rows = world
    other = M.ORBmatcher()
    rng = np.random.default_rng(76)
    fresh_rows = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (2000, 8192, 700)]
    fresh = [resident(M, other, r, rng) for r in fresh_rows]
    frames = fresh + [F for _, F in named]
    all_rows = fresh_rows + rows
    groups = shape_points(rng, all_rows, len(fresh) + CRAFTED)
    groups += [(np.array([0, 1, 2, 1]), np.array([1999, 8191, 699, 0]))]
    check_points(mt, oracle, frames, all_rows, groups)


def test_argument_errors(M, world):
    """Each refused argument returns BORB_ERR_INVALID_ARG with an error text naming the point or frame-table entry, no launch, and
    best_idx / desc_out untouched; no observation at all means no launch."""
    from orb_slam2_b200 import _lib
    mt, named, rows = world
    lib = mt._lib
    good = [F.resident for _, F in named[:3]]
    n0 = good[0].n

    def call(handles, n_frames, obs_f, obs_k, off, n_points, best=True, desc=True):
        out_b = np.full(max(n_points, 1), 77, np.int32)
        out_d = np.full((max(n_points, 1), 32), 99, np.uint8)
        obs_f, obs_k, off = [np.ascontiguousarray(a, np.int32) for a in (obs_f, obs_k, off)]
        c0 = launches(mt)
        st = lib.borb_distinctive_descriptors_frames(mt._h, handles, n_frames, obs_f.ctypes.data, obs_k.ctypes.data, off.ctypes.data,
                                                     n_points, out_b.ctypes.data if best else None, out_d.ctypes.data if desc else None)
        return st, lib.borb_last_error().decode(), launches(mt) - c0, out_b, out_d

    def table(fs):
        return (C.c_void_p * len(fs))(*[f._h.value if f is not None else None for f in fs])

    def refused(text, *args, **kw):
        st, err, nl, b, d = call(*args, **kw)
        assert st == 1 and text in err and nl == 0, (st, err, nl)
        assert np.all(b == 77) and np.all(d == 99)

    ok_f, ok_k, ok_off = [0, 1, 2], [0, 1, 2], [0, 2, 3]
    st, err, nl, b, d = call(table(good), 3, ok_f, ok_k, ok_off, 2)
    assert st == 0 and nl == 1 and b[0] >= 0 and b[1] == 0
    refused("frame 1:", table([good[0], None, good[2]]), 3, ok_f, ok_k, ok_off, 2)
    refused("point 1:", table(good), 3, [0, 1, 3], ok_k, ok_off, 2)
    refused("point 0:", table(good), 3, [-1, 1, 2], ok_k, ok_off, 2)
    refused("point 1:", table(good), 3, [0, 0, 0], [0, 1, n0], ok_off, 2)
    refused("point 0:", table(good), 3, [0, 0, 0], [-1, 1, 2], ok_off, 2)
    refused("point 0:", table(good), 3, ok_f, ok_k, [1, 2, 3], 2)
    refused("point 1:", table(good), 3, ok_f, ok_k, [0, 2, 1], 2)
    big = 1 << 16
    refused("point 1:", table(good), 3, np.zeros(big + 1, np.int32), np.zeros(big + 1, np.int32), [0, 1, big + 1], 2)
    refused("null", table(good), 3, ok_f, ok_k, ok_off, 2, best=False)
    refused("null", table(good), 3, ok_f, ok_k, ok_off, 2, desc=False)
    if _lib.device_count() > 1:
        far_mt = M.ORBmatcher(device=1)
        far = resident(M, far_mt, rows[0][:100], np.random.default_rng(77)).resident
        refused("frame 2 ", table([good[0], good[1], far]), 3, ok_f, ok_k, ok_off, 2)
    st, err, nl, b, d = call(table(good), 3, [0], [0], [0, 0, 0], 2)             # points without observations: no launch
    assert st == 0 and nl == 0 and np.all(b[:2] == -1) and np.all(d == 99)
    st, err, nl, b, d = call(None, 0, [0], [0], [0], 0, best=False, desc=False)   # nothing at all
    assert st == 0 and nl == 0
