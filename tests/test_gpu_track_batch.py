"""GPU parity of the batched Tracking-thread searches: borb_search_local_points_batch (Tracking::SearchLocalPoints of many
camera streams) and borb_search_by_projection_last_batch (SearchByProjection(CurrentFrame, LastFrame) of many streams).  Every
job must equal the oracle restatement and the single call bit for bit; the batch is one launch sequence whatever its size, and
argument errors are refused before anything is launched."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from tests import match_fixtures as mf

pytestmark = pytest.mark.gpu

BF = 40.0


@pytest.fixture(scope="module")
def M():
    from orb_slam2_b200 import matcher
    return matcher


@pytest.fixture(scope="module")
def views(oracle):
    return {s: mf.two_views(oracle, s) for s in (7, 8)}


def launches(mt):
    n = C.c_uint64(0)
    assert mt._lib.borb_matcher_launch_count(mt._h, C.byref(n)) == 0
    return n.value


def reanchor(a, Pw, Tcw, normal=None):
    """The same scene in another world frame: a rotation by `a` about y and a shift, so that every job has its own pose."""
    Rg = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    tg = np.array([0.7 * a, -0.2, 1.5 * a])
    Pw2 = (Pw.astype(np.float64) @ Rg.T + tg).astype(np.float32)
    R, t = Tcw[:, :3].astype(np.float64), Tcw[:, 3].astype(np.float64)
    T2 = np.zeros((3, 4), np.float32)
    T2[:, :3] = R @ Rg.T
    T2[:, 3] = t - R @ Rg.T @ tg
    Ow = (-(T2[:, :3].T @ T2[:, 3])).astype(np.float32)
    n2 = None if normal is None else (normal.astype(np.float64) @ Rg.T).astype(np.float32)
    return Pw2, T2, Ow, n2


def take(P, idx, valid=None):
    """P restricted to / repeated along idx."""
    return dataclasses.replace(P, world_pos=P.world_pos[idx], descriptors=P.descriptors[idx], max_distance=P.max_distance[idx],
                               min_distance=P.min_distance[idx], normal=P.normal[idx], angle=P.angle[idx],
                               valid=valid if valid is not None else (None if P.valid is None else P.valid[idx]))


def local_job(M, v, seed, a, idx=None, valid="fixture", occupied=True, has_obs=True):
    F, P, Tcw, _, K = mf.world_points_case(v, seed)
    F = M.FrameView(F.mvKeysUn, F.mDescriptors, F.mvScaleFactors, F.bounds, mvuRight=v["ur"], occupied=F.occupied if occupied else None)
    Pw, T2, Ow, nr = reanchor(a, P.world_pos, Tcw, P.normal)
    P = dataclasses.replace(P, world_pos=Pw, normal=nr)
    if idx is not None:
        P = take(P, idx)
    if valid is None:
        P = dataclasses.replace(P, valid=None)
    elif isinstance(valid, str) and valid == "none":
        P = dataclasses.replace(P, valid=np.zeros(len(P.world_pos), np.uint8))
    elif not isinstance(valid, str):
        P = dataclasses.replace(P, valid=valid)
    rng = np.random.default_rng(seed)
    ho = (rng.random(len(P.world_pos)) < 0.9).astype(np.uint8) if has_obs else None
    return F, P, (T2, Ow), K, ho


def oracle_local(M, oracle, F, P, pose, K, th, ratio, ho):
    fr = oracle.port_is_in_frustum(F, P, pose[0], pose[1], K, BF, 0.5)
    mps = M.MapPointsView(fr["proj_x"], fr["proj_y"], fr["proj_xr"], fr["level"], fr["view_cos"], P.descriptors, valid=fr["in_view"],
                          has_obs=ho)
    n_o, m_o = oracle.port_search_by_projection(F, mps, th, ratio)
    return fr, n_o, m_o


FIELDS = ("in_view", "proj_x", "proj_y", "proj_xr", "level", "view_cos", "match")


def test_local_points_batch_equals_oracle_and_single_calls(M, oracle, views):
    mt = M.ORBmatcher(0.8, True)
    n_rep = 9                                                   # a local map longer than BORB_MATCH_MAX_FEATURES
    n_kr = len(views[7]["kr"])
    rng = np.random.default_rng(3)
    long_idx = np.tile(np.arange(n_kr), n_rep)
    long_valid = (rng.random(len(long_idx)) < 0.08).astype(np.uint8)
    specs = [  # (seed view, fixture seed, angle, th, idx, valid, occupied, has_obs)
        (7, 77, 0.00, 1.0, None, "fixture", True, True),       # ~900 valid: 1024-thread resolve
        (8, 78, 0.10, 3.0, np.arange(150), "fixture", False, False),   # < 256 valid next to the large ones
        (7, 79, -0.10, 5.0, np.arange(0), "fixture", True, True),     # empty list
        (8, 80, 0.20, 3.0, None, "none", True, True),         # no valid point
        (7, 81, 0.05, 3.0, long_idx, long_valid, True, True),  # > 8192 points, ~700 valid
        (8, 82, -0.05, 1.0, None, None, True, True),           # valid = NULL
        (7, 83, 0.15, 5.0, np.arange(300), "fixture", False, True),
    ]
    assert len(long_idx) > 8192 and 512 < long_valid.sum() < 8192
    frames, points, poses, Ks, ths, obs = [], [], [], [], [], []
    for (s, fs, a, th, idx, valid, occ, ho_on) in specs:
        F, P, pose, K, ho = local_job(M, views[s], fs, a, idx, valid, occ, ho_on)
        frames.append(F); points.append(P); poses.append(pose); Ks.append(K); ths.append(th); obs.append(ho)
    # a frame without features: isInFrustum still runs, nothing can match
    F0, P0, pose0, K0, ho0 = local_job(M, views[8], 84, 0.3, np.arange(200))
    F0 = M.FrameView(F0.mvKeysUn[:0], F0.mDescriptors[:0], F0.mvScaleFactors, F0.bounds)
    frames.append(F0); points.append(P0); poses.append(pose0); Ks.append(K0); ths.append(3.0); obs.append(ho0)
    resident = [dataclasses.replace(F.make_resident(mt), occupied=F.occupied) for F in frames]
    got = mt.SearchLocalPointsBatch(resident, points, poses, Ks, BF, ths, has_obs=obs)
    assert len(got) == len(frames)
    for j, (F, P, pose, K, th, ho) in enumerate(zip(frames, points, poses, Ks, ths, obs)):
        single = mt.SearchLocalPoints(resident[j], P, pose[0], pose[1], K, BF, th, has_obs=ho)
        for f in FIELDS:
            assert np.array_equal(got[j][f], single[f]), (j, f)               # bit-identical floats
        assert got[j]["nmatches"] == single["nmatches"], j
        n = len(P.world_pos)
        if n == 0:
            assert all(len(got[j][f]) == 0 for f in FIELDS) and got[j]["nmatches"] == 0
            continue
        if len(F.mvKeysUn) == 0:
            fr = oracle.port_is_in_frustum(F, P, pose[0], pose[1], K, BF, 0.5)
        else:
            fr, n_o, m_o = oracle_local(M, oracle, F, P, pose, K, th, 0.8, ho)
        assert np.array_equal(got[j]["in_view"], fr["in_view"]), j
        for f in ("proj_x", "proj_y", "proj_xr", "level", "view_cos"):
            assert np.array_equal(got[j][f], fr[f]), (j, f)
        if len(F.mvKeysUn) == 0:
            assert fr["count"] > 20 and np.all(got[j]["match"] == -1) and got[j]["nmatches"] == 0
        else:
            assert got[j]["nmatches"] == n_o and np.array_equal(got[j]["match"], m_o), (j, int((got[j]["match"] != m_o).sum()))
    assert not np.any(got[3]["in_view"]) and np.all(got[3]["match"] == -1) and got[3]["nmatches"] == 0
    assert got[0]["nmatches"] > 30 and got[1]["nmatches"] > 0 and got[4]["nmatches"] > 10 and got[5]["nmatches"] > 30


def last_job(M, v, seed, a, n_last=None):
    Cur, Last, Tcw, K = mf.last_frame_case(v, seed)
    Pw, T2, _, _ = reanchor(a, Last.world_pos, Tcw)
    Last = dataclasses.replace(Last, world_pos=Pw)
    if n_last is not None:
        Last = dataclasses.replace(Last, mvKeysUn=Last.mvKeysUn[:n_last], world_pos=Last.world_pos[:n_last], descriptors=Last.descriptors[:n_last],
                                   valid=Last.valid[:n_last], has_obs=Last.has_obs[:n_last])
    return Cur, Last, T2, K


@pytest.mark.parametrize("ori", [False, True])
def test_last_frame_batch_equals_oracle_and_single_calls(M, oracle, views, ori):
    mt = M.ORBmatcher(0.9, ori)
    specs = [  # (view, fixture seed, angle, th, forward, backward, occupied, n_last)
        (7, 27, 0.00, 7.0, False, False, True, None),
        (8, 28, 0.10, 15.0, True, False, False, None),
        (7, 29, -0.10, 40.0, False, True, True, None),           # lists longer than a warp
        (8, 30, 0.05, 150.0, True, True, True, None),            # lists longer than the sort capacity
        (7, 31, 0.20, 15.0, False, False, False, 100),           # a small job next to the large ones
        (8, 32, -0.20, 7.0, False, True, True, 0),               # empty last frame
        (7, 33, 0.12, 15.0, True, False, True, None),
    ]
    curs, lasts, poses, Ks, ths, fws, bws = [], [], [], [], [], [], []
    for (s, fs, a, th, fw, bw, occ, nl) in specs:
        Cur, Last, T, K = last_job(M, views[s], fs, a, nl)
        if not occ:
            Cur = dataclasses.replace(Cur, occupied=None)
        curs.append(Cur); lasts.append(Last); poses.append(T); Ks.append(K); ths.append(th); fws.append(fw); bws.append(bw)
    # a current frame without features
    Cur0, Last0, T0, K0 = last_job(M, views[8], 34, 0.3, 50)
    curs.append(M.FrameView(Cur0.mvKeysUn[:0], Cur0.mDescriptors[:0], Cur0.mvScaleFactors, Cur0.bounds))
    lasts.append(Last0); poses.append(T0); Ks.append(K0); ths.append(15.0); fws.append(False); bws.append(False)
    resident = [dataclasses.replace(F.make_resident(mt), occupied=F.occupied) for F in curs]
    got = mt.SearchByProjectionLastBatch(resident, lasts, poses, Ks, BF, ths, fws, bws)
    assert len(got) == len(curs)
    culled = 0
    for j in range(len(curs)):
        n_s, s_s = mt.SearchByProjectionLast(resident[j], lasts[j], poses[j], Ks[j], BF, ths[j], fws[j], bws[j])
        n_g, s_g = got[j]
        assert n_g == n_s and np.array_equal(s_g, s_s), (j, int((s_g != s_s).sum()))
        assert len(s_g) == len(curs[j].mvKeysUn)
        if len(curs[j].mvKeysUn) and len(lasts[j].mvKeysUn):
            n_o, s_o = oracle.port_search_by_projection_last(curs[j], lasts[j], poses[j], Ks[j], BF, ths[j], fws[j], bws[j], ori)
            assert n_g == n_o and np.array_equal(s_g, s_o), (j, int((s_g != s_o).sum()))
        else:
            assert n_g == 0 and np.all(s_g == -1)
        culled += int((s_g == -2).sum())
    assert got[0][0] > 20 and got[5][0] == 0
    if not ori:
        assert culled == 0


def test_one_launch_sequence_whatever_the_job_count(M, oracle, views):
    mt = M.ORBmatcher(0.8, True)
    F, P, pose, K, ho = local_job(M, views[7], 77, 0.0)
    FR = F.make_resident(mt)
    Cur, Last, T, K2 = last_job(M, views[8], 28, 0.1)
    CR = Cur.make_resident(mt)
    PF, mps = mf.projection_case(views[7], 100, n_mp=50)
    PR = PF.make_resident(mt)
    deltas = []
    for n in (1, 8):
        c0 = launches(mt)
        mt.SearchLocalPointsBatch([FR] * n, [P] * n, [pose] * n, K, BF, 3.0, has_obs=[ho] * n)
        c1 = launches(mt)
        mt.SearchByProjectionLastBatch([CR] * n, [Last] * n, [T] * n, K2, BF, 15.0)
        c2 = launches(mt)
        mt.SearchByProjectionBatch([PR] * n, [mps] * n, 3.0)
        c3 = launches(mt)
        deltas.append((c1 - c0, c2 - c1, c3 - c2))
    assert deltas[0] == deltas[1] == (3, 3, 2), deltas

    # the single calls: the same sequence on a resident frame, one grid sort more on a host view
    def count(call):
        c0 = launches(mt)
        call()
        return launches(mt) - c0

    for frame, local_frame, cur, grid in ((PR, FR, CR, 0), (PF, F, Cur, 1)):
        assert count(lambda: mt.SearchByProjection(frame, mps, 3.0)) == 2 + grid
        assert count(lambda: mt.SearchLocalPoints(local_frame, P, pose[0], pose[1], K, BF, 3.0, has_obs=ho)) == 3 + grid
        assert count(lambda: mt.SearchByProjectionLast(cur, Last, T, K2, BF, 15.0)) == 3 + grid


def test_argument_errors_name_the_job_and_launch_nothing(M, oracle, views):
    from orb_slam2_b200._lib import BorbError
    mt = M.ORBmatcher(0.8, True)
    F, P, pose, K, ho = local_job(M, views[7], 77, 0.0)
    FR = F.make_resident(mt)

    def refused(call, job):
        c0 = launches(mt)
        with pytest.raises(BorbError) as ei:
            call()
        assert ei.value.status == 1 and f"job {job}:" in str(ei.value), str(ei.value)
        assert launches(mt) == c0

    # a host view
    refused(lambda: mt.SearchLocalPointsBatch([FR, F], [P, P], [pose, pose], K, BF, 3.0), 1)
    # more than BORB_MATCH_MAX_FEATURES valid points
    big = take(P, np.tile(np.arange(len(P.world_pos)), 9), valid=np.ones(9 * len(P.world_pos), np.uint8))
    refused(lambda: mt.SearchLocalPointsBatch([FR, FR, FR], [P, P, big], [pose] * 3, K, BF, 3.0), 2)
    # log_scale_factor <= 0
    FZ = dataclasses.replace(FR, mfLogScaleFactor=0.0)
    refused(lambda: mt.SearchLocalPointsBatch([FR, FZ], [P, P], [pose, pose], K, BF, 3.0), 1)
    FN = dataclasses.replace(FR, mfLogScaleFactor=-0.2)
    refused(lambda: mt.SearchLocalPointsBatch([FN], [P], [pose], K, BF, 3.0), 0)
    # last frame: host view, last-frame octave outside the frame's levels
    Cur, Last, T, K2 = last_job(M, views[8], 28, 0.1)
    CR = Cur.make_resident(mt)
    refused(lambda: mt.SearchByProjectionLastBatch([CR, Cur], [Last, Last], [T, T], K2, BF, 15.0), 1)
    bad = Last.mvKeysUn.copy()
    bad["octave"][5] = len(Cur.mvScaleFactors)
    refused(lambda: mt.SearchByProjectionLastBatch([CR, CR, CR], [Last, Last, dataclasses.replace(Last, mvKeysUn=bad)], [T] * 3, K2, BF, 15.0), 2)
    # SearchByProjection(F, vpMapPoints): host view, predicted level outside the frame's levels
    PF, mps = mf.projection_case(views[7], 100, n_mp=50)
    PR = PF.make_resident(mt)
    refused(lambda: mt.SearchByProjectionBatch([PR, PF], [mps, mps], 3.0), 1)
    lvl = mps.mnTrackScaleLevel.copy()
    lvl[3] = len(PF.mvScaleFactors)
    bad_mps = dataclasses.replace(mps, mnTrackScaleLevel=lvl, valid=None)
    refused(lambda: mt.SearchByProjectionBatch([PR, PR, PR], [mps, mps, bad_mps], 3.0), 2)
    # the handle still works after the refusals
    got = mt.SearchLocalPointsBatch([FR], [P], [pose], K, BF, 3.0, has_obs=[ho])[0]
    single = mt.SearchLocalPoints(FR, P, pose[0], pose[1], K, BF, 3.0, has_obs=ho)
    assert got["nmatches"] == single["nmatches"] > 100 and np.array_equal(got["match"], single["match"])
