"""CPU: the matcher port (oracle/orb_port_match.cpp) equals the verbatim Frame.cc / ORBmatcher.cc on the float decision-boundary
cases of tests/proj_geometry.py, the verbatim build decides the two members of every boundary pair differently, and the cases
reach every class of proj_geometry.CLASSES."""
import numpy as np
import pytest

from tests import proj_geometry as G


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_matchref() and oracle.have_frameref()):
        pytest.skip("oracle/_ref/libmatchref.so or libframeref.so not built (reference tree absent)")
    return oracle


def _ids():
    return [f"{c['cls']}-{c['member']}" for c in G.cases()]


def port_equals_reference(O, c, method):
    """Asserts that the port and the verbatim build agree on one method of case c."""
    got, want = G.run_port(O, c, method), G.run_ref(O, c, method)
    if method == "local":
        fr_p, n_p, match = got
        fr_r, (n_r, owner), mps = want
        assert G.frustum_equal(fr_p, fr_r), (fr_p, fr_r)
        assert n_p == n_r and np.array_equal(O.owner_from_matches(c["F"], mps, match), owner)
    elif method in ("last", "kf", "sim3proj"):
        occ = c["F"].occupied if method != "last" else None
        assert got[0] == want[0] and np.array_equal(O.owner_from_state(occ, got[1]), want[1]), (got, want)
    elif method in ("fuse", "fuse_kf", "sim3"):
        assert got[0] == want[0] and np.array_equal(got[1], want[1]), (got, want)
    elif method == "proj":
        assert got[0] == want[0] and np.array_equal(O.owner_from_matches(c["F"], c["mps"], got[1]), want[1]), (got, want)
    elif method == "tri":
        assert np.array_equal(got, want), (got, want)


@pytest.mark.parametrize("i", range(len(G.cases())), ids=_ids())
def test_port_equals_reference(O, i):
    c = G.cases()[i]
    for method in G.methods(c):
        port_equals_reference(O, c, method)


@pytest.mark.parametrize("cls", sorted(G.CLASSES))
def test_pair_members_are_decided_differently(O, cls):
    pair = {c["member"]: c for c in G.cases() if c["cls"] == cls}
    assert sorted(pair) == [0, 1]
    assert G.decided(O, pair[0]) is True and G.decided(O, pair[1]) is False, cls


def test_camera_centre_point_is_in_view_with_nan_track_fields(O):
    """Frame::isInFrustum of a point at the camera centre with mfMinDistance == 0: in view, u = v = u_r = viewCos = NaN, level
    0 — and SearchByProjection then finds no candidate for it."""
    c = next(c for c in G.cases() if c["cls"] == "camera_centre" and c["member"] == 0)
    for fr in (G.run_ref(O, c, "local")[0], G.run_port(O, c, "local")[0]):
        assert fr["in_view"][0] == 1 and fr["level"][0] == 0
        assert all(np.isnan(fr[f][0]) for f in G.FLOAT_FIELDS)
    fr, n, match = G.run_port(O, c, "local")
    assert match[0] == -1 and (match[1:] >= 0).all()


def test_every_class_is_reached():
    assert {c["cls"] for c in G.cases()} == set(G.CLASSES)
    assert set(G.DECIDER) | {c["cls"] for c in G.cases() if "kind" in c} == set(G.CLASSES)
    assert not set(G.CLASSES) & set(G.NOT_COVERED)


def test_reference_pose_arithmetic_is_restated(O):
    """The camera centres and the identity Sim3 the cases hand to the port (and to the CUDA library, where the reference is
    absent) are bit for bit what the reference computes."""
    bits = lambda a: np.asarray(a, np.float32).view(np.uint32)
    for c in G.cases():
        if "kind" not in c:
            assert np.array_equal(bits(O.ref_camera_center(c["Tcw"])), bits(c["Ow"])), c["cls"]
    S12, S21 = O.ref_sim3_mats(1.0, np.eye(3, dtype=np.float32), np.zeros(3, np.float32))
    assert np.array_equal(bits(S12), bits(G.S12_ID)) and np.array_equal(bits(S21), bits(G.S21_ID))
    for sim in (G.SIM_A, G.SIM_B):
        S12, S21 = O.ref_sim3_mats(*sim)
        mine = G.sim3_mats(*sim)
        assert np.array_equal(bits(S12), bits(mine[0])) and np.array_equal(bits(S21), bits(mine[1]))
    for c in G.cases():
        if c.get("kind") == "sim3":
            assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(O.ref_sim3_mats(*c["sim"]), (c["S12"], c["S21"]))), c["cls"]


def test_forward_backward_is_restated(O):
    """The forward / backward flags the cases hand to the port and to the CUDA library are the reference's own decision
    (ORBmatcher.cc:1338-1349) on the case's two poses."""
    n = 0
    for c in G.cases():
        if "Tlast" in c:
            assert O.ref_forward_backward(c["Tcw"], c["Tlast"], G.MB, False) == (c["fwd"], c["bwd"]), (c["cls"], c["member"])
            assert G.forward_backward(c["Tcw"], c["Tlast"]) == (c["fwd"], c["bwd"])
            n += 1
    assert n == 2 * (len(G.LEVEL_PAIRS) + 2)
    flags = {(c["fwd"], c["bwd"]) for c in G.cases() if "Tlast" in c}
    assert flags == {(True, False), (False, True), (False, False)}


def test_pairs_sit_on_their_bounds():
    """The kept member of each pair sits exactly on the bound where the gate is strict or inclusive, so that < and <= (or the
    float and double forms of a test) are told apart by the pair."""
    cs = {(c["cls"], c["member"]): c for c in G.cases()}
    P0 = np.array(G.U0_CAM, np.float32) - G.T_CW[:, 3]
    PO, dist = G.norm_po(P0)
    assert np.float32(np.float32(0.8) * cs["frustum_min_dist", 0]["P"].min_distance[0]) == dist
    assert G.project_frustum(G.cam_point(G.T_CW, P0)) == (G.U0, G.V0)
    assert G.epipole() == (G.U0, G.V0)
    assert np.float32(np.float32(1.2) * cs["frustum_max_dist", 0]["P"].max_distance[0]) == dist
    z = [G.cam_point(cs["pcz_sign", m]["Tcw"], cs["pcz_sign", m]["P"].world_pos[0])[2] for m in (0, 1)]
    assert z[0] == 0 and np.signbit(z[0]) and z[1] < 0
    half32 = np.float32(np.float32(0.5) * dist)
    in_float = [not (G.dot32(PO, cs["fuse_normal_dot", m]["P"].normal[0]) < half32) for m in (0, 1)]
    assert in_float != [True, False]                       # the float form of the viewing-angle test decides the pair otherwise
    y = [cs["tri_dsqr", m]["kf1"].mvKeysUn["y"][0] for m in (0, 1)]
    o = cs["tri_dsqr", 0]["kf2"].mvKeysUn["octave"][0]
    assert [np.float32(v * v) < np.float32(np.float32(3.84) * G.SIGMA2[o]) for v in y] != [True, False]
    # tlc.z == mb exactly in the rejected members of fwd_bwd_mb_*, one step beyond it in the kept ones
    tlc = {k: G.cam_point(c["Tlast"], G.camera_centre(c["Tcw"]))[2] for k, c in cs.items() if k[0].startswith("fwd_bwd_mb")}
    assert tlc["fwd_bwd_mb_fwd", 1] == G.MB and tlc["fwd_bwd_mb_fwd", 0] == G.step(G.MB, 1)
    assert tlc["fwd_bwd_mb_bwd", 1] == -G.MB and tlc["fwd_bwd_mb_bwd", 0] == -G.step(G.MB, 1)
    # PredictScale: the ratio of the lower member is sf^2 as the float pyramid holds it, the upper member's one step above
    a, b = G.predict_scale_pair()
    assert np.float32(a / dist) == np.float32(G.SCALE[2] / G.SCALE[0]) and G.predict_scale(a, dist) == G.PS_LEVEL
    assert G.predict_scale(b, dist) == G.PS_LEVEL + 1
    # SearchBySim3: dist3D is the norm of the chained camera-frame point, and the kept member sits on the bound
    d3, (mn, _), (_, mx) = G.sim3_dist_pairs()
    for side in (12, 21):
        c = cs[f"sim3_min_dist_{side}", 0]
        P, T, S = (c["P1"], c["T1w"], c["S21"]) if side == 12 else (c["P2"], c["T2w"], c["S12"])
        pc = G.sim3_chain(T, S, P.world_pos[0])
        assert G.norm3(pc) == d3 and np.float32(np.float32(0.8) * P.min_distance[0]) == d3 and P.min_distance[0] == mn
        other = G.norm3(G.cam_point(T, P.world_pos[0])) / d3         # the chain's other point: outside [0.8, 1.2] times as far
        assert not 0.5 < other < 1.5, other
        c = cs[f"sim3_max_dist_{side}", 0]
        P = c["P1"] if side == 12 else c["P2"]
        assert np.float32(np.float32(1.2) * P.max_distance[0]) == d3 and P.max_distance[0] == mx
    for side, key in ((12, ("P1", "T1w", "S21")), (21, ("P2", "T2w", "S12"))):
        z = [G.sim3_chain(cs[f"sim3_depth_{side}", m][key[1]], cs[f"sim3_depth_{side}", m][key[2]], cs[f"sim3_depth_{side}", m][key[0]].world_pos[0])
             for m in (0, 1)]
        z_other = [G.cam_point(cs[f"sim3_depth_{side}", m][key[1]], cs[f"sim3_depth_{side}", m][key[0]].world_pos[0])[2] for m in (0, 1)]
        assert z[0][2] > 0 > z[1][2] and min(z_other) > 0


def test_level_pairs_straddle_their_windows():
    """Each level_* pair puts the kept member's key octave inside the window of its mode and the rejected member's outside,
    restated from GetFeaturesInArea (Frame.cc:327-380) with the windows of ORBmatcher.cc:1385-1390."""
    def inside(mode, o, ko):
        lo, hi = {"fwd": (o, -1), "bwd": (0, o), "none": (o - 1, o + 1)}[mode]
        if not (lo > 0 or hi >= 0):
            return True
        return ko >= lo and (hi < 0 or ko <= hi)
    assert {o for members in G.LEVEL_PAIRS.values() for _, o, _ in members} == {0, 3, 7}
    for cls, (kept, rejected) in G.LEVEL_PAIRS.items():
        assert inside(*kept) and not inside(*rejected), cls
        assert all(0 <= ko < G.N_LEVELS for _, _, ko in (kept, rejected))


def test_rotation_boundaries_are_placed():
    """rot = -0.0 is bin 0 and rot = -2^-149 is bin 12 (360.0f*(1/30), not wrapped); the x.5 pair has the product exactly 0.5
    (bin 1, half away from zero) and one step below it (bin 0), where floor(x + 0.5f) would give 1."""
    b = G.rot_boundaries()
    assert [G.rot_bin(*a) for a in b["zero"]] == [0, 12]
    assert [G.rot_bin(*a) for a in b["half"]] == [1, 0]
    lo, hi = G.rot_half_pair()
    assert np.float32(hi * G.FACTOR) == 0.5 and np.floor(np.float32(np.float32(lo * G.FACTOR) + np.float32(0.5))) == 1
    for bins in G.ROT_BINS.values():
        counts = sorted(np.bincount(bins, minlength=30), reverse=True)
        assert counts[:4] == [3, 3, 2, 1] and bins.count(0 if bins[0] == 0 else 1) == 3


def test_area_edge_keys_lie_in_the_window_edge_cell():
    """The key each area_edge_* pair keeps sits in the window's edge cell on its side, so a window one cell narrower there
    would lose the match (Frame.cc:332-344 and PosInGrid, restated)."""
    for c in G.cases():
        if not c["cls"].startswith("area_edge") or c["member"] != 0:
            continue
        _, _, axis, side = G.AREA_EDGES[c["cls"]]
        k = c["F"].mvKeysUn[0]
        cell = G.grid_cell(c["F"], k["x"], k["y"])
        win = G.area_window(c["F"], c["mps"].mTrackProjX[0], c["mps"].mTrackProjY[0], G.AREA_R)
        edge = win[2 * axis + (1 if side > 0 else 0)]
        assert cell is not None and cell[axis] == edge, (c["cls"], cell, win)


DENSE = G.dense_classes()


@pytest.mark.parametrize("cls", DENSE)
def test_dense_port_equals_reference(O, cls):
    """Both members of every world-point class inside a natural ~1000-point call: the port equals the verbatim build on every
    method, and the verbatim build still decides the boundary point differently between the two members."""
    pair = {c["member"]: G.dense_case(O, c) for c in G.cases() if c["cls"] == cls and "kind" not in c}
    for c in pair.values():
        assert len(c["P"].world_pos) > 500
        for method in G.methods(c):
            port_equals_reference(O, c, method)
    assert G.decided(O, pair[0]) is True and G.decided(O, pair[1]) is False, cls
