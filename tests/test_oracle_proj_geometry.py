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
