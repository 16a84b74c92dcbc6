"""CPU: the port (oracle/orb_port_*.cpp) equals the verbatim Frame.cc / ORBmatcher.cc on the non-finite and int-overflowing cases
of tests/nonfinite_cases.py, the verbatim build decides the two members of every pair differently, every class is reached, and
every float-to-int conversion of the device code is in the inventory."""
import numpy as np
import pytest

from tests import nonfinite_cases as N
from tests import test_oracle_proj_geometry as TG

CASES = N.cases()


@pytest.fixture(scope="module")
def O(oracle):
    if not (oracle.have_matchref() and oracle.have_frameref()):
        pytest.skip("oracle/_ref/libmatchref.so or libframeref.so not built (reference tree absent)")
    return oracle


def port_equals_reference(O, c, method):
    got, want = N.run_port(O, c, method), N.run_ref(O, c, method)
    if method == "grid":
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), (got, want)
    elif method == "init":
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and N.G.same_float(got[2], want[2]), (got, want)
    else:
        TG.port_equals_reference(O, c, method)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['cls']}-{c['member']}" for c in CASES])
def test_port_equals_reference(O, i):
    c = CASES[i]
    for method in N.methods(c):
        port_equals_reference(O, c, method)


@pytest.mark.parametrize("cls", sorted(N.CLASSES))
def test_pair_members_are_decided_differently(O, cls):
    pair = {c["member"]: c for c in CASES if c["cls"] == cls}
    assert sorted(pair) == [0, 1]
    assert N.decided(O, pair[0]) is True and N.decided(O, pair[1]) is False, cls


def test_every_class_is_reached():
    assert {c["cls"] for c in CASES} == set(N.CLASSES)
    assert not set(N.CLASSES) & set(N.NOT_COVERED)


def test_pairs_sit_on_their_bounds():
    """The radius pairs put the window's far edge one float step below 2^31 and on it; the grid pairs put the finite key into
    column / row 0, the cell the device conversion of NaN (0) would give."""
    assert N.x86_int(np.float32(np.nan)) == N.INT_MIN and N.x86_int(np.float32(np.inf)) == N.INT_MIN
    assert N.x86_int(np.float32(2.0 ** 31)) == N.INT_MIN and N.x86_int(N.G.step(2.0 ** 31, -1)) == 2 ** 31 - 128
    assert N.x86_int(np.float32(-2.0 ** 31)) == N.INT_MIN and N.x86_int(np.float32(-0.5)) == 0
    for c in CASES:
        if c.get("kind") == "grid":
            k = c["F"].mvKeysUn[c["key"]]
            cell = N.grid_cell(c["F"].bounds, k["x"], k["y"])
            assert (cell is None) == bool(c["member"]), c["cls"]
            if cell is not None:
                assert cell[0 if c["cls"] == "grid_nan_x" else 1] == 0
    edges = {}
    for c in CASES:
        if c["cls"].startswith("radius_th") and c["cls"] != "radius_th_proj":
            x = np.float32(np.float32(np.float32(N.G.U0) + np.float32(c["th"])) * np.float32(0.1))
            edges.setdefault(c["cls"], []).append(np.ceil(x))
    for cls, (a, b) in edges.items():
        assert a < 2.0 ** 31 <= b, cls


@pytest.mark.parametrize("bounds", [(0.0, 0.0, 640.0, 480.0), (3.75, 2.5, 636.0, 478.25)])
def test_grid_with_nan_keys_port_equals_reference(O, bounds):
    """NaN, +-inf and +-FLT_MAX keys among ordinary ones: the port's grid (restated PosInGrid) equals Frame.cc cell by cell, and
    every non-finite key is in no cell."""
    k = N.G._keys([(x, y) for x in (0.0, 17.5, 320.0, 620.0) for y in (0.0, 33.0, 460.0)])
    specials = np.array([np.nan, np.inf, -np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max], np.float32)
    extra = N.G._keys([(0.0, 0.0)] * (2 * len(specials)))
    extra["x"][:len(specials)] = specials; extra["y"][:len(specials)] = 10.0
    extra["y"][len(specials):] = specials; extra["x"][len(specials):] = 10.0
    keys = np.concatenate([k, extra])
    cs_p, ci_p = O.port_assign_grid(keys, bounds)
    cs_r, ci_r = O.ref_assign_grid(keys, bounds)
    assert np.array_equal(cs_p, cs_r) and np.array_equal(ci_p, ci_r)
    assert set(ci_r[:cs_r[-1]].tolist()) == set(range(len(k)))


def test_undistort_calibrations_give_nan_keys(oracle):
    """The borb_frames_from_extractor calibrations of the GPU tests really make the port's UndistortKeyPoints return NaN keys, and
    the port's grid of them (Frame.cc's PosInGrid, pinned by test_grid_with_nan_keys_port_equals_reference) holds no key."""
    keys, _ = oracle.PortExtractor(1000)(N.undistort_image())
    h, w = N.undistort_image().shape
    for K, dist in N.NAN_CALIBRATIONS:
        p = oracle.port_rgbd_frame(keys, np.array(K, np.float32), np.array(dist, np.float32), 40.0, np.zeros((h, w), np.float32))
        ku = p["keys_un"]
        assert len(ku) > 100 and (np.isnan(ku["x"]) | np.isnan(ku["y"])).all(), (K, dist)
        cs, ci = oracle.port_assign_grid(ku, p["bounds"])
        assert cs[-1] == 0
        if oracle.have_frameref():
            cs_r, ci_r = oracle.ref_assign_grid(ku, p["bounds"])
            assert np.array_equal(cs, cs_r)


def test_inventory_lists_every_conversion():
    """Every float-to-int conversion in csrc/k_*.cu and match_rules.cuh has an inventory row naming its input domain and the
    class that covers it or why no non-finite value reaches it; a row whose line is gone fails too."""
    found = N.scan_conversions()
    rows = {(f, line): (dom, cover) for f, line, dom, cover in N.INVENTORY}
    missing = [f"{f}:{lines} {line}" for (f, line), lines in sorted(found.items()) if (f, line) not in rows]
    assert not missing, "conversions without an inventory row:\n" + "\n".join(missing)
    stale = sorted(set(rows) - set(found))
    assert not stale, stale
    assert all(dom and cover for dom, cover in rows.values())
    covered = {w for *_, cover in N.INVENTORY for w in cover.replace(";", " ").split() if w in N.CLASSES}
    assert {"grid_nan_x", "grid_nan_y", "nan_centre_proj_x", "nan_centre_proj_y"} <= covered
