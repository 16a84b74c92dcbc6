"""The poisoned-memory catalogue (tests/poison_cases.py) entry of borb_frame_from_extractors: the case that drives it, registered in
the catalogue's CASES and COVERED tables when this module is imported, so that tests/test_poison_catalogue.py accounts for the entry
point and tests/test_gpu_poison.py runs the case under 0x00, 0xFF and 0x7F with the rest of the catalogue."""
from tests import frame_input_cases as fic
from tests import poison_cases as P
from tests.test_cabi import declared_symbols


def fx_ctor(c):
    """borb_frame_from_extractors: a stereo frame on two handles of different nfeatures (XA left, XB right), then an RGB-D frame
    on XA with a float depth map and a distorted camera."""
    M = c.M
    L, R = c.pairs[0]
    c.XA.extract_enqueue(L)
    c.XB.extract_enqueue(R)
    F, hs = M.frame_from_extractors(c.mt, c.XA, c.XB, P.K_CAM, bf=P.BF, fx=P.FX, mode=1)
    K, dist = fic.DIST_CASES["tum1_5"]
    c.XA.extract_enqueue(c.mono[0])
    G, hr = M.frame_from_extractors(c.mt, c.XA, None, K, dist, bf=40.0, mode=2, depth=fic.edge_depth_float(21))
    out = dict(stereo=hs, rgbd=hr, dev=[F.resident.read(stereo=True), G.resident.read(stereo=True)])
    F.resident.close()
    G.resident.close()
    return out


P.CASES.setdefault("fx_ctor", fx_ctor)
P.COVERED.setdefault("borb_frame_from_extractors", ("fx_ctor",))


def test_catalogue_drives_the_constructor():
    assert "borb_frame_from_extractors" in declared_symbols()
    assert P.CASES["fx_ctor"] is fx_ctor and P.COVERED["borb_frame_from_extractors"] == ("fx_ctor",)
    assert "borb_frame_from_extractors" not in P.NOT_COVERED
