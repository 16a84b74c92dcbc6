"""GPU: no result of libborb depends on memory a call did not write.  The catalogue of tests/poison_cases.py runs once with poisoning
off (the baseline: the fixtures' own tests pin these inputs to the port) and again with every reused or recycled buffer filled with
0x00, 0xFF and 0x7F before each call writes it (borb_debug_set_poison); every output must be byte-identical to the baseline.
0x00 leaves counters and "found" flags at zero, 0xFF every int at -1 (the "no match" value) and every float NaN, 0x7F large positive
ints and floats near 3.4e38 that match no sentinel: a kernel that skips writing -1 passes under 0xFF only, one that drops a counter
memset under 0x00 only.  The positive controls read back memory the library never writes, so a switch that did nothing fails."""
import ctypes as C

import numpy as np
import pytest

from tests import poison_cases as P

pytestmark = pytest.mark.gpu

BYTES = (0x00, 0xFF, 0x7F)


def run_catalogue(ctx):
    """{case: outputs or the exception text} for every case of the catalogue, in catalogue order."""
    got = {}
    for name, case in P.CASES.items():
        try:
            got[name] = P.outputs(case(ctx))
        except Exception as e:          # noqa: BLE001 - reported per case by the tests below
            got[name] = f"{type(e).__name__}: {e}"
    return got


@pytest.fixture(scope="module")
def world(oracle):
    from orb_slam2_b200 import _lib
    so = _lib.load()
    so.borb_debug_set_poison(-1)
    ctx = P.Ctx(oracle)
    try:
        yield dict(so=so, lib=_lib, ctx=ctx, base=run_catalogue(ctx))
    finally:
        so.borb_debug_set_poison(-1)         # no later module inherits the switch
        ctx.close()


def test_baseline_runs(world):
    failed = {n: r for n, r in world["base"].items() if isinstance(r, str)}
    assert not failed, failed


def test_frame_from_view_has_no_depth(world):
    """borb_frame_create keeps the view's mvuRight and writes no mvDepth, so borb_debug_frame_read refuses the depth of such a frame
    (BORB_ERR_INVALID_ARG) instead of returning what an earlier frame left in the recycled block."""
    out = world["base"]["mt_frame_create"]
    assert not isinstance(out, str), out
    assert np.frombuffer(out["out.depth_status"][2], np.int32)[0] == 1
    v = world["ctx"].big
    assert out["out.ur"][2] == np.ascontiguousarray(v["ur"][:1000], np.float32).tobytes()
    assert out["out.stereo.keys_un"][2] == np.ascontiguousarray(v["kl"][:1000]).tobytes()


@pytest.mark.parametrize("byte", BYTES, ids=[f"0x{b:02X}" for b in BYTES])
def test_poisoned_run_equals_baseline(world, byte):
    so, base = world["so"], world["base"]
    assert so.borb_debug_set_poison(byte) == 0
    try:
        got = run_catalogue(world["ctx"])
    finally:
        assert so.borb_debug_set_poison(-1) == 0
    diffs = []
    for name, want in base.items():
        have = got[name]
        if isinstance(want, str) or isinstance(have, str):
            diffs.append((name, have if isinstance(have, str) else "baseline failed"))
            continue
        if set(have) != set(want):
            diffs.append((name, sorted(set(have) ^ set(want))[:5]))
            continue
        diffs += [(name, k) for k in sorted(want) if have[k] != want[k]]
    cases = sorted({n for n, _ in diffs})
    assert not diffs, (f"{len(diffs)} outputs of {cases} differ", diffs[:20])


def test_positive_control(world):
    """With poisoning on, memory no call writes holds the byte.
    - borb_extract copies `cap` keypoints and descriptors per image from the workspace; describe_kernel writes only the first n, so
      entries n..cap-1 are the extraction step's fill of ws.kps / ws.desc.
    - borb_frames_from_extractor copies n_frames x cap host keypoints out of the matcher's result region; frame_build_kernel writes
      the first n_keys[i] of frame i, so a frame with fewer keypoints than cap returns the Call's fill of the arena after them."""
    so, lib, ctx = world["so"], world["lib"], world["ctx"]
    byte = 0x5A
    assert so.borb_debug_set_poison(byte) == 0
    try:
        X = ctx.XA
        img = np.ascontiguousarray(ctx.mono[0])
        h, w = img.shape
        cap = X.capacity(w, h)
        kps = np.zeros(cap, lib.KP_DTYPE); desc = np.zeros((cap, 32), np.uint8); n = C.c_int32(0)
        lib.check(so.borb_extract(X._h, img.ctypes.data, w, h, w, lib.ptr(kps), lib.ptr(desc), cap, C.byref(n)), "borb_extract")
        X._last_n = 1
        assert 0 < n.value < cap
        assert set(kps[n.value:].tobytes()) == {byte} and set(desc[n.value:].tobytes()) == {byte}

        outs = X.extract_batch(ctx.mono[:2])
        nk = np.array([len(outs[0][0]), len(outs[1][0]) // 2], np.int32)
        fcap = int(nk.max())
        ku = np.zeros((2, fcap), lib.KP_DTYPE)
        cam = ctx.M._CameraC(*P.K_CAM, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
        b4 = np.zeros(4, np.float32)
        handles = (C.c_void_p * 2)()
        images = np.array([0, 1], np.int32)
        lib.check(so.borb_frames_from_extractor(ctx.mt._h, X._h, lib.ptr(images), 2, lib.ptr(nk), C.byref(cam), 0, None, 0, 1.0, 0,
                                                lib.ptr(ku), None, None, fcap, lib.ptr(b4), handles), "borb_frames_from_extractor")
        for hnd in handles:
            so.borb_frame_destroy(hnd)
        short = int(nk.argmin())
        assert nk[short] < fcap
        assert set(ku[short, nk[short]:].tobytes()) == {byte}
        assert ku[short, :nk[short]].tobytes() != bytes([byte]) * (int(nk[short]) * 28)
    finally:
        assert so.borb_debug_set_poison(-1) == 0
