"""CPU: the rBRIEF tap order of describe_kernel (borb_debug_brief_slots).  Every orientation bin must fetch each of the 512
pattern points exactly once, with the pattern's own coordinates, or descriptors would change; the points are sorted by their
rotated row at the bin's centre angle, which is what keeps one gather instruction on a few adjacent rows."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def table():
    import __graft_entry__ as g
    from orb_slam2_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        g.build()
    so = _lib.load()
    nb = C.c_int32(0)
    _lib.check(so.borb_debug_brief_slots(None, 0, C.byref(nb)), "borb_debug_brief_slots")
    t = np.zeros(nb.value * 512, np.uint32)
    _lib.check(so.borb_debug_brief_slots(t.ctypes.data, t.size, C.byref(nb)), "borb_debug_brief_slots")
    return t.reshape(nb.value, 512)


def pattern_points():
    """bit_pattern_31_ from the oracle's copy: (512, 2) int, point 2t + i = point i of test t."""
    with open(os.path.join(ROOT, "oracle", "orb_pattern.inc")) as f:
        body = "\n".join(ln for ln in f.read().splitlines() if not ln.lstrip().startswith("//"))
    return np.array([int(v) for v in re.findall(r"-?\d+", body)], np.int64).reshape(512, 2)


def decode(t):
    t = t.astype(np.int64)
    return (t & 0xFF) - 128, ((t >> 8) & 0xFF) - 128, t >> 16


def test_bin_count(table):
    assert table.shape[0] in (16, 32, 64)


def test_every_bin_is_a_permutation_of_the_pattern(table):
    pts = pattern_points()
    for b, row in enumerate(table):
        x, y, p = decode(row)
        assert np.array_equal(np.sort(p), np.arange(512)), f"bin {b}: not a permutation of the 512 points"
        assert np.array_equal(x, pts[p, 0]) and np.array_equal(y, pts[p, 1]), f"bin {b}: coordinates differ from the pattern"


def test_rows_ascend_at_the_bin_centre(table):
    nb = table.shape[0]
    spans = []
    for b, row in enumerate(table):
        x, y, _ = decode(row)
        th = (b + 0.5) * 2 * np.pi / nb
        r = np.floor(x * np.sin(th) + y * np.cos(th) + 0.5)
        assert np.all(np.diff(r) >= 0), f"bin {b}: rotated rows not ascending"
        spans.append(np.mean([len(np.unique(r[k:k + 32])) for k in range(0, 512, 32)]))
    print(f"{nb} bins: rotated rows per 32-lane gather at the bin centre, mean {np.mean(spans):.2f}, worst bin {np.max(spans):.2f}")
    assert np.max(spans) <= 4.0
