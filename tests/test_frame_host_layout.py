"""CPU: the ctypes mirror of borb_frame_host in orb_slam2_b200/matcher.py has the layout include/borb.h gives it (sizeof and every
offsetof, as a C compiler lays the struct out)."""
import ctypes as C
import os
import subprocess

from tests.test_bow_score_layout import ROOT, program

FIELDS = ("cap", "keys", "desc", "keys_right", "desc_right", "keys_un", "u_right", "depth", "cell_start", "cell_idx", "n", "n_right",
          "bounds")


def test_frame_host_ctypes_layout_matches_the_header(tmp_path):
    from orb_slam2_b200 import matcher
    src = tmp_path / "frame_host_layout.c"
    src.write_text(program("borb_frame_host", FIELDS))
    exe = tmp_path / "frame_host_layout"
    subprocess.check_call(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    cls = matcher._FrameHostC
    assert int(out["size"]) == C.sizeof(cls)
    assert [name for name, _ in cls._fields_] == list(FIELDS)
    for f in FIELDS:
        assert int(out[f]) == getattr(cls, f).offset, f
