"""CPU: the ctypes mirror of borb_init_job in orb_slam2_b200/matcher.py has the layout include/borb.h gives it (sizeof and every
offsetof, as a C compiler lays the struct out)."""
import ctypes as C
import os
import subprocess
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("initial", "current", "prev_matched", "window_size", "matches12")

PROG = textwrap.dedent('''
    #include <stddef.h>
    #include <stdio.h>
    #include "borb.h"
    int main(void) {
        printf("size %zu\\n", sizeof(borb_init_job));
    FIELDS
        return 0;
    }
''').replace("FIELDS", "\n".join(f'    printf("{f} %zu\\n", offsetof(borb_init_job, {f}));' for f in FIELDS))


def test_init_job_ctypes_layout_matches_the_header(tmp_path):
    from orb_slam2_b200.matcher import _InitJobC
    src = tmp_path / "init_job_layout.c"
    src.write_text(PROG)
    exe = tmp_path / "init_job_layout"
    subprocess.check_call(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(_InitJobC)
    assert [name for name, _ in _InitJobC._fields_] == list(FIELDS)
    for f in FIELDS:
        assert int(out[f]) == getattr(_InitJobC, f).offset, f
