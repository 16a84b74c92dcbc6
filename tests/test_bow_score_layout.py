"""CPU: the ctypes mirrors of borb_bow_ref and borb_bow_score_job in orb_slam2_b200/matcher.py have the layout include/borb.h gives
them (sizeof and every offsetof, as a C compiler lays the structs out)."""
import ctypes as C
import os
import subprocess
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = {"borb_bow_ref": ("_BowRefC", ("frame", "db", "slot")),
           "borb_bow_score_job": ("_BowScoreJobC", ("query", "targets", "n_targets", "score"))}


def program(struct, fields):
    lines = "\n".join(f'    printf("{f} %zu\\n", offsetof({struct}, {f}));' for f in fields)
    return textwrap.dedent('''
        #include <stddef.h>
        #include <stdio.h>
        #include "borb.h"
        int main(void) {
            printf("size %zu\\n", sizeof(STRUCT));
        FIELDS
            return 0;
        }
    ''').replace("STRUCT", struct).replace("FIELDS", lines)


@pytest.mark.parametrize("struct", sorted(STRUCTS))
def test_bow_score_ctypes_layout_matches_the_header(tmp_path, struct):
    from orb_slam2_b200 import matcher
    cls_name, fields = STRUCTS[struct]
    cls = getattr(matcher, cls_name)
    src = tmp_path / f"{struct}_layout.c"
    src.write_text(program(struct, fields))
    exe = tmp_path / f"{struct}_layout"
    subprocess.check_call(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(cls)
    assert [name for name, _ in cls._fields_] == list(fields)
    for f in fields:
        assert int(out[f]) == getattr(cls, f).offset, f
