"""CPU: the ctypes mirrors of borb_kf_projection_job, borb_sim3_projection_job and borb_sim3_job in orb_slam2_b200/matcher.py have the
layout include/borb.h gives them (sizeof and every offsetof, as a C compiler lays the structs out)."""
import ctypes as C
import os
import subprocess
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = {
    "borb_kf_projection_job": ("_KfProjectionJobC", ("cur", "pts", "Tcw", "Ow", "fx", "fy", "cx", "cy", "log_scale_factor", "th",
                                                     "orb_dist", "state_cur")),
    "borb_sim3_projection_job": ("_Sim3ProjectionJobC", ("kf", "pts", "Tcw", "Ow", "fx", "fy", "cx", "cy", "log_scale_factor", "th",
                                                         "state_kf")),
    "borb_sim3_job": ("_Sim3JobC", ("kf1", "kf2", "pts1", "pts2", "T1w", "T2w", "S12", "S21", "fx", "fy", "cx", "cy",
                                    "log_scale_factor1", "log_scale_factor2", "th", "match12")),
}


@pytest.mark.parametrize("struct", sorted(STRUCTS))
def test_pose_search_job_ctypes_layout_matches_the_header(tmp_path, struct):
    from orb_slam2_b200 import matcher
    cls_name, fields = STRUCTS[struct]
    cls = getattr(matcher, cls_name)
    body = "\n".join([f'    printf("size %zu\\n", sizeof({struct}));'] +
                     [f'    printf("{f} %zu\\n", offsetof({struct}, {f}));' for f in fields])
    src = tmp_path / "layout.c"
    src.write_text(textwrap.dedent('''
        #include <stddef.h>
        #include <stdio.h>
        #include "borb.h"
        int main(void) {
        BODY
            return 0;
        }
    ''').replace("BODY", body))
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == C.sizeof(cls)
    assert [name for name, _ in cls._fields_] == list(fields)
    for f in fields:
        assert int(out[f]) == getattr(cls, f).offset, f
