"""The REAL vocabulary (reference Vocabulary/ORBvoc.txt.tar.gz: k=10, L=6, 1,082,073 nodes, 971,814 words) through the product:
tests/golden/voc_real.npz holds BowVector / FeatureVector of three golden descriptor sets as the reference's own DBoW2 (compiled
verbatim) computes them; oracle/_ref/orbvoc_arrays.npz (git-ignored, written by build() with the reference's own DBoW2 loader,
oracle_lib.build_voc_arrays, and kept with the other oracle/_ref builds) holds the parsed tree.  Checked here: borb_voc_create + borb_compute_bow on the real tree, the text loader on a text file rebuilt
in ORBvoc.txt's format (with its trailing newline), the packed blob round trip; load / upload times are printed."""
import os
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARR = os.path.join(ROOT, "oracle", "_ref", "orbvoc_arrays.npz")
SETS = ["extract_kitti_2000", "extract_euroc_1200", "extract_tum_1000"]


@pytest.fixture(scope="module")
def real():
    if not os.path.exists(ARR):
        pytest.skip("oracle/_ref/orbvoc_arrays.npz absent (build() writes it where the reference tree is present)")
    a = np.load(ARR)
    return dict(parent=a["parent"], is_leaf=a["is_leaf"], desc=a["desc"], weight=a["weight"], k=int(a["k"][0]), L=int(a["L"][0]))


def _check(voc, g):
    for name in SETS:
        d = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["descriptors"]
        bow, fv = voc.ComputeBoW(d, 4)
        assert np.array_equal(np.fromiter(bow.keys(), np.uint32, len(bow)), g[name + "_bow_word"]), name
        assert np.array_equal(np.fromiter(bow.values(), np.float64, len(bow)), g[name + "_bow_value"]), name      # bit-identical doubles
        assert np.array_equal(fv.node_id, g[name + "_fv_node"]) and np.array_equal(fv.start, g[name + "_fv_start"]) and np.array_equal(fv.feat_idx, g[name + "_fv_idx"]), name


def test_real_vocabulary_transform_matches_verbatim_dbow2(real, tmp_path):
    from orb_slam2_b200 import matcher as M
    g = np.load(os.path.join(ROOT, "tests", "golden", "voc_real.npz"))
    assert len(real["parent"]) == int(g["n_nodes"][0]) == 1082073 and int(real["is_leaf"].sum()) == int(g["n_words"][0])
    t0 = time.perf_counter()
    voc = M.ORBVocabulary.from_arrays(real["parent"], real["is_leaf"], real["desc"], real["weight"], real["k"], real["L"])
    t_create = time.perf_counter() - t0
    _check(voc, g)
    ptr, nbytes = voc.blob()
    v2 = M.ORBVocabulary.from_blob(ptr, nbytes)                          # what a rank adopts after the NCCL broadcast
    _check(v2, g)
    # ORBvoc.txt rebuilt from the arrays (same format, trailing newline included) -> borb_voc_load_text
    path = str(tmp_path / "ORBvoc.txt")
    t0 = time.perf_counter()
    n = len(real["parent"])
    body = np.concatenate([real["parent"][1:, None].astype(np.int64), real["is_leaf"][1:, None].astype(np.int64), real["desc"][1:].astype(np.int64)], 1)
    lines = [" ".join(map(str, row)) for row in body.tolist()]
    w = real["weight"][1:]
    with open(path, "w") as f:
        f.write(f"{real['k']} {real['L']} 0 0\n")
        f.write("\n".join(f"{ln} {repr(float(x))}" for ln, x in zip(lines, w)))
        f.write("\n")
    t_write = time.perf_counter() - t0
    t0 = time.perf_counter()
    v3 = M.ORBVocabulary.loadFromTextFile(path)
    t_load = time.perf_counter() - t0
    _check(v3, g)
    print(f"\nreal ORBvoc: {n} nodes, packed blob {nbytes / 1e6:.1f} MB; borb_voc_create {t_create * 1e3:.0f} ms, text rebuilt in {t_write:.1f} s "
          f"({os.path.getsize(path) / 1e6:.0f} MB), borb_voc_load_text {t_load:.2f} s")
