"""Real-vocabulary pin (VERDICT r01 item 8).  Run in the build container, where /root/reference exists:
    python tools/make_golden_voc.py
1. untars /root/reference/Vocabulary/ORBvoc.txt.tar.gz (1,082,073 nodes, 145 MB of text) into /tmp;
2. loads it with the reference's own DBoW2 (oracle/_ref/libdbowref.so: TemplatedVocabulary::loadFromTextFile compiled verbatim).
   loadFromTextFile loops `while(!f.eof())` (TemplatedVocabulary.h:1379-1420), so the file's trailing newline gives the reference a
   bogus extra node with uninitialised fields; the pin loads a copy without that newline, where the reference is well defined;
3. transforms the committed golden descriptor sets (tests/golden/extract_*.npz) with the VERBATIM DBoW2 (levelsup 4, what
   Frame::ComputeBoW asks for) and stores BowVector + FeatureVector in tests/golden/voc_real.npz (small, committed);
4. checks that the oracle port's loader + transform reproduce them.  The parsed tree itself (oracle/_ref/orbvoc_arrays.npz,
   what tests/test_gpu_voc_real.py pushes through the CUDA library) is written by build(): oracle_lib.build_voc_arrays."""
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_lib as O     # noqa: E402

TAR = "/root/reference/Vocabulary/ORBvoc.txt.tar.gz"
TMP = "/tmp/orbvoc"
SETS = ["extract_kitti_2000", "extract_euroc_1200", "extract_tum_1000"]


def main():
    O.build()
    os.makedirs(TMP, exist_ok=True)
    txt = os.path.join(TMP, "ORBvoc.txt")
    if not os.path.exists(txt):
        subprocess.check_call(["tar", "xzf", TAR, "-C", TMP])
    raw = open(txt, "rb").read()
    assert raw.endswith(b"\n")
    nonl = os.path.join(TMP, "ORBvoc_nonl.txt")
    open(nonl, "wb").write(raw.rstrip(b"\n"))
    t0 = time.perf_counter()
    ref = O.RefVocabulary(nonl)
    t_ref = time.perf_counter() - t0
    print(f"verbatim DBoW2 loadFromTextFile: {ref.words} words in {t_ref:.1f}s")
    t0 = time.perf_counter()
    port = O.PortVocabulary.load_text(txt)
    e = port.export()
    print(f"oracle port loader: {len(e['parent'])} nodes (k={e['k']}, L={e['L']}) in {time.perf_counter() - t0:.1f}s")
    assert int(e["is_leaf"].sum()) == ref.words
    out = {}
    for name in SETS:
        g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
        desc = g["desc"] if "desc" in g else g["descriptors"]
        bow, fn, fs, fi = ref.transform(desc, 4)
        bw, bv, (pn, ps, pi) = O.port_compute_bow(port, desc, 4)
        assert list(bow.keys()) == bw.tolist() and list(bow.values()) == bv.tolist(), name
        assert np.array_equal(fn, pn) and np.array_equal(fs, ps) and np.array_equal(fi, pi), name
        out[name + "_bow_word"] = np.array(list(bow.keys()), np.uint32)
        out[name + "_bow_value"] = np.array(list(bow.values()), np.float64)
        out[name + "_fv_node"] = fn; out[name + "_fv_start"] = fs; out[name + "_fv_idx"] = fi
        print(f"{name}: {len(desc)} descriptors -> {len(bow)} words, {len(fn)} nodes (port == verbatim DBoW2)")
    out["n_nodes"] = np.array([len(e["parent"])]); out["n_words"] = np.array([ref.words])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "voc_real.npz"), **out)
    print("wrote tests/golden/voc_real.npz")


if __name__ == "__main__":
    main()
