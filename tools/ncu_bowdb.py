"""Profiling driver for bowdb_match_kernel / bowdb_finalize_kernel: builds the configs[4] database (tools/bench_configs.py:config4)
and runs a few SearchByBoW sweeps.  Use under ncu:
    ncu --set full --import-source on -k regex:bowdb -c 4 -o gpurun_out/bowdb python tools/ncu_bowdb.py"""
import sys, os, json, time
import ctypes as C
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam2_b200 import matcher as M, sharding, synth, _lib
from orb_slam2_b200.extractor import ORBextractor

n_kf = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
voc = M.ORBVocabulary.from_arrays(*sharding.random_vocabulary_arrays(10, 6, 7), 10, 6)
X = ORBextractor(1200)
rng = np.random.default_rng(1)
n_src = 40
outs = X.extract_batch([synth.mono_frame(50 + i, 0, 0, 752, 480) for i in range(n_src)])
mt = M.ORBmatcher(0.75, True)
db = M.KeyFrameDatabase(mt)
for j in range(n_kf):
    k, d = outs[j % n_src]
    if j >= n_src:
        flip = (rng.random((len(d), 32, 8)) < 0.04)
        d = d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)
    bow, fv = voc.transform(d, 4)
    db.add(M.KeyFrameView(mvKeysUn=k, mDescriptors=d, mFeatVec=fv, has_mp=np.ones(len(k), np.uint8)), bow)
qk, qd = outs[3]
flip = (rng.random((len(qd), 32, 8)) < 0.02)
qd = qd ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(qd), 32)
qbow, qfv = voc.transform(qd, 4)
F = M.KeyFrameView(mvKeysUn=qk, mDescriptors=qd, mFeatVec=qfv)
db.query(qbow)
nm, off, pairs = db.SearchByBoWPairs(None, F)
cap = int(nm.sum()) + 1024
so = _lib.load()
so.borb_matcher_set_timing(mt._h, 1)
ts = []
for _ in range(reps):
    db.SearchByBoWPairs(None, F, pairs_cap=cap)
    f = C.c_float(0); so.borb_matcher_last_kernel_ms(mt._h, C.byref(f)); ts.append(round(f.value, 5))
so.borb_matcher_set_timing(mt._h, 0)
print(json.dumps({"pairs": int(nm.sum()), "kernel_ms": ts}))
