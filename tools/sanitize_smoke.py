"""Small end-to-end exercise of every kernel for compute-sanitizer (memcheck / racecheck) — dev tooling."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from oracle import oracle_lib as O
from orb_slam2_b200 import synth
from orb_slam2_b200.extractor import ORBextractor
from orb_slam2_b200 import matcher as M
from tests import match_fixtures as mf

L, R, _ = synth.stereo_pair(3, 0, 0, 640, 480)
G = ORBextractor(1000)
out = G.stereo_frames([L, L], [R, R], 40.0, 525.0)
print("stereo", len(out[0]["mvKeys"]), int((out[0]["mvuRight"] >= 0).sum()))
G2 = ORBextractor(500)
k, d = G2(synth.white_noise(1, 400, 300))
print("noise", len(k))
# one Frame constructor of each kind on the frame's own handles (borb_frame_from_extractors)
XL, XR = ORBextractor(1000), ORBextractor(1200)
XL.extract_enqueue(L); XR.extract_enqueue(R)
Fs, hs = M.frame_from_extractors(M.ORBmatcher(0.8, True), XL, XR, (525.0, 525.0, 319.5, 239.5), bf=40.0, mode=1)
XL.extract_enqueue(L)
Fd, hd = M.frame_from_extractors(M.ORBmatcher(0.8, True), XL, None, (525.0, 525.0, 319.5, 239.5), (0.26, -0.95, 0.0, 0.0, 1.16), bf=40.0,
                                 mode=2, depth=np.full(L.shape, 6000, np.uint16), depth_factor=1.0 / 5000.0)
XL.extract_enqueue(R)
Fm, hm = M.frame_from_extractors(M.ORBmatcher(0.8, True), XL, None, (525.0, 525.0, 319.5, 239.5))
print("frame ctors", len(hs["mvKeys"]), int((hs["mvuRight"] >= 0).sum()), int((hd["mvDepth"] > 0).sum()), len(hm["cell_idx"]))
# geometry edges (tests/extract_geometry.py): the smallest accepted frame, a frame whose level-0 pitch is exactly its width + 8
# (no slack after the padding), and a level 0 one candidate over the quadtree's on-chip limit
from tests import extract_geometry as EG
print("smallest", len(ORBextractor(1000)(synth.mono_frame(2, 0, 0, 221, 221))[0]))
print("tight pitch", len(ORBextractor(1000)(synth.white_noise(3, 376, 240))[0]))
# FAST bands (tests/test_gpu_fast_bands.py): KITTI-shaped, R = 2/2/1/2/1/1/2/1 with a last band of one cell row on level 0
# (11 rows, R = 2); 221x221, whose top levels have a one-row cell grid (R = 1)
from tests import test_gpu_fast_bands as FB
for (bw, bh), nf in (((1242, 375), 2000), ((221, 221), 1000)):
    lv = EG.geometry(bw, bh, nfeatures=nf)[0]
    print("bands", (bw, bh), [FB.rows_per_blk(v) for v in lv], [FB.bands(v)[-1][1] for v in lv],
          len(ORBextractor(nf)(synth.mono_frame(6, 0, 0, bw, bh))[0]))
G3 = ORBextractor(EG.DOT_NFEATURES)
k = G3(EG.dot_image(5121, *synth.KITTI, 1))[0]
print("5121 candidates", len(G3.debug_candidates(0)), len(k))
v = mf.two_views(O, 7)
F, mps = mf.projection_case(v, 1)
mt = M.ORBmatcher(0.8, True)
print("proj", mt.SearchByProjection(F, mps, 3.0)[0])
Cur, Last, Tcw, K = mf.last_frame_case(v, 2)
print("last", mt.SearchByProjectionLast(Cur, Last, Tcw, K, 40.0, 7.0)[0])
Fw, Pw, Tw, Ow, Kw = mf.world_points_case(v, 4)
print("kf/sim3", mt.SearchByProjectionKF(Fw, Pw, Tw, Ow, Kw, 10.0, 100)[0], mt.SearchByProjectionSim3(Fw, Pw, Tw, Ow, Kw, 10)[0])
KFf, Pf, Tf, Owf, Kf, bff = mf.fuse_case(v, 5)
print("fuse", mt.Fuse(KFf, Pf, Tf, Owf, Kf, bff, 3.0)[0], mt.Fuse(KFf, Pf, Tf, Owf, Kf, bff, 3.0, Scw=True)[0])
print("sim3", mt.SearchBySim3(*mf.sim3_case(v, 6), 7.5)[0])
bb = (0.0, 0.0, float(v["w"]), float(v["h"]))
print("init", mt.SearchForInitialization(M.FrameView(v["kl"], v["dl"], v["scale"], bb), M.FrameView(v["kr"], v["dr"], v["scale"], bb),
                                         np.stack([v["kl"]["x"], v["kl"]["y"]], 1), 100)[0])
pv = O.PortVocabulary.random(10, 3, 5)
e = pv.export()
voc = M.ORBVocabulary.from_arrays(e["parent"], e["is_leaf"], e["desc"], e["weight"], e["k"], e["L"])
kf1, kf2 = mf.keyframe_views(v, pv, 3, levelsup=1)
print("bow", mt.SearchByBoW(kf1, kf2)[0], mt.SearchByBoW_KF(kf1, kf2)[0], len(mt.SearchForTriangulation(kf1, kf2, mf.rectified_F12(1), (-1000.0, 200.0))))
print("voc", voc.transform_raw(v["dl"], 1)[0][:4])
db = M.KeyFrameDatabase(mt)
bow1, _ = voc.transform(v["dl"], 1)
bow2, _ = voc.transform(v["dr"], 1)
db.add(kf1, bow1); db.add(kf2, bow2)
print("kfdb", db.query(bow1)[0], db.SearchByBoW([0, 1], kf2)[0])
print("distinctive", mt.ComputeDistinctiveDescriptors([v["dl"][:9], v["dl"][:1], v["dl"][:0], v["dl"][:70]]))
# matcher envelope (tests/match_envelope.py): 8192 x 8192 SearchByProjection, and a SearchByBoW whose one node is wider than
# the distance-matrix path
from tests import match_envelope as ME
c8 = ME.case(O, "self_kitti_8192")
print("proj 8192", mt.SearchByProjection(c8["F"], c8["mps"], c8["th"])[0])
cb = ME.case(O, "bow_one_node_8192")
print("bow wide node", mt.SearchByBoW(cb["kf1"], cb["kf2"])[0], mt.SearchByBoW_KF(cb["kf1"], cb["kf2"])[0])

# ---- round 2 kernels: device-side Frame tail (RGB-D), resident frames + in-place (pinned) inputs/outputs of the small calls,
# CTA-wide claim resolution, database SearchByBoW (node-major items, compact pairs), ComputeBoW, persistent scoring kernel
import dataclasses
X = ORBextractor(1000)
imgs = [synth.mono_frame(40 + i, 0, 0, 640, 480) for i in range(2)]
outs = X.extract_batch(imgs)
rng = np.random.default_rng(0)
raw = (5000.0 * (1.5 + 0.5 * rng.random((480, 640)))).astype(np.uint16)
TUM1_K = (517.306408, 516.469215, 318.643040, 255.313989)
TUM1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)
frames, host = M.frames_from_extractor(mt, X, [1, 0], [len(outs[1][0]), len(outs[0][0])], TUM1_K, TUM1_DIST, bf=40.0, mode=2,
                                       depth=[raw, raw], depth_factor=np.float32(1.0 / 5000.0))
keys_un, desc = host["keys_un"][0], outs[1][1]
vv = dict(w=640, h=480, kl=keys_un, dl=desc, kr=keys_un, dr=desc, ur=host["u_right"][0], disp=np.zeros((480, 640), np.float32),
          scale=X.GetScaleFactors(), sigma2=X.GetScaleSigmaSquares())
Fh, mps2 = mf.projection_case(vv, 9, n_mp=300)
FR = dataclasses.replace(frames[0], occupied=Fh.occupied)
print("resident proj", mt.SearchByProjection(FR, mps2, 3.0)[0])
Cur2, Last2, Tcw2, K2 = mf.last_frame_case(vv, 3)
CurR = dataclasses.replace(frames[0], occupied=Cur2.occupied)
print("resident last", mt.SearchByProjectionLast(CurR, Last2, Tcw2, K2, 40.0, 7.0)[0])
voc6 = M.ORBVocabulary.from_arrays(*__import__("orb_slam2_b200.sharding", fromlist=["x"]).random_vocabulary_arrays(10, 4, 7), 10, 4)
db2 = M.KeyFrameDatabase(mt)
for j in range(12):
    k_, d_ = outs[j % 2]
    flip = (rng.random((len(d_), 32, 8)) < 0.03)
    d_ = d_ ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d_), 32)
    bow_, fv_ = voc6.ComputeBoW(d_, 2)
    hm = (rng.random(len(k_)) < 0.6).astype(np.uint8)
    db2.add(M.KeyFrameView(mvKeysUn=k_, mDescriptors=d_, mFeatVec=fv_, has_mp=hm), bow_)
qb, qf = voc6.ComputeBoW(outs[0][1], 2)
Fq = M.KeyFrameView(mvKeysUn=outs[0][0], mDescriptors=outs[0][1], mFeatVec=qf)
nm, off, pairs = db2.SearchByBoWPairs(None, Fq)
print("bowdb pairs", int(nm.sum()), "query", db2.query(qb)[0][:4], "dense", db2.SearchByBoW(np.arange(12, dtype=np.int32), Fq)[0][:4])

# relocalisation batch: two databases, one call mixing a frame block in shared memory and one in global memory (6000 features)
from orb_slam2_b200._lib import KP_DTYPE
kb = np.zeros(6000, KP_DTYPE)
kb["x"] = rng.uniform(20, 600, 6000); kb["y"] = rng.uniform(20, 440, 6000); kb["angle"] = rng.uniform(0, 360, 6000); kb["size"] = 31.0; kb["class_id"] = -1
db3 = M.KeyFrameDatabase(mt)
for j in range(3):
    bow_, fv_ = voc6.ComputeBoW(outs[1][1], 2)
    db3.add(M.KeyFrameView(mvKeysUn=outs[1][0], mDescriptors=outs[1][1], mFeatVec=fv_, has_mp=np.ones(len(outs[1][0]), np.uint8)), bow_)
FR0 = M.FrameView(outs[0][0], outs[0][1], X.GetScaleFactors(), (0.0, 0.0, 640.0, 480.0)).make_resident(mt)
FB = M.FrameView(kb, rng.integers(0, 256, (6000, 32), dtype=np.uint8), X.GetScaleFactors(), (0.0, 0.0, 640.0, 480.0)).make_resident(mt)
mt.ComputeBoWBatch(voc6, [FR0, FB], 2, want_host=False)
print("kfdb query batch", [q[0][:3] for q in mt.KfdbQueryBatch([db2, db3], [FR0, FB])])
print("bow score batch", [s[:3] for s in mt.BowScoreBatch([(FR0, [(db2, 0), FB, (db3, 2)]), ((db3, 1), [FR0, (db2, 5)])])])
print("bowdb batch", [int(r[0].sum()) for r in mt.SearchByBoWDbBatch([db2, db3, db2], [None, None, [0, 5, 5]], [FR0, FB, FB])])
K_S, I34, Z3 = (525.0, 525.0, 319.5, 239.5), np.eye(4, dtype=np.float32)[:3], np.zeros(3, np.float32)
def _slots(F, z=5.0):                                                   # one MapPoint per feature, back-projected at depth z
    k = F.mvKeysUn
    Pw = np.stack([(k["x"] - K_S[2]) * z / K_S[0], (k["y"] - K_S[3]) * z / K_S[1], np.full(len(k), z)], 1).astype(np.float32)
    d = np.linalg.norm(Pw, axis=1).astype(np.float32)
    return M.WorldPointsView(Pw, F.mDescriptors, (d * np.float32(1.2) ** k["octave"]).astype(np.float32), np.full(len(k), 0.1, np.float32),
                             (Pw / d[:, None]).astype(np.float32), k["angle"].astype(np.float32))
Pr0, PrB = _slots(FR0), _slots(FB)
print("pose search batches", mt.SearchBySim3Batch([FR0, FR0], [FR0, FB], [Pr0, Pr0], [Pr0, PrB], [(I34, I34)] * 2, [(I34, I34)] * 2, K_S, 7.5)[0][0], mt.SearchByProjectionKFBatch([FR0, FB], [Pr0, Pr0], [(I34, Z3)] * 2, K_S, 10.0, 100)[0][0], mt.SearchByProjectionSim3Batch([FR0, FB], [PrB, Pr0], [(I34, Z3)] * 2, K_S, 10)[0][0])
print("init batch", [r[0] for r in mt.SearchForInitializationBatch([FR0, FR0, FB], [FR0, FB, FR0], [np.stack([outs[0][0]["x"], outs[0][0]["y"]], 1)] * 2 + [np.stack([kb["x"], kb["y"]], 1)], [100, 100, 30])])

# place-recognition envelope (tests/bow_envelope.py): the flat 70,000-word vocabulary, the 8192 x 8192 one-node database search,
# and a job table of 2 * n_SM + 1 small shared-memory jobs (some CTA loads three or more frame blocks)
from tests import bow_envelope as BE
af = BE.vocabulary("flat70000")
vf = M.ORBVocabulary.from_arrays(af["parent"], af["is_leaf"], af["desc"], af["weight"], af["k"], af["L"])
print("flat voc", vf.transform_raw(BE.descriptors("flat70000")["high_ranks"], 0)[0][:4])
c1 = BE.search_case("one_node_8192")
db4 = M.KeyFrameDatabase(mt)
for kf_ in c1["kfs"]:
    db4.add(kf_, {0: 1.0})
print("bowdb one node 8192", db4.SearchByBoWPairs(None, c1["F"])[0])
import torch
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
print("bowdb table", sum(int(r[0].sum()) for r in mt.SearchByBoWDbBatch(db2, [[j % 12] for j in range(2 * n_sm + 1)], [FR0] * (2 * n_sm + 1))))
