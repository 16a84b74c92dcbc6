"""Stage-by-stage GPU-vs-oracle diagnostic (run on a machine with the GPU). Prints mismatch counts; never asserts.
Test tooling: uses the oracle as the checker."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from oracle import oracle_lib as O
from orb_slam2_b200 import synth
from orb_slam2_b200.extractor import ORBextractor

def sort_rows(a):
    if len(a) == 0: return a
    return a[np.lexsort((a[:, 0], a[:, 1]))]

def diag_image(name, img, nf):
    print(f"== {name} {img.shape} nf={nf}")
    G = ORBextractor(nf)
    P = O.PortExtractor(nf)
    t = time.time(); kg, dg = G(img); tg = time.time() - t
    kp, dp = P(img)
    print(f"  gpu n={len(kg)} port n={len(kp)}  (gpu call {tg*1e3:.1f} ms)")
    for l in range(8):
        pg, pp = G.pyramid(l), P.level(l)
        bad_p = -1 if pg.shape != pp.shape else int((pg != pp).sum())
        cg, cp = sort_rows(G.debug_candidates(l)), sort_rows(P.candidates(l))
        same_c = cg.shape == cp.shape and np.array_equal(cg, cp)
        sg = G.debug_selected(l)
        # port selected: kp rows of this level in order
        m = kp["octave"] == l
        bg, bp = G.debug_blurred(l), P.blurred(l)
        bad_b = -1 if (bp is None or bg.shape != bp.shape) else int((bg != bp).sum())
        print(f"  L{l}: pyr diff {bad_p:6d} | cand gpu {len(cg):5d} port {len(cp):5d} same={same_c} | sel gpu {len(sg):4d} port {int(m.sum()):4d} | blur diff {bad_b}")
        if not same_c and len(cg) and len(cp):
            sgp = set(map(tuple, cg.tolist())); spp = set(map(tuple, cp.tolist()))
            print("      only gpu:", sorted(sgp - spp)[:5], " only port:", sorted(spp - sgp)[:5])
    n = min(len(kg), len(kp))
    if len(kg) == len(kp):
        for f in kg.dtype.names:
            bad = int((kg[f] != kp[f]).sum())
            if bad: print(f"  field {f}: {bad} mismatches; first at {np.nonzero(kg[f] != kp[f])[0][:5]}", kg[f][kg[f] != kp[f]][:3], kp[f][kg[f] != kp[f]][:3])
        bd = (dg != dp).any(axis=1)
        print(f"  keypoints equal: {np.array_equal(kg, kp)}  descriptor rows differing: {int(bd.sum())}")
        if bd.any():
            i = np.nonzero(bd)[0][0]
            print("   first bad desc idx", i, "bits differing", int(np.unpackbits(dg[i] ^ dp[i]).sum()), kg[i])
    else:
        print("  COUNT MISMATCH")
    return G

def diag_stereo(seed):
    L, R, _ = synth.stereo_pair(seed, 0, 0)
    bf, fx = 386.1448, 718.856
    G = ORBextractor(2000)
    out = G.stereo_frames([L], [R], bf, fx)[0]
    E1, E2 = O.PortExtractor(2000), O.PortExtractor(2000)
    kl, dl = E1(L); kr, dr = E2(R)
    ur, dp, sad = O.port_stereo(kl, dl, kr, dr, [E1.level(i) for i in range(8)], [E2.level(i) for i in range(8)], E1.scale, E1.inv_scale, bf, fx)
    print(f"== stereo seed {seed}: kps L equal {np.array_equal(out['mvKeys'], kl)} R equal {np.array_equal(out['mvKeysRight'], kr)}")
    if len(ur) == len(out['mvuRight']):
        print(f"   matched gpu {(out['mvuRight']>=0).sum()} port {(ur>=0).sum()}  uRight equal {np.array_equal(out['mvuRight'], ur)} depth equal {np.array_equal(out['mvDepth'], dp)}")
        bad = np.nonzero(out['mvuRight'] != ur)[0]
        if len(bad): print("   first diffs", bad[:5], out['mvuRight'][bad[:5]], ur[bad[:5]])

if __name__ == "__main__":
    O.build()
    diag_image("kitti-synth", synth.mono_frame(1, 0, 0, *synth.KITTI), 2000)
    diag_image("tum-synth", synth.mono_frame(2, 0, 0, *synth.TUM), 1000)
    diag_image("noise", synth.white_noise(3, 640, 360), 1000)
    diag_stereo(1)
    G = ORBextractor(2000)
    G.set_timing(True)
    imgs = [synth.mono_frame(5, 0, i, *synth.KITTI) for i in range(16)]
    for rep in range(3):
        t = time.time(); r = G.extract_batch(imgs); dt = time.time() - t
        print(f"batch16 extract: {dt*1e3:.2f} ms  stages {G.stage_times()}")
