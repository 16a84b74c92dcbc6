"""Generates tests/golden/*.npz from the REFERENCE ITSELF (oracle/_ref: /root/reference/src/ORBextractor.cc
compiled verbatim + cv shim pinned to cv2 4.13 + monotonic allocator) — run in the build container where
/root/reference exists:   python tests/golden/make_golden.py
The stereo vectors were written with the line-by-line restatement of Frame.cc:466-640 fed with the reference extractor's outputs;
tests/test_golden_oracle.py::test_stereo_golden_equals_verbatim_frame_cc shows that the reference's own Frame.cc, compiled verbatim
(oracle/_ref/libframeref.so), produces exactly the same numbers."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle_lib as O          # noqa: E402
from orb_slam2_b200 import synth            # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = {  # name: (w, h, nfeatures, iniTh, minTh, seed)   — BASELINE.json configs' shapes
    "kitti_2000": (1242, 375, 2000, 20, 7, 100),
    "kitti0412_2000": (1241, 376, 2000, 12, 7, 101),   # Examples/Stereo/KITTI04-12.yaml
    "tum_1000": (640, 480, 1000, 20, 7, 102),
    "euroc_1200": (752, 480, 1200, 20, 7, 103),
    "tum_mono_init_2000": (640, 480, 2000, 20, 7, 104),  # Tracking.cc:125 mpIniORBextractor = 2*nFeatures
    "kitti_seed21_2000": (1242, 375, 2000, 20, 7, 21),   # test_gpu_extract.py::test_matches_verbatim_reference_build
}


def main():
    O.build()
    assert O.have_ref(), "needs /root/reference"
    for name, (w, h, nf, ini, mn, seed) in CASES.items():
        img = synth.mono_frame(seed, 0, 0, w, h)
        R = O.RefExtractor(nf, 1.2, 8, ini, mn)
        k, d = R(img)
        np.savez_compressed(os.path.join(HERE, f"extract_{name}.npz"), keypoints=k, descriptors=d,
                            meta=np.array([w, h, nf, ini, mn, seed], np.int32))
        print(name, len(k))
    # stereo (config 2): KITTI-shaped pair
    L, Rimg, _ = synth.stereo_pair(200, 0, 0)
    bf, fx = 386.1448, 718.856
    EL, ER = O.RefExtractor(2000), O.RefExtractor(2000)
    kl, dl = EL(L)
    kr, dr = ER(Rimg)
    ur, dp, sad = O.port_stereo(kl, dl, kr, dr, [EL.level(i) for i in range(8)], [ER.level(i) for i in range(8)],
                                EL.scale, EL.inv_scale, bf, fx)
    np.savez_compressed(os.path.join(HERE, "stereo_kitti_2000.npz"), kl=kl, dl=dl, kr=kr, dr=dr, u_right=ur, depth=dp,
                        meta=np.array([1242, 375, 2000, 200], np.int32), cam=np.array([bf, fx], np.float64))
    print("stereo", int((ur >= 0).sum()), "matches")


if __name__ == "__main__":
    main()
