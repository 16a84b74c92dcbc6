"""GPU: describe_kernel fetches a keypoint's rBRIEF taps in the order of its orientation bin (borb_debug_brief_slots).  At the
three benchmark geometries the angles and descriptors must equal the port's, with keypoints in every bin, so that every bin's
tap order has produced descriptors that were checked."""
import ctypes as C

import numpy as np
import pytest

from orb_slam2_b200 import synth
from tests.test_gpu_extract import assert_kps_equal

pytestmark = pytest.mark.gpu
GEOMETRIES = [(synth.KITTI, 2000), (synth.TUM, 1000), (synth.EUROC, 1200)]


def n_bins():
    from orb_slam2_b200 import _lib
    nb = C.c_int32(0)
    _lib.check(_lib.load().borb_debug_brief_slots(None, 0, C.byref(nb)), "borb_debug_brief_slots")
    return nb.value


def bins_of(angle, nb):
    """describe_kernel's bin: min((int)(angle * (float)(nb / 360.0)), nb - 1), float32 product."""
    return np.minimum((angle.astype(np.float32) * np.float32(nb / 360.0)).astype(np.int32), nb - 1)


@pytest.mark.parametrize("shape,nf", GEOMETRIES, ids=lambda v: f"{v[0]}x{v[1]}" if isinstance(v, tuple) else str(v))
def test_descriptors_match_port_in_every_bin(oracle, shape, nf):
    from orb_slam2_b200.extractor import ORBextractor
    w, h = shape
    nb = n_bins()
    frames = [synth.mono_frame(61, 0, i, w, h) for i in range(2)] + [synth.white_noise(62, w, h)]
    G, P = ORBextractor(nf), oracle.PortExtractor(nf)
    counts = np.zeros(nb, np.int64)
    for i, ((kg, dg), img) in enumerate(zip(G.extract_batch(frames), frames)):
        kp, dp = P(img)
        assert_kps_equal(kg, dg, kp, dp)
        counts += np.bincount(bins_of(kg["angle"], nb), minlength=nb)
    print(f"{w}x{h} @{nf}: keypoints per orientation bin {counts.tolist()}")
    assert (counts > 0).all(), f"bins without keypoints: {np.nonzero(counts == 0)[0].tolist()}; counts {counts.tolist()}"
