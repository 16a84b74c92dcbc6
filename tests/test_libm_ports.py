"""CPU: the C twins of the device-side libm ports (glibc sinf/cosf in k_describe.cu, glibc logf in k_match.cu) agree with the
host libm — sinf/cosf for EVERY float in [0, 2*pi] (about 6 s), logf on every 61st positive normal float (the exhaustive run,
`check_logf` without an argument, takes ~25 s and was 0 mismatches; DESIGN.md section 2).  The twins' constant tables must
equal the device tables value for value, and orbport_libm (the host reference of tests/test_gpu_device_math.py, which sweeps
the device functions themselves) must be the host libm."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "libm_ports")
CSRC = os.path.join(ROOT, "orb_slam2_b200", "csrc")


def _build(tmp_path, name, extra=()):
    exe = tmp_path / name
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", *extra, "-o", str(exe), os.path.join(SRC, name + ".c"), "-lm"])
    return str(exe)


def test_sincosf_port_exhaustive(tmp_path):
    out = subprocess.run([_build(tmp_path, "check_sincosf")], capture_output=True, text=True, timeout=300).stdout
    assert "cos mismatches=0 sin mismatches=0" in out, out


def test_logf_port_sampled(tmp_path):
    out = subprocess.run([_build(tmp_path, "check_logf"), "61"], capture_output=True, text=True, timeout=300).stdout
    assert "mismatches: nofma 0, fma 0" in out, out


# ---- the C twins carry their own copies of the constant tables: tie them to the tables nvcc compiles into libborb.so
NUM = re.compile(r"[-+]?(?:0x[0-9a-fA-F]*\.?[0-9a-fA-F]*p[-+]?\d+|\d+\.\d*)")


def _initializer(path, start):
    """The numeric literals of the brace initializer that follows `start` in `path`, in source order."""
    txt = open(path).read()
    i = txt.index(start)
    body = txt[txt.index("{", i):txt.index("};", i)]
    return [float.fromhex(t) if "x" in t else float(t) for t in NUM.findall(body)]


def _literal(path, name):
    """The numeric literal that follows `name` in `path`."""
    txt = open(path).read()
    return float.fromhex(NUM.search(txt, txt.index(name)).group(0))


def test_sincosf_tables_match_the_device_port():
    dev = _initializer(os.path.join(CSRC, "k_describe.cu"), "d_sincos[2] =")
    twin = _initializer(os.path.join(SRC, "check_sincosf.c"), "T[2] =")
    assert len(dev) == 2 * 14, dev                      # sign[4], hpi_inv, hpi, c0..c4, s1..s3, for each of the two tables
    assert dev == twin, [(i, a.hex(), b.hex()) for i, (a, b) in enumerate(zip(dev, twin)) if a != b]


def test_logf_tables_match_the_device_port():
    dev = _initializer(os.path.join(CSRC, "k_match.cu"), "d_logf =")
    assert len(dev) == 16 + 16 + 4, dev                 # invc[16], logc[16], ln2, a0, a1, a2
    pairs = _initializer(os.path.join(SRC, "check_logf.c"), "T[16] =")
    twin = pairs[0::2] + pairs[1::2] + [_literal(os.path.join(SRC, "check_logf.c"), "Ln2 =")] \
        + _initializer(os.path.join(SRC, "check_logf.c"), "A[3] =")
    assert dev == twin, [(i, a.hex(), b.hex()) for i, (a, b) in enumerate(zip(dev, twin)) if a != b]


def test_orbport_libm_is_the_host_libm(oracle):
    """orbport_libm, the host reference of the device sweeps (tests/test_gpu_device_math.py), calls libm itself."""
    libm = C.CDLL("libm.so.6")
    rng = np.random.default_rng(5)
    x = np.concatenate([rng.uniform(0, 7, 3000), rng.uniform(0, 120, 1000), np.exp(rng.uniform(-80, 80, 3000))]).astype(np.float32)
    x[:4] = [0.0, 1.0, np.float32(np.pi / 4), np.float32(2 * np.pi)]
    for fn, name in ((oracle.LIBM_SINF, "sinf"), (oracle.LIBM_COSF, "cosf"), (oracle.LIBM_LOGF, "logf")):
        f = getattr(libm, name)
        f.restype, f.argtypes = C.c_float, [C.c_float]
        want = np.array([f(float(v)) for v in x], np.float32)
        got = oracle.port_libm(fn, x)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), name
