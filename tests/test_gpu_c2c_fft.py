"""FourierC2c lanes on the lane FFT (OP_CFFT): an n-point complex FFT over the lane's 2n reals, forward unnormalised, backward
conj -> FFT -> conj with 1/n, modes in natural FFT order.  Power-of-two sizes run on the compile-time-geometry instances
(cfft_fast), 3 * 2^k and 5 * 2^k on the generic ones (op_cfft with the odd pass of lane_fft).

Every case forces its layout through the switches make_cfg reads at space creation (B2_E, B2_LN, B2_NOFAST) and proves it with
Space2.layout() before anything else.  Forward and backward are checked against numpy's FFT applied here (np.fft.fft / ifft along
axis 0, the oracle's 1-D Chebyshev transform along axis 1), so the check does not rest on the oracle's c2c code.
tests/test_emu_c2c_fft.py runs the lanes of n <= 128 on the emulator build."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH, CD, CN, C2C = 0, 1, 2, 5
SWITCHES = ("B2_E", "B2_LN", "B2_NOFAST")
TOL = 1e-10

# (id, environment, c2c n, expected (E, LN, TPL, fast)) of the lanes along axis 0: the natural layouts of every FFT size, then
# forced layouts, so that every compile-time instance a c2c lane can reach and every generic (E, LN) pair runs at least once
CASES = [
    ("n32", {}, 32, (4, 4, 8, 1)),
    ("n64", {}, 64, (8, 4, 8, 1)),
    ("n128", {}, 128, (8, 4, 16, 1)),
    ("n256", {}, 256, (8, 4, 32, 1)),
    ("n512", {}, 512, (8, 4, 64, 1)),
    ("n1024", {}, 1024, (16, 4, 64, 1)),
    ("r3-96", {}, 96, (4, 4, 24, 0)),
    ("r5-160", {}, 160, (4, 4, 40, 0)),
    ("r3-192", {}, 192, (8, 4, 24, 0)),
    ("r5-320", {}, 320, (8, 4, 40, 0)),
    ("r3-384", {}, 384, (8, 4, 48, 0)),
    ("r5-640", {}, 640, (8, 4, 80, 0)),
    ("r3-768", {}, 768, (8, 4, 96, 0)),
    ("e16-128", {"B2_E": "16"}, 128, (16, 4, 8, 1)),
    ("e16-256", {"B2_E": "16"}, 256, (16, 4, 16, 1)),
    ("e16-512", {"B2_E": "16"}, 512, (16, 4, 32, 1)),
    ("e4-64", {"B2_E": "4"}, 64, (4, 4, 16, 1)),
    ("e4-128", {"B2_E": "4"}, 128, (4, 4, 32, 1)),
    ("nofast-32", {"B2_NOFAST": "1"}, 32, (4, 4, 8, 0)),
    ("nofast-64", {"B2_NOFAST": "1"}, 64, (8, 4, 8, 0)),
    ("nofast-1024", {"B2_NOFAST": "1"}, 1024, (16, 4, 64, 0)),
    ("r3-e16-384", {"B2_E": "16"}, 384, (16, 4, 24, 0)),
    ("r5-e16-640", {"B2_E": "16"}, 640, (16, 4, 40, 0)),
    ("ln2-64", {"B2_LN": "2"}, 64, (4, 2, 16, 0)),
    ("ln2-128", {"B2_LN": "2"}, 128, (8, 2, 16, 0)),
    ("ln2-1024", {"B2_LN": "2"}, 1024, (16, 2, 64, 0)),
    ("r3-ln2-192", {"B2_LN": "2"}, 192, (4, 2, 48, 0)),
    ("r5-ln2-320", {"B2_LN": "2"}, 320, (4, 2, 80, 0)),
    ("r3-ln2-384", {"B2_LN": "2"}, 384, (8, 2, 48, 0)),
    ("r5-ln2-640", {"B2_LN": "2"}, 640, (8, 2, 80, 0)),
    ("r3-e16-ln2-768", {"B2_E": "16", "B2_LN": "2"}, 768, (16, 2, 48, 0)),
]
CASE = {c[0]: c[1:] for c in CASES}
CROSS = 65   # the Chebyshev axis 1


def layout(sp, orient=1):
    import rustpde_mpi_b200 as b2

    s = b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))
    lay = tuple(s.layout(orient)[k] for k in ("E", "LN", "TPL", "fast"))
    s.close()
    return lay


def smooth_phys(n, m, seed, band=None):
    """complex values on the c2c x Chebyshev grid whose modes along axis 0 are |k| <= band (n / 4 by default): random
    coefficients, smooth along axis 1 (a few low Chebyshev polynomials)"""
    rng = np.random.default_rng(seed)
    band = n // 4 if band is None else band
    c = np.zeros(n, dtype=np.complex128)
    k = np.r_[0:band + 1, n - band:n]
    c[k] = rng.standard_normal(k.size) + 1j * rng.standard_normal(k.size)
    y = -np.cos(np.pi * np.arange(m) / (m - 1))
    prof = np.stack([np.polynomial.chebyshev.chebval(y, rng.standard_normal(4)) for _ in range(3)])
    return np.fft.ifft(c)[:, None] * prof[0][None, :] + np.fft.ifft(np.roll(c, 1))[:, None] * prof[1][None, :] + 0.1 * prof[2][None, :]


def numpy_errors(kind1, n, m, seed=21):
    """forward and backward of a c2c n x (kind1, m) space against np.fft applied along axis 0, on random and on smooth
    band-limited values: {name: relative max-norm error}"""
    import rustpde_mpi_b200 as b2
    from oracle import rustpde_oracle as o

    from tests import gpu_checks as g

    cheb = o.Base(kind1, m)
    f = b2.Field2(b2.Space2((C2C, n), (kind1, m)))
    rng = np.random.default_rng(seed)
    errs = {}
    inputs = {"random": rng.uniform(-1, 1, (n, m)) + 1j * rng.uniform(-1, 1, (n, m)), "smooth": smooth_phys(n, m, seed)}
    for name, v in inputs.items():
        f.v = v
        f.forward()
        errs[f"forward-{name}"] = g.relerr(f.vhat, np.fft.fft(cheb.forward(v, axis=1), axis=0))
    shape = f.vhat.shape
    spec = {"random": rng.standard_normal(shape) + 1j * rng.standard_normal(shape),
            "smooth": np.fft.fft(cheb.forward(inputs["smooth"], axis=1), axis=0)}
    for name, a in spec.items():
        f.vhat = a
        f.backward()
        errs[f"backward-{name}"] = g.relerr(f.v, cheb.backward(np.fft.ifft(a, axis=0), axis=1))
    return errs


def case_errors(n, cross=CROSS):
    """numpy_errors on c2c x cd; round trip, to_ortho, from_ortho and the gradients (1,0), (2,0), (3,0), (2,1) with a scale on
    c2c x cd and c2c x cn; HholtzAdi, Hholtz and Poisson on both against the oracle: {name: error}"""
    from tests import gpu_checks as g

    errs = {k: v for k, v in numpy_errors(CD, n, cross).items()}
    for kind1 in (CD, CN):
        sp = (C2C, n, kind1, cross)
        tag = g.KIND_NAME[kind1]
        errs[f"{tag} roundtrip"] = g.check_roundtrip_layout(*sp)
        for op in ("forward", "backward", "to_ortho", "from_ortho", "hholtz", "hholtz_tensor", "poisson"):
            errs[f"{tag} {op}"] = getattr(g, "check_" + op)(*sp)
        for d in ((1, 0), (2, 0), (3, 0), (2, 1)):
            errs[f"{tag} gradient{d}"] = g.check_gradient(*sp, d, scale=(1.7, 0.6))
    return errs


# every case in a process of its own: the layout switches are read when a space is created
SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
if sys.argv[2] == "emu":
    from tests import emu
    emu.activate()
from tests import test_gpu_c2c_fft as t
case, cross, sequences = json.loads(sys.argv[1])
_, n, want = t.CASE[case]
for kind1 in (t.CD, t.CN):
    lay = t.layout((t.C2C, n, kind1, cross))
    assert lay == tuple(want), (case, kind1, lay, want)
errs = t.case_errors(n, cross)
bad = {k: e for k, e in errs.items() if not e < t.TOL}
if sequences:
    from tests import gpu_checks as g
    bad.update(g.sequence_failures(g.run_sequences((t.C2C, n, t.CD, cross))))
assert not bad, bad
print("worst", max(errs.values()))
print("ok")
''' % ROOT


def run_case(case, where, cross=CROSS, sequences=True):
    env = dict({k: v for k, v in os.environ.items() if k not in SWITCHES}, **CASE[case][0])
    r = subprocess.run([sys.executable, "-c", SCRIPT, json.dumps([case, cross, sequences]), where], capture_output=True,
                       text=True, timeout=3600, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASE))
def test_c2c_fft_case(case):
    """layout, forward / backward against np.fft (random and smooth), round trip, to_ortho / from_ortho, gradients, HholtzAdi,
    Hholtz and Poisson at 1e-10, and the call sequence (NaN-filled destinations, padding) on c2c x cd"""
    run_case(case, "gpu")


# The third derivative of a smooth field after a backward and a forward transform at n = 1024, where the transform's rounding in
# the small high modes is amplified by k^3.  Measured on an H100 (SXM, 700 W): 1.8e-12 with the FFT; the dense 2n x 2n matrices
# that ran this size before gave 1.0e-12 on the same field.  The bound keeps ~3x headroom over the FFT's figure.
D3_BOUND = 5e-12


def third_derivative_error(n=1024, m=CROSS):
    """backward (n-point FFT) -> forward -> d^3/dx^3 of a smooth band-limited field against the exact spectral derivative of its
    coefficients; relative max-norm error"""
    import rustpde_mpi_b200 as b2

    from tests import gpu_checks as g

    f = b2.Field2(b2.Space2((C2C, n), (CD, m)))
    rng = np.random.default_rng(3)
    a = np.zeros(f.vhat.shape, dtype=np.complex128)
    band = n // 8
    k = np.r_[0:band + 1, n - band:n]
    a[k, :8] = (rng.standard_normal((k.size, 8)) + 1j * rng.standard_normal((k.size, 8))) * np.exp(-(np.minimum(k, n - k) / (band / 4.0)) ** 2)[:, None]
    f.vhat = a
    f.backward()
    f.forward()
    got = f.gradient((3, 0)).get()
    kk = np.where(2 * np.arange(n) >= n, np.arange(n) - n, np.arange(n)).astype(np.float64)
    fo = b2.Field2(b2.Space2((C2C, n), (CD, m)))
    fo.vhat = a * ((1j * kk) ** 3)[:, None]
    ref = fo.to_ortho().get()
    return g.relerr(got, ref)


@pytest.mark.gpu
def test_c2c_third_derivative_accuracy():
    import rustpde_mpi_b200 as b2

    s = b2.Space2((C2C, 1024), (CD, CROSS))
    assert s.layout(1)["fast"] == 1
    s.close()
    e = third_derivative_error()
    print(f"[c2c] n = 1024 smooth field, d3/dx3 after backward + forward: relative error {e:.2e}")
    assert e <= D3_BOUND, e
