"""The banded operators' coefficients (csrc/band_coef.cuh) as the H100 forms them, bit for bit against the host's values.

The lane kernel forms the to_ortho / from_ortho stencils and the MatVecFdma coefficients in registers: the reciprocal starts from
the hardware's rcp.approx.ftz.f64 and takes two Newton steps, the ChebNeumann quotient k / (k + 2) one more correction.  The claim
is that this reproduces the host's s2 (Base1::init_host) and Base1::pv, i.e. the correctly rounded 1.0 / x and k / (k + 2.0),
bit for bit.  test_emu_band_coefficients.py checks the same arithmetic on the emulator, whose seed is its own 20-bit reciprocal;
here tests/band_coef_harness.cu, compiled with the library's nvcc for sm_90a, evaluates on the GPU:

- every family at every element i < n + 8 for n = 2^k + 1, 9 .. 8193;
- the BandPairs<BC_PV0, BC_PV2, BC_PV4> chunk walk (pv0 carried along a chunk) for chunks of 5, 9 and 17 pairs;
- bc_rcp of the three pv denominators and bc_div(i, i + 2) for every i < 2^20,

and numpy computes the host's values in IEEE double the way the host writes them.  CPU: the harness compiles (a build break
shows without a GPU)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rustpde_mpi_b200", "csrc")
HARNESS = os.path.join(ROOT, "tests", "band_coef_harness.cu")
NS = [2 ** k + 1 for k in range(3, 14)]   # 9 .. 8193
CPS = (5, 9, 17)
NQ = 1 << 20
FAMILIES = ("unit", "sten_d", "sten_n", "s2_d", "s2_n", "pv0", "pv2", "pv4")   # BC_UNIT .. BC_PV4


def compile_harness(out_dir):
    from rustpde_mpi_b200 import build

    exe = os.path.join(out_dir, "band_coef_harness")
    cmd = [build.NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC, "-o", exe, HARNESS]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return exe


# ---- the host's values (IEEE double, as b200pde.cu writes them) ----
def host_s2(kind_neumann, k):
    """Base1::init_host: s2[k] = -1 (ChebDirichlet) or -(k / (k + 2.0)) * (k / (k + 2.0)) (ChebNeumann)"""
    k = np.asarray(k, dtype=np.float64)
    if not kind_neumann:
        return np.full(k.shape, -1.0)
    q = k / (k + 2.0)
    return -q * q


def host_pv(i, off):
    """Base1::pv without its range: 0.25 at r = 2, else 1.0 / (4 r (r - 1)) (off 0), -1.0 / (2 (r^2 - 1)) (2), 1.0 / (4 r (r + 1)) (4)"""
    r = np.asarray(i, dtype=np.float64) + 2.0
    with np.errstate(divide="ignore"):
        if off == 0:
            return np.where(r == 2.0, 0.25, 1.0 / (4.0 * r * (r - 1.0)))
        if off == 2:
            return -1.0 / (2.0 * (r * r - 1.0))
        return 1.0 / (4.0 * r * (r + 1.0))


def host_families(n):
    """[family][i] for i < n + 8: the value band_coef(f, i, n) must reproduce"""
    i = np.arange(n + 8)
    m = n - 2
    zero = np.zeros(n + 8)
    sten = (i >= 2) & (i < n)
    return np.stack([
        np.ones(n + 8),
        np.where(sten, host_s2(False, np.maximum(i - 2, 0)), zero),
        np.where(sten, host_s2(True, np.maximum(i - 2, 0)), zero),
        np.where(i < m, host_s2(False, i), zero),
        np.where(i < m, host_s2(True, i), zero),
        np.where(i < m, host_pv(i, 0), zero),
        np.where(i < m - 2, host_pv(i, 2), zero),
        np.where(i < m - 4, host_pv(i, 4), zero),
    ])


def host_pairs(n, cp):
    """[element i][pv0, pv2, pv4] over the elements the chunk walk of chunks of cp pairs covers"""
    nch = len(range(0, (n + 4 + 1) // 2, cp))
    i = np.arange(2 * cp * nch)
    m = n - 2
    return np.stack([np.where(i < m, host_pv(i, 0), 0.0), np.where(i < m - 2, host_pv(i, 2), 0.0),
                     np.where(i < m - 4, host_pv(i, 4), 0.0)], axis=1)


def host_quotients():
    i = np.arange(NQ, dtype=np.float64)
    r = i + 2.0
    q = np.stack([1.0 / (4.0 * r * (r - 1.0)), 1.0 / (2.0 * (r * r - 1.0)), 1.0 / (4.0 * r * (r + 1.0)), i / (i + 2.0)], axis=1)
    q[0] = 0.0
    return q


def first_mismatch(got, want):
    """index of the first element whose bit pattern differs, or None"""
    bad = np.flatnonzero(got.view(np.uint64).ravel() != want.view(np.uint64).ravel())
    return None if bad.size == 0 else int(bad[0])


def compare(buf):
    """walk the harness output in its order; returns (number of values compared, list of mismatch descriptions)"""
    pos, checked, bad = 0, 0, []

    def take(want, what):
        nonlocal pos, checked
        want = np.ascontiguousarray(want, dtype=np.float64)
        got = buf[pos:pos + want.size].reshape(want.shape)
        assert got.size == want.size, f"harness output ends inside {what}"
        pos += want.size
        checked += want.size
        j = first_mismatch(got, want)
        if j is not None:
            idx = np.unravel_index(j, want.shape)
            g, w = got[idx], want[idx]
            bad.append(f"{what} at {tuple(int(v) for v in idx)}: got {g!r} ({int(np.float64(g).view(np.uint64)):#018x}) "
                       f"want {w!r} ({int(np.float64(w).view(np.uint64)):#018x}); "
                       f"{int((got.view(np.uint64) != want.view(np.uint64)).sum())} mismatches")

    for n in NS:
        fam = host_families(n)
        for f, name in enumerate(FAMILIES):
            take(fam[f], f"family {name} n={n} [i]")
        for cp in CPS:
            take(host_pairs(n, cp), f"pairs C={cp} n={n} [i, (pv0, pv2, pv4)]")
    take(host_quotients(), "quotients [i, (bc_rcp(4r(r-1)), bc_rcp(2(r^2-1)), bc_rcp(4r(r+1)), bc_div(i, i+2))]")
    assert pos == buf.size, (pos, buf.size)
    return checked, bad


def test_band_coef_harness_compiles_for_sm90a():
    with tempfile.TemporaryDirectory() as d:
        assert os.path.exists(compile_harness(d))


@pytest.mark.gpu
def test_band_coefficients_on_the_gpu_match_host_bit_for_bit():
    with tempfile.TemporaryDirectory() as d:
        exe = compile_harness(d)
        out = os.path.join(d, "coef.bin")
        r = subprocess.run([exe, out], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        buf = np.fromfile(out, dtype=np.float64)
    checked, bad = compare(buf)
    print(f"[band-coef] {checked} coefficients compared bit for bit, {len(bad)} groups with mismatches")
    for b in bad:
        print(f"[band-coef] {b}")
    assert not bad, bad
