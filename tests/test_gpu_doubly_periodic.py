"""Doubly periodic spaces, fourier_c2c(nx) x fourier_r2c(ny): physical values real (nx, ny), spectrum complex (nx, ny/2 + 1) with
the x modes in FFT order; forward = np.fft.rfft2, backward = np.fft.irfft2(., s=(nx, ny)).  The lanes along y are r2c lanes; the
lanes along x are split c2c lanes: lane 2j holds Re and lane 2j + 1 Im of column j, each runs the real FFT (OP_RFFT) and OP_CPAIR
joins the two half spectra into the complex one (lane_kernel.cuh, op_split).

Every case forces its layout through the switches make_cfg reads at space creation (B2_E, B2_LN, B2_NOFAST) and proves the layout
of its axis with Space2.layout() before anything else.  Transforms are checked against numpy's rfft2 / irfft2, gradients and the
solvers against the oracle's 1-D operators composed here.  tests/test_emu_doubly_periodic.py runs the small cases on the emulator."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R2C, C2C = 4, 5
SWITCHES = ("B2_E", "B2_LN", "B2_NOFAST")
TOL = 1e-10
CROSS = 64   # size of the other axis


def _cases():
    """(id, environment, nx, ny, axis, expected (E, LN, TPL, fast) of the lanes along that axis): natural layouts of the FFT sizes,
    then forced layouts, so that every compile-time instance and every generic (E, LN) pair an r2c lane reaches runs on each axis"""
    lays = [
        ("n64", {}, 64, (4, 4, 8, 1)), ("n128", {}, 128, (8, 4, 8, 1)), ("n256", {}, 256, (8, 4, 16, 1)),
        ("n512", {}, 512, (8, 4, 32, 1)), ("n1024", {}, 1024, (8, 4, 64, 1)), ("n2048", {}, 2048, (16, 4, 64, 1)),
        ("n4096", {}, 4096, (16, 4, 128, 1)), ("n8192", {}, 8192, (16, 2, 256, 1)),
        ("r3-192", {}, 192, (4, 4, 24, 0)), ("r5-320", {}, 320, (4, 4, 40, 0)), ("r3-384", {}, 384, (8, 4, 24, 0)),
        ("r3-768", {}, 768, (8, 4, 48, 0)), ("r3-1536", {}, 1536, (8, 4, 96, 0)), ("r3-3072", {}, 3072, (16, 4, 96, 0)),
        ("e16-256", {"B2_E": "16"}, 256, (16, 4, 8, 1)), ("e16-512", {"B2_E": "16"}, 512, (16, 4, 16, 1)),
        ("e16-1024", {"B2_E": "16"}, 1024, (16, 4, 32, 1)), ("e4-128", {"B2_E": "4"}, 128, (4, 4, 16, 1)),
        ("e4-256", {"B2_E": "4"}, 256, (4, 4, 32, 1)), ("ln2-4096", {"B2_LN": "2"}, 4096, (16, 2, 128, 1)),
        ("nofast-1024", {"B2_NOFAST": "1"}, 1024, (8, 4, 64, 0)), ("nofast-4096", {"B2_NOFAST": "1"}, 4096, (16, 4, 128, 0)),
        ("ln2-128", {"B2_LN": "2"}, 128, (4, 2, 16, 0)), ("ln2-256", {"B2_LN": "2"}, 256, (8, 2, 16, 0)),
        ("ln2-2048", {"B2_LN": "2"}, 2048, (16, 2, 64, 0)),
    ]
    out = []
    for name, env, n, want in lays:
        out.append((f"x-{name}", env, n, CROSS, 0, want))
        out.append((f"y-{name}", env, CROSS, n, 1, want))
    return out


CASES = _cases()
CASE = {c[0]: c[1:] for c in CASES}


def layout(nx, ny, axis):
    """(E, LN, TPL, fast) of the lanes along ``axis`` (orient 1: lanes along axis 0)"""
    import rustpde_mpi_b200 as b2

    s = b2.Space2((C2C, nx), (R2C, ny))
    lay = tuple(s.layout(1 - axis)[k] for k in ("E", "LN", "TPL", "fast"))
    s.close()
    return lay


def relerr(a, ref):
    a, ref = np.asarray(a), np.asarray(ref)
    assert a.shape == ref.shape, (a.shape, ref.shape)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-300))


def oracle_space(nx, ny):
    from oracle import rustpde_oracle as o

    return o.Space2(o.fourier_c2c(nx), o.fourier_r2c(ny))


def oracle_field(nx, ny):
    from oracle import rustpde_oracle as o

    return o.Field2(oracle_space(nx, ny))   # its operators (not its host arrays) serve as the solvers' reference


def rand_spec(nx, ny, rng):
    return rng.standard_normal((nx, ny // 2 + 1)) + 1j * rng.standard_normal((nx, ny // 2 + 1))


def smooth_phys(nx, ny, rng):
    """real values whose modes are |kx| <= nx / 4, ky <= ny / 4"""
    a = np.zeros((nx, ny // 2 + 1), dtype=np.complex128)
    bx, by = nx // 4, ny // 4
    kx = np.r_[0:bx + 1, nx - bx:nx]
    a[np.ix_(kx, np.arange(by + 1))] = rand_spec(kx.size, 2 * by, rng)
    return np.fft.irfft2(a, s=(nx, ny))


def decaying_spec(nx, ny, rng):
    """random spectrum decaying in |kx| + ky, so that third derivatives stay O(1) relative to the spectrum's scale"""
    kx = np.abs(np.fft.fftfreq(nx, 1.0 / nx))[:, None]
    ky = np.arange(ny // 2 + 1)[None, :]
    return rand_spec(nx, ny, rng) * np.exp(-((kx / (nx / 8.0)) ** 2 + (ky / (ny / 8.0)) ** 2))


def perturbed(a, seed):
    return a * (1.0 + 4e-16 * np.random.default_rng(seed).standard_normal(a.shape))


DERIVS = [(d0, d1) for d0 in range(4) for d1 in range(4)]


def grad_bound(d, a, scale, space):
    """TOL, or for a third derivative max(TOL, 10 x the oracle's last-bit yardstick) as the other third-derivative checks"""
    if 3 not in d:
        return TOL
    ref = space.gradient(a, d, scale)
    return max(TOL, 10.0 * relerr(space.gradient(perturbed(a, 77), d, scale), ref))


def solver_refs(nx, ny):
    """(name, c, oracle solver, library class) of HholtzAdi, Poisson and Hholtz"""
    import rustpde_mpi_b200 as b2
    from oracle import rustpde_oracle as o

    fo = oracle_field(nx, ny)
    return [("hholtz_adi", (0.02, 0.03), o.HholtzAdi(fo, [0.02, 0.03]), b2.HholtzAdi),
            ("poisson", (1.0, 1.0), o.Poisson(fo, [1.0, 1.0]), b2.Poisson),
            ("hholtz", (0.37, 1.3), o.Hholtz(fo, [0.37, 1.3]), b2.Hholtz)]


def solve_err(name, xg, xo):
    """Poisson::solve keeps the shifted-singular mode (0, 0), ~1e10 x the others: compared on its own, the rest without it"""
    if name != "poisson":
        return relerr(xg, xo)
    e00 = abs(xg[0, 0] - xo[0, 0]) / abs(xo[0, 0])
    xg, xo = xg.copy(), xo.copy()
    xg[0, 0] = xo[0, 0] = 0
    return max(e00, relerr(xg, xo))


def operator_errors(nx, ny, seed=21):
    """forward / backward against numpy on random and smooth values, round trip, to_ortho / from_ortho, every gradient d0, d1 <= 3
    scaled and unscaled, HholtzAdi, Poisson and Hholtz: ({name: error}, {name: bound})"""
    import rustpde_mpi_b200 as b2

    f = b2.Field2(b2.Space2((C2C, nx), (R2C, ny)))
    assert f.space.shape(b2.PHYSICAL) == ((nx, ny), False) and f.space.shape(b2.SPECTRAL) == ((nx, ny // 2 + 1), True)
    rng = np.random.default_rng(seed)
    errs = {}
    for name, v in (("random", rng.uniform(-1, 1, (nx, ny))), ("smooth", smooth_phys(nx, ny, rng))):
        f.v = v
        f.forward()
        errs[f"forward-{name}"] = relerr(f.vhat, np.fft.rfft2(v))
        f.backward()
        errs[f"roundtrip-{name}"] = relerr(f.v, v)
    for name, a in (("random", rand_spec(nx, ny, rng)), ("smooth", np.fft.rfft2(smooth_phys(nx, ny, rng)))):
        f.vhat = a
        f.backward()
        errs[f"backward-{name}"] = relerr(f.v, np.fft.irfft2(a, s=(nx, ny)))
    a = rand_spec(nx, ny, rng)
    f.vhat = a
    errs["to_ortho"] = relerr(f.to_ortho().get(), a)
    f.from_ortho(b2.DeviceArray(f.space, b2.ORTHO).set(2 * a))
    errs["from_ortho"] = relerr(f.vhat, 2 * a)
    bounds = {k: TOL for k in errs}
    space = oracle_space(nx, ny)
    a = decaying_spec(nx, ny, rng)
    f.vhat = a
    for d in DERIVS:
        for scale in ((1.7, 0.6), None):
            k = f"gradient{d}{'' if scale else '-unscaled'}"
            errs[k] = relerr(f.gradient(d, scale).get(), space.gradient(a, d, scale))
            bounds[k] = grad_bound(d, a, scale, space)
    rhs = rand_spec(nx, ny, rng)
    for name, c, so, cls in solver_refs(nx, ny):
        errs[name] = solve_err(name, cls(f, list(c)).solve(rhs).get(), so.solve(rhs))
        bounds[name] = TOL
    return errs, bounds


def call_sequence(nx, ny, seed=11):
    """One Field2, one ORTHO and one SPECTRAL output reused throughout, every destination NaN-filled before the operator that
    writes it: forward, to_ortho, from_ortho, backward, every gradient (scaled and unscaled), backward, forward, the three solvers
    twice each into the same output, and to_ortho after them (they share the space's scratch arrays).  Returns [(step, error,
    padding_excess of the destination)]; dealias must stay refused."""
    import rustpde_mpi_b200 as b2
    from rustpde_mpi_b200._lib import B2Error

    from tests import gpu_checks as g

    f = b2.Field2(b2.Space2((C2C, nx), (R2C, ny)))
    v, vhat = g.borrowed(f, 0), g.borrowed(f, 1)
    out, sout = b2.DeviceArray(f.space, b2.ORTHO), b2.DeviceArray(f.space, b2.SPECTRAL)
    rng = np.random.default_rng(seed)
    res = []
    x = rng.uniform(-1, 1, (nx, ny))
    f.v = x
    g.nan_fill(vhat); f.forward()
    res.append(("forward", relerr(f.vhat, np.fft.rfft2(x)), g.padding_excess(vhat)))
    ref = np.fft.rfft2(x)
    g.nan_fill(out); f.to_ortho(out=out)
    res.append(("to_ortho", relerr(out.get(), ref), g.padding_excess(out)))
    g.nan_fill(vhat); f.from_ortho(out)
    res.append(("from_ortho", relerr(f.vhat, ref), g.padding_excess(vhat)))
    g.nan_fill(v); f.backward()
    res.append(("backward", relerr(f.v, x), g.padding_excess(v)))
    space = oracle_space(nx, ny)
    a = decaying_spec(nx, ny, rng)
    f.vhat = a
    for d in DERIVS:
        for scale in ((1.5, 0.5), None):
            g.nan_fill(out); f.gradient(d, scale, out=out)
            # scaled so that sequence_failures' TOL stands for the step's own bound (grad_bound)
            e = relerr(out.get(), space.gradient(a, d, scale)) * TOL / grad_bound(d, a, scale, space)
            res.append((f"gradient{d}{'' if scale else '-unscaled'}", e, g.padding_excess(out)))
    try:
        f.dealias()
        res.append(("dealias refused", 1.0, 0.0))
    except B2Error:
        pass
    g.nan_fill(v); f.backward()
    res.append(("backward", relerr(f.v, np.fft.irfft2(a, s=(nx, ny))), g.padding_excess(v)))
    g.nan_fill(vhat); f.forward()
    res.append(("forward", relerr(f.vhat, np.fft.rfft2(np.fft.irfft2(a, s=(nx, ny)))), g.padding_excess(vhat)))
    rhs = rand_spec(nx, ny, rng)
    out.set(rhs)
    solvers = [(name, so, cls(f, list(c))) for name, c, so, cls in solver_refs(nx, ny)]
    for rep in range(2):
        for name, so, sg in solvers:
            g.nan_fill(sout); sg.solve(out, out=sout)
            res.append((f"{name}#{rep}", solve_err(name, sout.get(), so.solve(rhs)), g.padding_excess(sout)))
    f.vhat = a
    g.nan_fill(out); f.to_ortho(out=out)
    res.append(("to_ortho", relerr(out.get(), a), g.padding_excess(out)))
    return res


def sequence_failures(res, pad_tol=1e-13):
    return {f"{i}:{step}": (e, p) for i, (step, e, p) in enumerate(res) if not (e < TOL and p < pad_tol)}


def case_failures(nx, ny):
    errs, bounds = operator_errors(nx, ny)
    bad = {k: (e, bounds[k]) for k, e in errs.items() if not e < bounds[k]}
    bad.update(sequence_failures(call_sequence(nx, ny)))
    return bad, max(errs.values())


# every case in a process of its own: the layout switches are read when a space is created
SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
if sys.argv[2] == "emu":
    from tests import emu
    emu.activate()
from tests import test_gpu_doubly_periodic as t
case = json.loads(sys.argv[1])
_, nx, ny, axis, want = t.CASE[case]
lay = t.layout(nx, ny, axis)
assert lay == tuple(want), (case, lay, want)
bad, worst = t.case_failures(nx, ny)
assert not bad, bad
print("worst", worst)
print("ok")
''' % ROOT


def run_case(case, where):
    env = dict({k: v for k, v in os.environ.items() if k not in SWITCHES}, **CASE[case][0])
    r = subprocess.run([sys.executable, "-c", SCRIPT, json.dumps(case), where], capture_output=True, text=True, timeout=3600,
                       cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASE))
def test_doubly_periodic_case(case):
    """layout, transforms against numpy (random and smooth), round trip, to / from ortho, every gradient, HholtzAdi, Poisson and
    Hholtz, and the NaN-filled call sequence with its padding, at 1e-10 (third derivatives: max(1e-10, 10 x yardstick))"""
    run_case(case, "gpu")


@pytest.mark.gpu
def test_doubly_periodic_full_size():
    """4096 x 4096: forward and backward against numpy, and Poisson against the oracle"""
    import rustpde_mpi_b200 as b2

    n = 4096
    f = b2.Field2(b2.Space2((C2C, n), (R2C, n)))
    rng = np.random.default_rng(5)
    v = rng.uniform(-1, 1, (n, n))
    f.v = v
    f.forward()
    assert relerr(f.vhat, np.fft.rfft2(v)) < TOL
    a = rand_spec(n, n, rng)
    f.vhat = a
    f.backward()
    assert relerr(f.v, np.fft.irfft2(a, s=(n, n))) < TOL
    kx = np.fft.fftfreq(n, 1.0 / n)[:, None]
    ky = np.arange(n // 2 + 1)[None, :]
    lam = -kx ** 2 - 1e-10   # the oracle's FdmaTensor with diagonal systems, vectorised: f / (lam0 - c1 ky^2), c = (1, 1)
    xo = a / (lam - ky ** 2)
    assert solve_err("poisson", b2.Poisson(f, [1.0, 1.0]).solve(a).get(), xo) < TOL


# ---- Swift-Hohenberg, update_implicit of examples/swift_hohenberg_2d.rs:54-85, 280-302, composed from existing C-ABI calls ----
SH_R, SH_DT, SH_L = 0.35, 0.02, 20.0


def sh_matl(nx, ny):
    kx = np.fft.fftfreq(nx, 1.0 / nx)[:, None] / SH_L
    ky = np.arange(ny // 2 + 1)[None, :] / SH_L
    q = 1.0 - kx ** 2 - ky ** 2
    return 1.0 - SH_R * SH_DT + SH_DT * q * q


def sh_fix(vhat):
    """theta_hat[0, 0] = 0 and the Hermitian symmetry of the ky = 0 column (enforce_hermitian_symmetry)"""
    vhat[0, 0] = 0
    n = vhat.shape[0]
    i = np.arange(1, (n - 1) // 2 + 1)
    vhat[n - i, 0] = np.conj(vhat[i, 0])
    return vhat


def sh_numpy(theta0, steps):
    nx, ny = theta0.shape
    th = np.fft.rfft2(theta0)
    matl = sh_matl(nx, ny)
    for _ in range(steps):
        u = np.fft.irfft2(th, s=(nx, ny))
        rhs = th - SH_DT * np.fft.rfft2(u * u * u)
        th = sh_fix(rhs / matl)
    return th


def sh_gpu(theta0, steps):
    import ctypes as C

    import rustpde_mpi_b200 as b2
    from rustpde_mpi_b200._lib import check, lib

    from tests import gpu_checks as g

    nx, ny = theta0.shape
    f = b2.Field2(b2.Space2((C2C, nx), (R2C, ny)))
    v, vhat = g.borrowed(f, 0), g.borrowed(f, 1)
    sq = b2.DeviceArray(f.space, b2.PHYSICAL)
    rhs = b2.DeviceArray(f.space, b2.SPECTRAL)
    inv = 1.0 / sh_matl(nx, ny)
    minv = b2.DeviceArray(f.space, b2.SPECTRAL).set(inv + 1j * inv)   # Re and Im both 1 / matl: a pointwise product scales each mode
    f.v = theta0
    f.forward()
    for _ in range(steps):
        check(lib().b2_array_copy(rhs._h, vhat._h))
        f.backward()
        check(lib().b2_array_combine(sq._h, v._h, v._h, 0, C.c_double(1.0)))
        check(lib().b2_array_combine(v._h, v._h, sq._h, 0, C.c_double(1.0)))
        f.forward()
        rhs.axpy(-SH_DT, vhat)
        check(lib().b2_array_combine(vhat._h, rhs._h, minv._h, 0, C.c_double(1.0)))
        f.vhat = sh_fix(f.vhat)
    return f.vhat


@pytest.mark.gpu
@pytest.mark.parametrize("n", [128, 512])
def test_swift_hohenberg_implicit_steps(n):
    """50 implicit steps from the example's uniform +-0.1 random start against the same steps in numpy; the bound is max(1e-10,
    10 x the numpy run's own change when the start moves in the last bit)"""
    theta0 = np.random.default_rng(n).uniform(-0.1, 0.1, (n, n))
    ref = sh_numpy(theta0, 50)
    yard = relerr(sh_numpy(perturbed(theta0, 3), 50), ref)
    err = relerr(sh_gpu(theta0, 50), ref)
    print(f"[swift-hohenberg {n}^2] 50 steps: relative error {err:.2e}, yardstick {yard:.2e}")
    assert err < max(TOL, 10.0 * yard), (err, yard)
