"""Parity checks CUDA path (through the C ABI) vs the CPU oracle on the same seeded inputs.
Each check returns the relative error (max-norm of the difference / max-norm of the oracle
result).  Tolerance for f64 spectral coefficients: 1e-10 relative (BASELINE.json north_star)."""
import numpy as np

import rustpde_mpi_b200 as b2
from oracle import rustpde_oracle as o

TOL = 1e-10
KIND_NAME = {0: "ch", 1: "cd", 2: "cn", 3: "cdn", 4: "r2c", 5: "c2c"}


def relerr(a, ref):
    a, ref = np.asarray(a), np.asarray(ref)
    assert a.shape == ref.shape, (a.shape, ref.shape)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-300))


def mk(k0, n0, k1, n1):
    """(oracle Field2, CUDA Field2) on the same space."""
    fo = o.Field2(o.Space2(o.Base(k0, n0), o.Base(k1, n1)))
    fg = b2.Field2(b2.Space2((k0, n0), (k1, n1)))
    return fo, fg


def rand_phys(fo, rng, dist="normal"):
    """random physical values (complex on a FourierC2c axis 0)"""
    draw = (lambda: rng.standard_normal(fo.v.shape)) if dist == "normal" else (lambda: rng.uniform(-0.1, 0.1, fo.v.shape))
    return draw() + 1j * draw() if fo.v.dtype == np.complex128 else draw()


def rand_spec(fo, seed):
    rng = np.random.default_rng(seed)
    sh = fo.vhat.shape
    if fo.vhat.dtype == np.complex128:
        a = rng.standard_normal(sh) + 1j * rng.standard_normal(sh)
        a[0] = a[0].real  # DC and Nyquist modes of a real signal are real
        a[-1] = a[-1].real
        return a
    return rng.standard_normal(sh)


def check_roundtrip_layout(k0, n0, k1, n1, seed=0):
    fo, fg = mk(k0, n0, k1, n1)
    a = rand_spec(fo, seed)
    fg.vhat = a
    e1 = relerr(fg.vhat, a)
    v = rand_phys(fo, np.random.default_rng(seed))
    fg.v = v
    return max(e1, relerr(fg.v, v))


def check_forward(k0, n0, k1, n1, seed=1):
    fo, fg = mk(k0, n0, k1, n1)
    v = rand_phys(fo, np.random.default_rng(seed), "uniform")
    fo.v = v.copy(); fo.forward()
    fg.v = v; fg.forward()
    return relerr(fg.vhat, fo.vhat)


def check_backward(k0, n0, k1, n1, seed=2):
    fo, fg = mk(k0, n0, k1, n1)
    a = rand_spec(fo, seed)
    fo.vhat = a.copy(); fo.backward()
    fg.vhat = a; fg.backward()
    return relerr(fg.v, fo.v)


def check_to_ortho(k0, n0, k1, n1, seed=3):
    fo, fg = mk(k0, n0, k1, n1)
    a = rand_spec(fo, seed)
    fo.vhat = a.copy(); fg.vhat = a
    return relerr(fg.to_ortho().get(), fo.to_ortho())


def check_from_ortho(k0, n0, k1, n1, seed=4):
    fo, fg = mk(k0, n0, k1, n1)
    sh = fo.space.to_ortho(fo.vhat).shape
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(sh)
    if fo.vhat.dtype == np.complex128:
        a = a + 1j * rng.standard_normal(sh)
    fo.from_ortho(a.copy())
    fg.from_ortho(b2.DeviceArray(fg.space, b2.ORTHO).set(a))
    return relerr(fg.vhat, fo.vhat)


def check_gradient(k0, n0, k1, n1, deriv, scale=(1.5, 1.0), seed=5):
    fo, fg = mk(k0, n0, k1, n1)
    a = rand_spec(fo, seed)
    # physically sized spectrum: decay so that derivatives stay O(1)
    i = np.arange(a.shape[0])[:, None]; j = np.arange(a.shape[1])[None, :]
    a = a / (1.0 + i + j) ** 2
    fo.vhat = a.copy(); fg.vhat = a
    return relerr(fg.gradient(deriv, scale).get(), fo.gradient(deriv, scale))


def check_hholtz(k0, n0, k1, n1, c=(0.02, 0.03), seed=6):
    fo, fg = mk(k0, n0, k1, n1)
    ho = o.HholtzAdi(fo, list(c)); hg = b2.HholtzAdi(fg, list(c))
    sh = fo.space.to_ortho(fo.vhat).shape
    rng = np.random.default_rng(seed)
    rhs = rng.standard_normal(sh)
    if fo.vhat.dtype == np.complex128:
        rhs = rhs + 1j * rng.standard_normal(sh)
    return relerr(hg.solve(rhs).get(), ho.solve(rhs))


def check_poisson(k0, n0, k1, n1, c=(1.0, 1.0), seed=7):
    fo, fg = mk(k0, n0, k1, n1)
    eig = b2.poisson_eig(k0, n0, c[0]) if k0 in (1, 2) else None
    po = o.Poisson(fo, list(c), eig=eig); pg = b2.Poisson(fg, list(c))
    sh = fo.space.to_ortho(fo.vhat).shape
    rng = np.random.default_rng(seed)
    rhs = rng.standard_normal(sh)
    if fo.vhat.dtype == np.complex128:
        rhs = rhs + 1j * rng.standard_normal(sh)
    xo = po.solve(rhs); xg = pg.solve(rhs).get()
    xo[0, 0] = 0; xg[0, 0] = 0  # the shifted-singular mode is removed by the caller (navier_eq.rs:161)
    return relerr(xg, xo)


def check_hholtz_tensor(k0, n0, k1, n1, c=(0.37, 1.3), seed=9):
    """Hholtz (eigendecomposition form, src/solver/hholtz.rs) against the oracle; both sides get the same decomposition."""
    fo, fg = mk(k0, n0, k1, n1)
    eig = b2.hholtz_eig(k0, n0, c[0]) if k0 in (1, 2) else None
    ho = o.Hholtz(fo, list(c), eig=eig); hg = b2.Hholtz(fg, list(c))
    sh = fo.space.to_ortho(fo.vhat).shape
    rng = np.random.default_rng(seed)
    rhs = rng.standard_normal(sh)
    if fo.vhat.dtype == np.complex128:
        rhs = rhs + 1j * rng.standard_normal(sh)
    return relerr(hg.solve(rhs).get(), ho.solve(rhs))


def make_navier_pair(nx, ny, ra, pr, dt, aspect, periodic, init="modes", bc="rbc"):
    eig = None if periodic else b2.poisson_eig(b2.CHEB_NEUMANN, nx, 1.0 / aspect ** 2)
    no = o.Navier2D(nx, ny, ra, pr, dt, aspect, bc, periodic=periodic, pois_eig=eig)
    ng = b2.Navier2D(nx, ny, ra, pr, dt, aspect, bc, periodic=periodic)
    for nav in (no, ng):
        if init == "modes":
            nav.set_velocity(0.2, 1.0, 1.0)
            nav.set_temperature(0.2, 1.0, 1.0)
        else:
            nav.init_random(0.1)
    return no, ng


def navier_errors(no, ng):
    so, sg = no.state(), ng.state()
    out = {}
    for k in so:
        d = np.linalg.norm((sg[k] - so[k]).ravel())
        out[k] = float(d / max(np.linalg.norm(so[k].ravel()), 1e-300))
    return out


def check_navier(nx, ny, steps, periodic=False, ra=1e5, dt=0.01, init="modes", bc="rbc", mode=None):
    """``mode``: the step schedule of the CUDA side (Navier2D.set_mode: bit 0 fused, bit 1 no CUDA-graph replay, bit 2 no
    parallel branches); None keeps the default (fused, branches, graph replay)."""
    no, ng = make_navier_pair(nx, ny, ra, 1.0, dt, 1.0, periodic, init, bc)
    if mode is not None:
        ng.set_mode(mode)
    for _ in range(steps):
        no.update()
    ng.update(steps)
    return navier_errors(no, ng)


def check_navier_white_noise(nx, ny, steps, periodic=False, ra=1e5, dt=0.01):
    """White-noise initial fields (U(-0.1, 0.1) in physical space, navier.rs:171-182).  The projection step cancels a large
    divergent part of the intermediate velocity, so the step itself is conditioned well above rounding: returns the errors of the
    CUDA path against the oracle AND the yardstick = the oracle against itself when the same input is changed in the last bit
    (multiplied by 1 + 4e-16 N(0,1)); tests bound the error by max(TOL, 10 x yardstick) (same rule as test_gpu_parity_large)."""
    def fields(perturb):
        out = {}
        for name, seed in (("temp", 1), ("velx", 2), ("vely", 3)):
            f = np.random.default_rng(seed).uniform(-0.1, 0.1, size=(nx, ny))
            if perturb:
                f = f * (1.0 + 4e-16 * np.random.default_rng(100 + seed).standard_normal((nx, ny)))
            out[name] = f
        return out

    def start(nav, perturb):
        for name, f in fields(perturb).items():
            fld = getattr(nav, name)
            fld.v = f
            fld.forward()

    eig = None if periodic else b2.poisson_eig(b2.CHEB_NEUMANN, nx, 1.0)
    refs = []
    for perturb in (False, True):
        no = o.Navier2D(nx, ny, ra, 1.0, dt, 1.0, "rbc", periodic=periodic, pois_eig=eig)
        start(no, perturb)
        for _ in range(steps):
            no.update()
        refs.append(no)
    ng = b2.Navier2D(nx, ny, ra, 1.0, dt, 1.0, "rbc", periodic=periodic)
    start(ng, False)
    ng.update(steps)
    errs = navier_errors(refs[0], ng)
    yard = navier_errors(refs[0], refs[1])
    return errs, max(yard.values())


def check_diagnostics(nx, ny, steps, periodic=False):
    """Nu, Nuvol, Re (src/navier_stokes/functions.rs:146-233) after a few steps: CUDA path vs oracle, relative."""
    no, ng = make_navier_pair(nx, ny, 1e5, 1.0, 0.01, 1.0, periodic, "modes")
    for _ in range(steps):
        no.update()
    ng.update(steps)
    ref = (no.eval_nu(), no.eval_nuvol(), no.eval_re())
    got = (ng.eval_nu(), ng.eval_nuvol(), ng.eval_re())
    return max(abs(a - b) / abs(a) for a, b in zip(ref, got))
