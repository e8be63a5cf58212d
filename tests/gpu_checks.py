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


def decaying_spec(fo, seed):
    """random spectrum decaying like 1 / (1 + i + j)^2: physically sized, so that derivatives stay O(1)"""
    a = rand_spec(fo, seed)
    i = np.arange(a.shape[0])[:, None]; j = np.arange(a.shape[1])[None, :]
    return a / (1.0 + i + j) ** 2


def check_gradient(k0, n0, k1, n1, deriv, scale=(1.5, 1.0), seed=5):
    """``scale=None`` runs the unscaled path (a NULL scale through the C ABI)"""
    fo, fg = mk(k0, n0, k1, n1)
    a = decaying_spec(fo, seed)
    fo.vhat = a.copy(); fg.vhat = a
    return relerr(fg.gradient(deriv, scale).get(), fo.gradient(deriv, scale))


def op_errors(k0, n0, k1, n1, lane_axis):
    """Every field operator of one space against the oracle: forward, backward, to_ortho, from_ortho, the gradients (1,0),
    (0,1), (2,0), (0,2) and HholtzAdi (where neither axis is orthonormal Chebyshev) bounded by TOL; the third derivative along
    ``lane_axis`` by max(TOL, 10 x yardstick), the rule of the other third-derivative checks.  Returns ({op: error}, {op:
    (error, bound)} of the ops over their bound; NaN fails)."""
    sp = (k0, n0, k1, n1)
    errs = {op: globals()["check_" + op](*sp) for op in ("forward", "backward", "to_ortho", "from_ortho")}
    errs.update({f"gradient{d}": check_gradient(*sp, d) for d in ((1, 0), (0, 1), (2, 0), (0, 2))})
    if 0 not in (k0, k1):
        errs["hholtz_adi"] = check_hholtz(*sp)
    bound = {op: TOL for op in errs}
    d3 = (3, 0) if lane_axis == 0 else (0, 3)
    errs[f"gradient{d3}"], yard = check_gradient_yardstick(*sp, d3)
    bound[f"gradient{d3}"] = max(TOL, 10.0 * yard)
    return errs, {op: (e, bound[op]) for op, e in errs.items() if not e < bound[op]}


def neumann_stencil_mismatches(k0, n0, k1, n1):
    """to_ortho of a ChebNeumann lane next to an orthonormal Chebyshev axis (whose to_ortho is the identity), bit for bit.
    Lane l holds vhat_k = 1 at k = l (mod 4) and 0 elsewhere, so that one lane group covers every residue; the stencil
    ortho_j = vhat_j + s_{j-2} vhat_{j-2} then gives exactly 1 at j = l (mod 4), j < n - 2, exactly s_{j-2} = -((j-2) / j)^2
    at j = l + 2 (mod 4) (Base1::init_host: the IEEE quotient, squared) and 0 elsewhere.  Returns (number of elements whose
    bits differ, the first of them as (lane, j, got, want))."""
    lane_axis = 1 if k1 == CN else 0
    assert (k0, k1)[lane_axis] == CN and (k0, k1)[1 - lane_axis] == 0, (k0, k1)
    n, lanes = (n0, n1)[lane_axis], (n0, n1)[1 - lane_axis]
    m = n - 2
    l = np.arange(lanes)[:, None]
    k = np.arange(m)[None, :]
    vhat = (k % 4 == l % 4).astype(np.float64)
    j = np.arange(n)[None, :]
    jm2 = np.maximum(j - 2, 0).astype(np.float64)
    s = -(jm2 / (jm2 + 2.0)) ** 2
    want = np.where((j % 4 == l % 4) & (j < m), 1.0, np.where((j % 4 == (l + 2) % 4) & (j >= 2), s, 0.0))
    fg = b2.Field2(b2.Space2((k0, n0), (k1, n1)))
    fg.vhat = vhat if lane_axis == 1 else vhat.T
    got = fg.to_ortho().get()
    if lane_axis == 0:
        got = got.T
    got, want = np.ascontiguousarray(got) + 0.0, want + 0.0   # + 0.0: -0 and +0 compare equal (s_0 = -0)
    bad = np.argwhere(got.view(np.uint64) != want.view(np.uint64))
    if len(bad) == 0:
        return 0, None
    li, ji = bad[0]
    return len(bad), (int(li), int(ji), float(got[li, ji]), float(want[li, ji]))


def perturbed(a, seed):
    """``a`` changed in the last bit: multiplied by 1 + 4e-16 N(0,1) (the conditioning yardstick's input)"""
    return a * (1.0 + 4e-16 * np.random.default_rng(seed).standard_normal(a.shape))


def check_gradient_yardstick(k0, n0, k1, n1, deriv, scale=(1.5, 1.0), seed=5):
    """check_gradient's error AND the yardstick = the oracle against itself on the same spectrum changed in the last bit"""
    fo, fg = mk(k0, n0, k1, n1)
    a = decaying_spec(fo, seed)
    fo.vhat = a.copy(); fg.vhat = a
    ref = fo.gradient(deriv, scale)
    err = relerr(fg.gradient(deriv, scale).get(), ref)
    fo.vhat = perturbed(a, 1000 + seed)
    return err, relerr(fo.gradient(deriv, scale), ref)


# ---- the state a call leaves behind: padding and reused outputs ----
def borrowed(field, which):
    """non-owning DeviceArray over a field's ``v`` (which = 0) or ``vhat`` (1)"""
    import ctypes as C

    from rustpde_mpi_b200._lib import check, lib

    h = C.c_void_p()
    check(lib().b2_field_array(field._h, which, C.byref(h)))
    return b2.DeviceArray(field.space, b2.PHYSICAL if which == 0 else b2.SPECTRAL, handle=h, owner=False)


def padding_excess(arr):
    """|norm of the whole padded device array - norm of its logical elements| / the latter: nonzero when a store left
    anything in the padding (which the reductions over the padded array, norm2 / axpy / combine, would then see)"""
    host = float(np.linalg.norm(arr.get().ravel()))
    return abs(arr.norm() - host) / max(host, 1e-300)


def nan_fill(arr):
    """every logical element NaN (set() zeroes the padding before it uploads): an operator that leaves one unwritten fails"""
    shape = arr.local_shape()
    cx = arr.space.shape(arr.kind)[1]
    arr.set(np.full(shape, complex(np.nan, np.nan) if cx else np.nan))
    return arr


SEQ_DERIVS = ((1, 0), (0, 1), (2, 0), (0, 2), (1, 1), (3, 0), (0, 3))
CD, CN, R2C, C2C = 1, 2, 4, 5


def call_sequence(k0, n0, k1, n1, seed=11):
    """Generator over one space, one Field2, one ORTHO and one SPECTRAL output reused throughout; every destination is
    NaN-filled before the operator that writes it.  Yields (step, relative error against the oracle, padding_excess of the
    destination) after each step: forward, to_ortho, from_ortho, backward, gradients at SEQ_DERIVS (scaled and unscaled),
    dealias, backward, forward, then HholtzAdi / Poisson / Hholtz interleaved, each twice into the same output, and a last
    to_ortho after the solves (they share the space's scratch with the field operators)."""
    fo, fg = mk(k0, n0, k1, n1)
    v, vhat = borrowed(fg, 0), borrowed(fg, 1)
    out, sout = b2.DeviceArray(fg.space, b2.ORTHO), b2.DeviceArray(fg.space, b2.SPECTRAL)
    rng = np.random.default_rng(seed)

    fo.v = rand_phys(fo, rng, "uniform"); fg.v = fo.v
    nan_fill(vhat); fg.forward(); fo.forward()
    yield "forward", relerr(fg.vhat, fo.vhat), padding_excess(vhat)
    nan_fill(out); fg.to_ortho(out=out); ref = fo.to_ortho()
    yield "to_ortho", relerr(out.get(), ref), padding_excess(out)
    nan_fill(vhat); fg.from_ortho(out); fo.from_ortho(ref)
    yield "from_ortho", relerr(fg.vhat, fo.vhat), padding_excess(vhat)
    nan_fill(v); fg.backward(); fo.backward()
    yield "backward", relerr(fg.v, fo.v), padding_excess(v)

    a = decaying_spec(fo, seed)
    fo.vhat = a.copy(); fg.vhat = a
    for d in SEQ_DERIVS:
        for scale in ((1.5, 0.5), None):
            nan_fill(out); fg.gradient(d, scale, out=out)
            yield f"gradient{d}{'' if scale else '-unscaled'}", relerr(out.get(), fo.gradient(d, scale)), padding_excess(out)
    if k0 != C2C:   # the 2/3 rule is defined for r2c / Chebyshev mode order only
        fg.dealias(); o.dealias(fo.vhat)
        yield "dealias", relerr(fg.vhat, fo.vhat), padding_excess(vhat)
    nan_fill(v); fg.backward(); fo.backward()
    yield "backward", relerr(fg.v, fo.v), padding_excess(v)
    nan_fill(vhat); fg.forward(); fo.forward()
    yield "forward", relerr(fg.vhat, fo.vhat), padding_excess(vhat)

    solvers = []
    if 0 not in (k0, k1):
        solvers.append(("hholtz_adi", o.HholtzAdi(fo, [0.02, 0.03]), b2.HholtzAdi(fg, [0.02, 0.03])))
    # Poisson / Hholtz: the lane kernel runs their per-row LU along axis 1; a long confined axis 0 only adds the host LAPACK
    # eigendecomposition (tens of seconds beyond 1025 points)
    if k0 in (CD, CN, R2C) and k1 in (CD, CN) and (k0 == R2C or n0 <= 1025):
        eig = b2.poisson_eig(k0, n0, 1.0) if k0 != R2C else None
        solvers.append(("poisson", o.Poisson(fo, [1.0, 1.0], eig=eig), b2.Poisson(fg, [1.0, 1.0])))
        eig = b2.hholtz_eig(k0, n0, 0.37) if k0 != R2C else None
        solvers.append(("hholtz", o.Hholtz(fo, [0.37, 1.3], eig=eig), b2.Hholtz(fg, [0.37, 1.3])))
    if solvers:
        sh, cx = fg.space.shape(b2.ORTHO)
        rhs = rng.standard_normal(sh) + (1j * rng.standard_normal(sh) if cx else 0.0)
        out.set(rhs)
        for rep in range(2):
            for name, so, sg in solvers:
                nan_fill(sout); sg.solve(out, out=sout)
                xo, xg = so.solve(rhs), sout.get()
                if name == "poisson":
                    xo[0, 0] = 0; xg[0, 0] = 0   # the shifted-singular mode is removed by the caller (navier_eq.rs:161)
                yield f"{name}#{rep}", relerr(xg, xo), padding_excess(sout)
        nan_fill(out); fg.to_ortho(out=out)
        yield "to_ortho", relerr(out.get(), fo.to_ortho()), padding_excess(out)


def run_sequences(*spaces, seed=11):
    """Run the call sequences of several spaces in one context, alternating step by step (every step switches the space and
    with it the lane-kernel instances, the staging buffer size and the solver workspaces).  Returns {space: [(step, err,
    padding_excess)]}."""
    gens = {sp: call_sequence(*sp, seed=seed) for sp in spaces}
    res = {sp: [] for sp in spaces}
    while gens:
        for sp in list(gens):
            try:
                res[sp].append(next(gens[sp]))
            except StopIteration:
                del gens[sp]
    return res


def sequence_failures(res, pad_tol=1e-13):
    """the steps of run_sequences' result over TOL or the padding bound (NaN fails both)"""
    return {f"{sp}:{i}:{step}": (e, p) for sp, steps in res.items() for i, (step, e, p) in enumerate(steps)
            if not (e < TOL and p < pad_tol)}


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


def bench_coefficients(ra, dt, aspect=1.0, pr=1.0):
    """the Helmholtz coefficients of a Navier2D step, as b2_navier2d_create computes them: (c_velocity, c_temperature) with
    c = (dt nu / aspect^2, dt nu) and nu = sqrt(pr / (ra / 8)), ka = sqrt(1 / (ra / 8 pr)) (height 2, functions.rs:12-21)"""
    nu = np.sqrt(pr / (ra / 2.0 ** 3)); ka = np.sqrt(1.0 / ((ra / 2.0 ** 3) * pr))
    return (dt * nu / aspect ** 2, dt * nu), (dt * ka / aspect ** 2, dt * ka)


def check_solver_yardstick(name, k0, n0, k1, n1, c, seed=8):
    """``name`` in hholtz_adi / poisson / hholtz on a white-noise right-hand side: the error against the oracle AND the
    yardstick = the oracle against itself on the right-hand side changed in the last bit (x (1 + 4e-16 N(0,1)))"""
    fo, fg = mk(k0, n0, k1, n1)
    if name == "hholtz_adi":
        so, sg = o.HholtzAdi(fo, list(c)), b2.HholtzAdi(fg, list(c))
    else:
        eig = (b2.poisson_eig if name == "poisson" else b2.hholtz_eig)(k0, n0, c[0]) if k0 in (CD, CN) else None
        so, sg = (o.Poisson, o.Hholtz)[name == "hholtz"](fo, list(c), eig=eig), (b2.Poisson, b2.Hholtz)[name == "hholtz"](fg, list(c))
    sh, cx = fg.space.shape(b2.ORTHO)
    rng = np.random.default_rng(seed)
    rhs = rng.standard_normal(sh) + (1j * rng.standard_normal(sh) if cx else 0.0)
    xo, xp, xg = so.solve(rhs), so.solve(perturbed(rhs, 1000 + seed)), sg.solve(rhs).get()
    if name == "poisson":
        for x in (xo, xp, xg):
            x[0, 0] = 0   # the shifted-singular mode is removed by the caller (navier_eq.rs:161)
    return relerr(xg, xo), relerr(xp, xo)


def check_navier_padding(nav):
    """padding_excess of v and vhat of every state and work field of a CUDA Navier2D, and div_norm() against the host norm
    of div(): {name: value}"""
    out = {}
    for name in ("temp", "velx", "vely", "pres", "pseu"):
        f = getattr(nav, name)
        for which in (0, 1):
            out[f"{name}.{'vhat' if which else 'v'}"] = padding_excess(borrowed(f, which))
    d = float(np.linalg.norm(nav.div().ravel()))
    out["div_norm"] = abs(nav.div_norm() - d) / max(d, 1e-300)
    return out


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


def share_tempbc(no, ng):
    """Hand the oracle the CUDA side's boundary field tempbc.  Each side builds tempbc with its own grid, cos and transforms,
    so the coefficients differ by a transform's round-off (~1e-15 of the largest); with bc = "hc" tempbc varies along x and the
    step adds dt ka d2/dx2 tempbc, which multiplies that round-off in the high modes by ~k^4 (6e-10 in temp after two steps at
    1025 x 129).  With the same tempbc on both sides the comparison measures the step alone."""
    no.tempbc.vhat = np.array(ng.tempbc.vhat)
    no.tempbc.backward()


def check_navier(nx, ny, steps, periodic=False, ra=1e5, dt=0.01, init="modes", bc="rbc", mode=None, same_tempbc=False):
    """``mode``: the step schedule of the CUDA side (Navier2D.set_mode: bit 0 fused, bit 1 no CUDA-graph replay, bit 2 no
    parallel branches); None keeps the default (fused, branches, graph replay).  ``same_tempbc``: share_tempbc first."""
    no, ng = make_navier_pair(nx, ny, ra, 1.0, dt, 1.0, periodic, init, bc)
    if same_tempbc:
        share_tempbc(no, ng)
    if mode is not None:
        ng.set_mode(mode)
    for _ in range(steps):
        no.update()
    ng.update(steps)
    return navier_errors(no, ng)


def check_navier_tempbc_yardstick(nx, ny, steps, ra=1e5, dt=0.01, bc="hc", seeds=(1, 2)):
    """Smooth-state steps with each side's own tempbc: the errors of the CUDA path against the oracle AND the yardstick = the
    largest change of the oracle when tempbc's coefficients get a transform's round-off, + 4e-16 max|vhat| N(0,1) on every
    mode (share_tempbc: that round-off is the whole difference between the two sides' tempbc)."""
    eig = b2.poisson_eig(b2.CHEB_NEUMANN, nx, 1.0)
    ng = b2.Navier2D(nx, ny, ra, 1.0, dt, 1.0, bc)
    navs = [ng] + [o.Navier2D(nx, ny, ra, 1.0, dt, 1.0, bc, pois_eig=eig) for _ in range(1 + len(seeds))]
    for nav in navs:
        nav.set_velocity(0.2, 1.0, 1.0)
        nav.set_temperature(0.2, 1.0, 1.0)
    no, refs = navs[1], navs[2:]
    for nr, seed in zip(refs, seeds):
        vh = nr.tempbc.vhat
        nr.tempbc.vhat = vh + 4e-16 * np.abs(vh).max() * np.random.default_rng(seed).standard_normal(vh.shape)
        nr.tempbc.backward()
    for _ in range(steps):
        for nav in [no] + refs:
            nav.update()
    ng.update(steps)
    return navier_errors(no, ng), max(max(navier_errors(no, nr).values()) for nr in refs)


def check_navier_white_noise(nx, ny, steps, periodic=False, ra=1e5, dt=0.01, bc="rbc", same_tempbc=False):
    """White-noise initial fields (U(-0.1, 0.1) in physical space, navier.rs:171-182).  The projection step cancels a large
    divergent part of the intermediate velocity, so the step itself is conditioned well above rounding: returns the errors of the
    CUDA path against the oracle AND the yardstick = the oracle against itself when the same input is changed in the last bit
    (multiplied by 1 + 4e-16 N(0,1)); tests bound the error by max(TOL, 10 x yardstick) (same rule as test_gpu_parity_large).
    ``same_tempbc``: both oracle runs take the CUDA side's tempbc (share_tempbc)."""
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
    ng = b2.Navier2D(nx, ny, ra, 1.0, dt, 1.0, bc, periodic=periodic)
    refs = []
    for perturb in (False, True):
        no = o.Navier2D(nx, ny, ra, 1.0, dt, 1.0, bc, periodic=periodic, pois_eig=eig)
        if same_tempbc:
            share_tempbc(no, ng)
        start(no, perturb)
        for _ in range(steps):
            no.update()
        refs.append(no)
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
