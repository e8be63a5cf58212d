"""GPU parity at the BENCHMARKED configurations (BASELINE.json configs[1..4]): whole Navier2D steps from a random
initial state against the CPU checkers, plus the operator instances the small suite cannot reach (lanes longer than
4100 points) and a bit-exact test of the dealias index rule.

Checkers: the numpy oracle (pinned to the reference's goldens) where it finishes in seconds, and
oracle/cpu_restated.cpp (C++/OpenMP; tests/test_cpu_restated.py checks it against the numpy oracle) for the 4097^2 and
8192 x 4097 steps.  Tolerance: 1e-10 relative (north_star).  Both sides get the same host eigendecomposition of the
Poisson operator (DESIGN.md, "Poisson parity")."""
import numpy as np
import pytest

from tests import gpu_checks as g

pytestmark = pytest.mark.gpu
TOL = 1e-10


def _rel(a, ref):
    return float(np.abs(a - ref).max() / np.abs(ref).max())


def _make(kind, nx, ny, ra, dt, periodic, eig):
    if kind == "numpy":
        from oracle import rustpde_oracle as o

        nav = o.Navier2D(nx, ny, ra, 1.0, dt, 1.0, "rbc", periodic=periodic, pois_eig=eig)
        nav.nx, nav.ny = nx, ny
        return nav
    if kind == "cpp":
        from oracle import cpu_restated as cr

        return cr.Navier2D(nx, ny, ra, 1.0, dt, 1.0, "rbc", periodic=periodic, pois_eig=eig)
    import rustpde_mpi_b200 as b2

    return b2.Navier2D(nx, ny, ra, 1.0, dt, 1.0, "rbc", periodic=periodic, pois_eig=eig)


def _fields(nx, ny, perturb):
    """the bench's synthetic state: U(-0.1, 0.1) physical fields from default_rng(1/2/3) (navier.rs:171-182);
    ``perturb``: multiplied by (1 + 4e-16 N(0,1)) -- a rounding-level change of the input, the conditioning yardstick."""
    out = {}
    for name, seed in (("temp", 1), ("velx", 2), ("vely", 3)):
        f = np.random.default_rng(seed).uniform(-0.1, 0.1, size=(nx, ny))
        if perturb:
            f = f * (1.0 + 4e-16 * np.random.default_rng(100 + seed).standard_normal((nx, ny)))
        out[name] = f
    return out


def _run(nav, kind, init, steps, perturb=False):
    if init == "random":
        for name, f in _fields(nav.nx, nav.ny, perturb).items():
            if kind == "cpp":
                nav.set_v(name, f)
            else:
                fld = getattr(nav, name)
                fld.v = f
                fld.forward()
    else:                     # the reference example's smooth initial state (examples/navier_rbc.rs:18-22)
        nav.set_velocity(0.2, 1.0, 1.0)
        nav.set_temperature(0.2, 1.0, 1.0)
    if kind == "numpy":
        for _ in range(steps):
            nav.update()
    else:
        nav.update(steps)
    return nav.state()


def _errs(got, ref):
    return {k: _rel(got[k], v) for k, v in ref.items()}


def _step_parity(nx, ny, ra, dt, periodic, steps, checkers, init):
    """GPU against the checker(s).  Smooth initial state: 1e-10 (north_star).  White-noise initial state (what bench.py
    times): the projection step cancels a large divergent part of the intermediate velocity, which conditions the step
    itself at ~1e-8 on 1025^2 and ~1e-6 on 4097^2 -- two independent CPU restatements differ by that much, and so does ONE
    restatement when its input is changed in the last bit -- so the bound is the larger of 1e-10 and 10x the spread
    between two checkers (or between the checker and itself on a rounding-level perturbation of the same input)."""
    import rustpde_mpi_b200 as b2

    eig = None if periodic else b2.poisson_eig(b2.CHEB_NEUMANN, nx, 1.0)
    refs = [_run(_make(c, nx, ny, ra, dt, periodic, eig), c, init, steps) for c in checkers]
    if init == "random" and len(refs) == 1:
        refs.append(_run(_make(checkers[0], nx, ny, ra, dt, periodic, eig), checkers[0], init, steps, perturb=True))
    nav = _make("gpu", nx, ny, ra, dt, periodic, eig)
    got = _run(nav, "gpu", init, steps)   # default schedule: fused, parallel branches, CUDA-graph replay from the second step on
    nav.close()
    errs = _errs(got, refs[0])
    tol = TOL
    if init == "random":
        tol = max(TOL, 10.0 * max(_errs(refs[1], refs[0]).values()))
    print(f"{nx}x{ny} periodic={periodic} init={init}: GPU vs {checkers[0]} {errs}  tol {tol:.1e}")
    assert max(errs.values()) < tol, (errs, tol)


CFG = {"C2": (1025, 1025, 1e7, 1e-3, False), "C3": (2048, 1025, 1e7, 1e-3, True),
       "C4": (4097, 4097, 1e9, 1e-4, False), "C5": (8192, 4097, 1e10, 5e-5, True)}


@pytest.mark.parametrize("cfg", ["C2", "C3"])
def test_step_smooth_state_numpy_oracle(cfg):
    """configs[1], configs[2]: 2 steps from the example's smooth state against the numpy oracle, 1e-10."""
    _step_parity(*CFG[cfg], 2, ["numpy"], "smooth")


@pytest.mark.parametrize("cfg", ["C2", "C3"])
def test_step_random_state_two_checkers(cfg):
    """the bench's white-noise state at configs[1], configs[2]: numpy oracle, spread measured against the C++ checker."""
    _step_parity(*CFG[cfg], 2, ["numpy", "cpp"], "random")


@pytest.mark.parametrize("cfg", ["C4", "C5"])
def test_step_smooth_state_cpp_checker(cfg):
    """configs[3] (the default bench workload: parity-split GEMM operands, graph replay) and configs[4] (8192-point
    Fourier lanes): 2 steps from the smooth state against the C++ checker, 1e-10."""
    _step_parity(*CFG[cfg], 2, ["cpp"], "smooth")


def test_c4_random_state_cpp_checker():
    _step_parity(*CFG["C4"], 2, ["cpp"], "random")


LONG = [(1, 65, 0, 8193), (4, 8192, 1, 65), (0, 8193, 1, 65), (2, 65, 2, 8193)]
LONG_IDS = ["-".join(f"{g.KIND_NAME[s[i]]}{s[i+1]}" for i in (0, 2)) for s in LONG]
# HholtzAdi needs a base with boundary conditions (or Fourier) on both axes
LONG_CASES = [(sp, op, f"{op}-{sid}") for op in ["roundtrip_layout", "forward", "backward", "to_ortho", "from_ortho", "hholtz", "gradient"]
              for sp, sid in zip(LONG, LONG_IDS) if op != "hholtz" or 0 not in (sp[0], sp[2])]


@pytest.mark.parametrize("sp,op", [c[:2] for c in LONG_CASES], ids=[c[2] for c in LONG_CASES])
def test_long_lane_ops(sp, op):
    """8192 / 8193-point lanes (the C5 / 8193^2 kernel instances): transforms, derivatives and HholtzAdi."""
    if op == "gradient":
        e = max(g.check_gradient(*sp, d) for d in ((1, 0), (0, 1), (2, 0), (0, 2)))
    else:
        e = getattr(g, "check_" + op)(*sp)
    assert e == 0.0 if op == "roundtrip_layout" else e < TOL


@pytest.mark.parametrize("sp", [(1, 65, 1, 65), (2, 129, 1, 65), (4, 64, 1, 65), (4, 256, 2, 129), (0, 65, 0, 129), (1, 1025, 2, 129)])
def test_dealias_index_rule_bit_exact(sp):
    """dealias(): vhat[n_x.., :] = 0, vhat[:, n_y..] = 0 with n = shape * 2 / 3 (integer), everything else untouched
    bit for bit (src/navier_stokes/functions.rs:72-82)."""
    import rustpde_mpi_b200 as b2

    f = b2.Field2(b2.Space2((sp[0], sp[1]), (sp[2], sp[3])))
    shape, cx = f.space.shape(b2.SPECTRAL)
    rng = np.random.default_rng(5)
    a = rng.standard_normal(shape) + (1j * rng.standard_normal(shape) if cx else 0.0)
    f.vhat = a
    f.dealias()
    want = np.array(a, copy=True)
    want[shape[0] * 2 // 3:, :] = 0
    want[:, shape[1] * 2 // 3:] = 0
    assert np.array_equal(f.vhat, want)
