"""GPU parity (-m gpu) at transform sizes that are not 2^k (+1), and the FourierC2c base: the dense-matrix transforms (OP_DENSE) with the
generic-geometry operators.  Kept in the last GPU test file: these sizes are functional coverage of the reference's criterion benches
(benches/benchmark_navier.rs:6-7: 128, 264, 512 / 129, 265, 513), not the benchmarked path."""
import pytest

from tests import gpu_checks as g

pytestmark = pytest.mark.gpu

SIZES = [(128, 128, False), (264, 264, False), (265, 265, False), (512, 512, False), (264, 265, True), (100, 77, False)]


@pytest.mark.parametrize("nx,ny,periodic", SIZES)
def test_navier_reference_criterion_sizes(nx, ny, periodic):
    """Two steps from the reference example's smooth state (examples/navier_rbc.rs:18-22): 1e-10 on every field."""
    errs = g.check_navier(nx, ny, 2, periodic, 1e5, 0.01, "modes")
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.parametrize("nx,ny,periodic", SIZES)
def test_navier_reference_criterion_sizes_white_noise(nx, ny, periodic):
    """Two steps from white noise: bounded by the conditioning of the step itself (at 264^2 the velocity error exceeds 1e-10
    while the oracle moves by a comparable amount under a last-bit change of its input; temperature / pressure stay within 1e-10)."""
    errs, yard = g.check_navier_white_noise(nx, ny, 2, periodic)
    tol = max(g.TOL, 10.0 * yard)
    assert max(errs.values()) < tol, (errs, yard, tol)
    assert max(errs["temp"], errs["pres"]) < g.TOL, errs


def _assert_unsupported(sp, op):
    """A solver on a space it does not support fails at construction with B2_ERR_UNSUPPORTED (3) instead of solving wrongly."""
    import rustpde_mpi_b200 as b2

    _, fg = g.mk(*sp)
    make = {"hholtz": lambda: b2.HholtzAdi(fg, [0.02, 0.03]), "hholtz_tensor": lambda: b2.Hholtz(fg, [0.37, 1.3]),
            "poisson": lambda: b2.Poisson(fg, [1.0, 1.0])}[op]
    with pytest.raises(b2.B2Error, match=r"b200pde error 3:"):
        make()


@pytest.mark.parametrize("sp", [(1, 128, 1, 128), (2, 264, 1, 265), (4, 264, 2, 100), (0, 77, 0, 513)])
@pytest.mark.parametrize("op", ["forward", "backward", "hholtz"])
def test_field_ops_any_size(sp, op):
    if op == "hholtz" and 0 in (sp[0], sp[2]):   # HholtzAdi needs composite / Fourier axes: refused, not computed
        _assert_unsupported(sp, op)
        return
    assert getattr(g, "check_" + op)(*sp) < g.TOL


C2C_SPACES = [(5, 64, 1, 33), (5, 128, 2, 129), (5, 100, 1, 65), (5, 256, 0, 65)]


@pytest.mark.parametrize("sp", C2C_SPACES, ids=["-".join(f"{g.KIND_NAME[s[i]]}{s[i+1]}" for i in (0, 2)) for s in C2C_SPACES])
@pytest.mark.parametrize("op", ["roundtrip_layout", "forward", "backward", "to_ortho", "from_ortho", "gradient", "hholtz", "hholtz_tensor", "poisson"])
def test_fourier_c2c(sp, op):
    """FourierC2c on axis 0 (bases.rs:15): complex physical values, n modes in FFT order (no Navier2D configuration uses it)."""
    if op in ("hholtz", "hholtz_tensor", "poisson") and sp[2] == 0:   # the solvers need a composite Chebyshev axis 1
        _assert_unsupported(sp, op)
        return
    if op == "gradient":
        assert max(g.check_gradient(*sp, d) for d in ((1, 0), (0, 2), (2, 1), (3, 0))) < g.TOL
    else:
        e = getattr(g, "check_" + op)(*sp)
        assert e == 0.0 if op == "roundtrip_layout" else e < g.TOL
