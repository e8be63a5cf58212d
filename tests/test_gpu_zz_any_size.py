"""GPU parity (-m gpu) at transform sizes that are not 2^k (+1), and the FourierC2c base: the dense-matrix transforms (OP_DENSE) with the
generic-geometry operators.  Kept in the last GPU test file: these sizes are functional coverage of the reference's criterion benches
(benches/benchmark_navier.rs:6-7: 128, 264, 512 / 129, 265, 513), not the benchmarked path."""
import pytest

from tests import gpu_checks as g

pytestmark = pytest.mark.gpu

SIZES = [(128, 128, False), (264, 264, False), (265, 265, False), (512, 512, False), (264, 265, True), (100, 77, False),
         (1000, 129, False)]
# the lanes along axis 0 (orient 1) of a size's cd x cd space where a test depends on their layout: 1000-point lanes run the
# generic instance at TPL 32 (test_gpu_instances.layout_jobs checks this on the emulator)
SIZE_LAYOUTS = {(1000, 129, False): {"E": 16, "LN": 4, "TPL": 32, "fast": 0}}


def assert_size_layout(nx, ny, periodic):
    if (nx, ny, periodic) in SIZE_LAYOUTS:
        import rustpde_mpi_b200 as b2

        s = b2.Space2((1, nx), (1, ny))
        lay = s.layout(1)
        s.close()
        assert {k: lay[k] for k in ("E", "LN", "TPL", "fast")} == SIZE_LAYOUTS[(nx, ny, periodic)]


@pytest.mark.parametrize("nx,ny,periodic", SIZES)
def test_navier_reference_criterion_sizes(nx, ny, periodic):
    """Two steps from the reference example's smooth state (examples/navier_rbc.rs:18-22): 1e-10 on every field."""
    assert_size_layout(nx, ny, periodic)
    errs = g.check_navier(nx, ny, 2, periodic, 1e5, 0.01, "modes")
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.parametrize("nx,ny,periodic", SIZES)
def test_navier_reference_criterion_sizes_white_noise(nx, ny, periodic):
    """Two steps from white noise: bounded by the conditioning of the step itself (at 264^2 the velocity error exceeds 1e-10
    while the oracle moves by a comparable amount under a last-bit change of its input; temperature / pressure stay within 1e-10)."""
    assert_size_layout(nx, ny, periodic)
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


CH, CD, CN, R2C, C2C = 0, 1, 2, 4, 5
# (space, orient of the dense lane, TPL of the generic <16, 4, 0> instance it runs): the longest dense lanes, TPL 32 (lanes of
# 545 .. 1088 padded rows) and 64 (up to 2049 points), on both axes and for every base kind with a dense transform
DENSE = [((CD, 1000, CN, 65), 1, 32), ((CN, 2000, CD, 65), 1, 64), ((CD, 65, CD, 1000), 0, 32), ((CN, 65, CN, 2000), 0, 64),
         ((CH, 65, CH, 2000), 0, 64), ((R2C, 1000, CD, 65), 1, 32), ((R2C, 2046, CN, 65), 1, 64), ((C2C, 1000, CD, 65), 1, 64)]


def dense_id(sp):
    return "-".join(f"{g.KIND_NAME[sp[i]]}{sp[i + 1]}" for i in (0, 2))


@pytest.mark.parametrize("sp,orient,tpl", DENSE, ids=[dense_id(d[0]) for d in DENSE])
def test_dense_lanes_at_every_generic_tpl(sp, orient, tpl):
    """field ops, gradients, HholtzAdi and (where the space has them) Poisson and Hholtz with the dense-transform lane at TPL
    32 and 64"""
    import rustpde_mpi_b200 as b2

    s = b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))
    lay = s.layout(orient)
    s.close()
    assert {k: lay[k] for k in ("E", "LN", "TPL", "fast")} == {"E": 16, "LN": 4, "TPL": tpl, "fast": 0}
    errs, bad = g.op_errors(*sp, lane_axis=1 - orient)
    # Poisson / Hholtz: per-row LU along axis 1; a long confined axis 0 only adds the host's eigendecomposition
    if sp[0] in (CD, CN, R2C, C2C) and sp[2] in (CD, CN) and (sp[0] in (R2C, C2C) or sp[1] <= 1025):
        errs.update(poisson=g.check_poisson(*sp), hholtz=g.check_hholtz_tensor(*sp))
        bad.update({op: (errs[op], g.TOL) for op in ("poisson", "hholtz") if not errs[op] < g.TOL})
    print(f"[any-size] {dense_id(sp)}: worst err {max(errs.values()):.2e} ({max(errs, key=errs.get)})")
    assert not bad, bad


def test_dense_transform_size_limits():
    """a Chebyshev lane of 2048 points (N = 2047) runs the dense transform; 2050 (N = 2049) is refused with B2_ERR_UNSUPPORTED
    (3) at its first transform, on either axis; r2c with odd n and c2c beyond 1024 are refused when the space is created"""
    import rustpde_mpi_b200 as b2

    assert max(g.check_forward(CD, 2048, CN, 65), g.check_backward(CD, 2048, CN, 65)) < g.TOL
    for sp in ((CD, 2050, CN, 65), (CD, 65, CD, 2050)):
        f = b2.Field2(b2.Space2((sp[0], sp[1]), (sp[2], sp[3])))
        with pytest.raises(b2.B2Error, match=r"b200pde error 3:"):
            f.forward()
    for sp in ((R2C, 1001, CD, 65), (C2C, 1025, CD, 65)):
        with pytest.raises(b2.B2Error, match=r"b200pde error 3:"):
            b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))


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
