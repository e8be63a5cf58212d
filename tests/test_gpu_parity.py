"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle on the
same seeded inputs.  Tolerance: 1e-10 relative for f64 spectral coefficients (north_star); mode
indexing (dealias cut, singular-mode removal) is exact."""
import numpy as np
import pytest

from tests import gpu_checks as g

pytestmark = pytest.mark.gpu

SPACES = [(1, 65, 1, 65), (2, 129, 1, 65), (0, 65, 0, 129), (2, 129, 2, 129), (4, 64, 1, 65), (4, 128, 0, 129),
          (4, 256, 2, 65), (1, 257, 1, 513), (1, 1025, 2, 129), (4, 2048, 1, 129), (2, 2049, 1, 65), (1, 65, 2, 4097)]
IDS = ["-".join(f"{g.KIND_NAME[s[i]]}{s[i+1]}" for i in (0, 2)) for s in SPACES]


@pytest.mark.parametrize("sp", SPACES, ids=IDS)
def test_layout_roundtrip_is_exact(sp):
    assert g.check_roundtrip_layout(*sp) == 0.0


@pytest.mark.parametrize("sp", SPACES, ids=IDS)
@pytest.mark.parametrize("op", ["forward", "backward", "to_ortho", "from_ortho"])
def test_field_ops(sp, op):
    assert getattr(g, "check_" + op)(*sp) < g.TOL


# lanes that run the E = 16 instances at their natural size: (16,4,64) along axis 0, (16,4,128) along axis 1, r2c (16,4,64)
E16 = [(1, 2049, 2, 65), (2, 65, 1, 4097), (4, 2048, 2, 65)]
E16_IDS = ["-".join(f"{g.KIND_NAME[s[i]]}{s[i+1]}" for i in (0, 2)) for s in E16]


@pytest.mark.parametrize("sp", SPACES[:7] + E16, ids=IDS[:7] + E16_IDS)
@pytest.mark.parametrize("deriv", [(1, 0), (0, 1), (2, 0), (0, 2), (1, 1)])
def test_gradient(sp, deriv):
    assert g.check_gradient(*sp, deriv) < g.TOL


@pytest.mark.parametrize("sp", [s for s in SPACES if s[0] != 0 and s[2] != 0][:6] + E16)
def test_hholtz_adi(sp):
    assert g.check_hholtz(*sp) < g.TOL


# (2,57,2,129) / (1,63,1,129): parity blocks of 28 / 27 rows and a one-tile last column block of the eigen-transform GEMM
@pytest.mark.parametrize("sp", [(2, 65, 2, 65), (2, 129, 2, 65), (2, 257, 2, 257), (4, 64, 2, 65), (4, 256, 2, 129),
                                (2, 57, 2, 129), (1, 63, 1, 129)] + E16)
def test_poisson(sp):
    assert g.check_poisson(*sp) < g.TOL


@pytest.mark.parametrize("sp", [(1, 65, 1, 65), (2, 129, 1, 65), (1, 257, 2, 257), (4, 64, 1, 65), (4, 256, 2, 129),
                                (1, 57, 2, 129), (2, 63, 1, 129)])
def test_hholtz_tensor(sp):
    """Hholtz (src/solver/hholtz.rs:66-101): the eigendecomposition form of the Helmholtz solve (own FP64 GEMM path)."""
    assert g.check_hholtz_tensor(*sp) < g.TOL


def test_reference_goldens_through_cuda():
    import rustpde_mpi_b200 as b2
    from tests.test_oracle_golden import GOLD_P2D

    f = b2.Field2(b2.Space2(b2.cheb_dirichlet(8), b2.cheb_dirichlet(7)))
    x = b2.Poisson(f, [1.0, 1.0]).solve(np.tile(np.arange(1.0, 8.0), (8, 1))).get()
    np.testing.assert_allclose(x, GOLD_P2D, atol=1.5e-6)  # src/solver/poisson.rs:295-325


def test_transform_roundtrip_large():
    """size-independent property at a BASELINE size: backward(forward(v)) == v on 1025 x 1025."""
    import rustpde_mpi_b200 as b2

    f = b2.Field2(b2.Space2(b2.cheb_dirichlet(1025), b2.cheb_dirichlet(1025)))
    a = np.random.default_rng(0).standard_normal(f.space.shape_spectral())
    f.vhat = a
    f.backward()
    f.forward()
    assert g.relerr(f.vhat, a) < 1e-9  # composite round trip amplifies by cond(S^T S)


def test_dealias_index_rule_is_exact():
    """functions.rs:72-82: rows >= shape0*2/3 and cols >= shape1*2/3 are exactly zero after one step's
    convection transform; checked through a Navier2D step on pres-sized arrays is indirect, so check
    the operator directly on the oracle's rule via the conv pipeline of a 65x65 step."""
    no, ng = g.make_navier_pair(65, 65, 1e5, 1.0, 0.01, 1.0, False)
    no.update(); ng.update(1)
    assert max(g.navier_errors(no, ng).values()) < g.TOL


@pytest.mark.parametrize("periodic", [False, True])
def test_navier_10_steps(periodic):
    errs = g.check_navier(64 if periodic else 65, 65, 10, periodic)
    assert max(errs.values()) < g.TOL, errs


def test_navier_c1_100_steps():
    """BASELINE config C1: 129 x 129, Ra 1e5, dt 0.01, examples/navier_rbc.rs initial fields, 100 steps."""
    errs = g.check_navier(129, 129, 100)
    assert max(errs.values()) < g.TOL, errs


def test_navier_random_init_257():
    errs = g.check_navier(257, 257, 3, False, 1e7, 1e-3, "random")
    assert max(errs.values()) < g.TOL, errs


def test_navier_periodic_random_256x129():
    errs = g.check_navier(256, 129, 3, True, 1e7, 1e-3, "random")
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.parametrize("periodic", [False, True])
def test_diagnostics_nu_nuvol_re(periodic):
    """callback() diagnostics (SURVEY 8f item 1): transforms / projections / derivatives on the GPU, weighted means on the host."""
    assert g.check_diagnostics(64 if periodic else 65, 65, 3, periodic) < 1e-10


# ---- bc = "hc" (SURVEY 8a row M, 8f item 2): ChebDirichletNeumann temperature base, PdmaPlus2 Helmholtz solves ----
HC_SPACES = [(2, 65, 3, 65), (2, 129, 3, 257), (4, 128, 3, 129), (1, 65, 3, 1025)]


@pytest.mark.parametrize("sp", HC_SPACES, ids=["-".join(f"{g.KIND_NAME[s[i]]}{s[i+1]}" for i in (0, 2)) for s in HC_SPACES])
@pytest.mark.parametrize("op", ["forward", "backward", "to_ortho", "from_ortho", "hholtz"])
def test_hc_field_ops(sp, op):
    """cdn axis: three-term stencil (odd offsets), pentadiagonal from_ortho, PdmaPlus2 (pdma_plus2.rs:45-157) in HholtzAdi."""
    assert getattr(g, "check_" + op)(*sp) < g.TOL


@pytest.mark.parametrize("periodic", [False, True])
def test_navier_hc_steps(periodic):
    """Navier2D::new_confined / new_periodic with bc = "hc" (navier.rs:245-252, 366-372; bc_hc boundary field)."""
    errs = g.check_navier(128 if periodic else 129, 129, 5, periodic, bc="hc")
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.parametrize("periodic,shape,shape2", [(False, (65, 65), (129, 65)), (True, (64, 65), (128, 129))])
def test_snapshot_write_read_and_interpolation(periodic, shape, shape2, tmp_path):
    """navier_io.rs:21-62 + field/io.rs:75-84,151-176: same grid = identical state, other grid = interpolate_2d + backward."""
    import rustpde_mpi_b200 as b2
    from rustpde_mpi_b200 import snapshot as sn

    a = b2.Navier2D(*shape, 1e5, 1.0, 0.01, 1.0, "rbc", periodic=periodic)
    a.update(3)
    fn = str(tmp_path / "snap.npz")
    a.write(fn)
    b = b2.Navier2D(*shape, 1e5, 1.0, 0.01, 1.0, "rbc", periodic=periodic)
    b.read(fn)
    assert abs(b.get_time() - a.get_time()) < 1e-15
    for k, v in a.state().items():
        assert np.array_equal(b.state()[k], v), k
    a.update(2); b.update(2)                       # a restarted run continues bit-identically
    for k, v in a.state().items():
        assert np.array_equal(b.state()[k], v), k
    c = b2.Navier2D(*shape2, 1e5, 1.0, 0.01, 1.0, "rbc", periodic=periodic)
    c.read(fn)
    data = sn.load_datasets(fn)
    for attr, group in sn.FIELD_GROUPS:
        f = getattr(c, attr)
        sh, cx = f.space.shape(b2.SPECTRAL)
        want = sn.read_vhat(data, group, sh, cx, periodic)
        assert np.array_equal(f.vhat, want), attr
