"""The operators as the time step and its callers use them, on the GPU (-m gpu).  The parity tests run every operator once
on fresh, zero-filled objects; here:

- call sequences on one space (gpu_checks.call_sequence): every destination NaN-filled before the operator that writes it,
  one ORTHO and one SPECTRAL output reused throughout, all three solvers interleaved on the space's shared scratch; after
  every step the oracle at TOL and no stray value in the padding (padding_excess < 1e-13; norm2 / axpy / combine run over
  the padded array).  At every lane-kernel instance of test_gpu_instances.CASES (forced and asserted the same way), the cdn
  cases, r2c x cdn, c2c x cd;
- a small and a large space alternating step by step in one context (staging buffer growth, per-instance launch attributes);
- every derivative order (d0, d1) in 0..3, scaled and unscaled;
- HholtzAdi / Poisson / Hholtz at the Helmholtz coefficients of the benchmarked configurations (c = dt nu / s^2 ~ 9e-5 ..
  1.4e-9) on their lane lengths, white-noise right-hand sides;
- the padding of every Navier2D field after steps in every schedule and at the forced layouts, and div_norm() against the
  host norm of div().

Bounds: TOL, except where the operation itself is conditioned above rounding: there max(TOL, 10 x yardstick), the oracle
against itself on the input changed in the last bit (the rule of check_navier_white_noise)."""
import pytest

from tests import gpu_checks as g
from tests import test_gpu_instances as ti
from tests.test_gpu_parity import E16, E16_IDS, IDS, SPACES

pytestmark = pytest.mark.gpu
CD, CN, CDN, R2C, C2C = 1, 2, 3, 4, 5
PAD_TOL = 1e-13


def sid(sp):
    return "-".join(f"{g.KIND_NAME[sp[i]]}{sp[i + 1]}" for i in (0, 2))


def report(tag, res):
    worst = max((e for steps in res.values() for _, e, _ in steps), default=0.0)
    pad = max((p for steps in res.values() for _, _, p in steps), default=0.0)
    print(f"[call-contract] {tag}: worst err {worst:.2e}, worst padding_excess {pad:.2e}")


def assert_sequences(tag, *spaces):
    res = g.run_sequences(*spaces)
    report(tag, res)
    bad = g.sequence_failures(res, PAD_TOL)
    assert not bad, bad


# ---- call sequences ----
@pytest.mark.parametrize("case,sp,orient", ti.PLACED, ids=ti.PLACED_IDS)
def test_instance_call_sequence(case, sp, orient, monkeypatch):
    ti.set_env(monkeypatch, ti.CASE[case][1])
    assert ti.layout_of(sp, orient) == ti.want(case)
    assert_sequences(f"seq {case} {sid(sp)}", sp)


@pytest.mark.parametrize("case", ti.CDN_CASES)
def test_instance_cdn_call_sequence(case, monkeypatch):
    ti.set_env(monkeypatch, ti.CASE[case][1])
    sp = ti.cdn_space(case)
    assert ti.layout_of(sp, 0) == ti.want(case)
    assert_sequences(f"seq {case} {sid(sp)}", sp)


CN_PLACED = [(c, sp, orient) for c, k, sp, orient in ti.KIND_PLACED if k == CN]


@pytest.mark.parametrize("case,sp,orient", CN_PLACED, ids=[f"{c}-cn-axis{1 - o}" for c, _, o in CN_PLACED])
def test_instance_cn_call_sequence(case, sp, orient, monkeypatch):
    ti.set_env(monkeypatch, ti.CASE[case][1])
    assert ti.layout_of(sp, orient) == ti.want(case)
    assert_sequences(f"seq {case} {sid(sp)}", sp)


@pytest.mark.parametrize("sp", [(R2C, 64, CDN, 65), (C2C, 16, CD, 65)], ids=sid)
def test_call_sequence(sp, monkeypatch):
    ti.set_env(monkeypatch, {})
    assert_sequences(f"seq {sid(sp)}", sp)


def test_two_spaces_in_one_context(monkeypatch):
    """steps alternate between a 65- and a 4097-point lane space"""
    ti.set_env(monkeypatch, {})
    assert_sequences("two spaces", (CD, 65, CN, 65), (CD, 4097, CN, 65))


# ---- third derivatives ----
ALL_DERIVS = [(d0, d1) for d0 in range(4) for d1 in range(4)]


def assert_gradients(tag, sp, derivs):
    errs = {}
    for d in derivs:
        for scale in ((1.5, 1.0), None):
            errs[(d, scale)] = g.check_gradient_yardstick(*sp, d, scale)
    worst = max(errs.items(), key=lambda kv: kv[1][0])
    print(f"[call-contract] {tag}: worst err {worst[1][0]:.2e} at {worst[0]} (yardstick {worst[1][1]:.2e}), "
          f"largest yardstick {max(y for _, y in errs.values()):.2e}")
    bad = {k: v for k, v in errs.items() if not v[0] < max(g.TOL, 10.0 * v[1])}
    assert not bad, bad


@pytest.mark.parametrize("sp", SPACES[:7] + E16 + [(C2C, 16, CD, 65)], ids=IDS[:7] + E16_IDS + ["c2c16-cd65"])
def test_every_derivative_order(sp, monkeypatch):
    ti.set_env(monkeypatch, {})
    assert_gradients(f"deriv {sid(sp)}", sp, ALL_DERIVS)


@pytest.mark.parametrize("case,sp,orient", ti.PLACED, ids=ti.PLACED_IDS)
def test_instance_third_derivatives(case, sp, orient, monkeypatch):
    ti.set_env(monkeypatch, ti.CASE[case][1])
    assert ti.layout_of(sp, orient) == ti.want(case)
    assert_gradients(f"deriv3 {case} {sid(sp)}", sp, [(3, 0), (0, 3)])


# ---- solvers at the benchmarked coefficients ----
# C1: 129^2, Ra 1e5, dt 1e-2 (test_gpu_parity.test_navier_c1_100_steps); C2..C5: test_gpu_parity_large.CFG
BENCH = {"C1": (1e5, 1e-2), "C2": (1e7, 1e-3), "C4": (1e9, 1e-4), "C5": (1e10, 5e-5)}   # C3 steps at C2's Ra and dt
COEFFS = sorted({c for ra, dt in BENCH.values() for c in g.bench_coefficients(ra, dt)})
LANES = (1025, 2049, 4097, 8193)
SOLVER_SPACES = ([("hholtz_adi", (CD, n, CD, 65)) for n in LANES] + [("hholtz_adi", (CD, 65, CD, n)) for n in LANES]
                 + [("hholtz_adi", (CD, 65, CDN, n)) for n in LANES] + [("hholtz_adi", (R2C, n, CD, 65)) for n in (2048, 8192)]
                 + [(s, (CN, 65, CN, n)) for s in ("poisson", "hholtz") for n in LANES]
                 + [(s, (CN, 1025, CN, 65)) for s in ("poisson", "hholtz")])


@pytest.mark.parametrize("name,sp", SOLVER_SPACES, ids=[f"{s}-{sid(sp)}" for s, sp in SOLVER_SPACES])
def test_solver_at_benchmarked_coefficients(name, sp, monkeypatch):
    """every coefficient of C1..C5 (Poisson: its fixed (1, 1) on the same lanes); the per-row LU of Poisson / Hholtz runs
    along axis 1, axis 0 goes through the eigen-transform GEMM"""
    ti.set_env(monkeypatch, {})
    cs = [(1.0, 1.0)] if name == "poisson" else COEFFS
    errs = {c: g.check_solver_yardstick(name, *sp, c) for c in cs}
    for c, (e, y) in errs.items():
        print(f"[call-contract] {name} {sid(sp)} c=({c[0]:.2e}, {c[1]:.2e}): err {e:.2e}, yardstick {y:.2e}")
    bad = {c: v for c, v in errs.items() if not v[0] < max(g.TOL, 10.0 * v[1])}
    assert not bad, bad


# ---- Navier2D padding ----
def assert_navier_padding(tag, nav):
    p = g.check_navier_padding(nav)
    print(f"[call-contract] {tag}: worst padding_excess {max(p.values()):.2e}")
    assert max(p.values()) < PAD_TOL, p


@pytest.mark.parametrize("mode", [1, 0, 3, 5], ids=["fused", "unfused", "fused-nograph", "fused-nobranches"])
@pytest.mark.parametrize("periodic", [False, True])
def test_navier_padding_in_every_schedule(mode, periodic, monkeypatch):
    ti.set_env(monkeypatch, {})
    ng = g.b2.Navier2D(128 if periodic else 129, 129, 1e5, 1.0, 0.01, 1.0, "rbc", periodic=periodic)
    ng.set_mode(mode)
    ng.update(3)
    assert_navier_padding(f"navier mode {mode} periodic {periodic}", ng)


@pytest.mark.parametrize("mode", [1, 0, 3, 5], ids=["fused", "unfused", "fused-nograph", "fused-nobranches"])
@pytest.mark.parametrize("periodic", [False, True])
def test_navier_hc_padding_in_every_schedule(mode, periodic, monkeypatch):
    ti.set_env(monkeypatch, {})
    ng = g.b2.Navier2D(128 if periodic else 129, 129, 1e5, 1.0, 0.01, 1.0, "hc", periodic=periodic)
    ng.set_mode(mode)
    ng.update(3)
    assert_navier_padding(f"navier hc mode {mode} periodic {periodic}", ng)


@pytest.mark.parametrize("name", sorted(ti.STEPS))
def test_navier_padding_at_forced_layouts(name, monkeypatch):
    env, nx, ny, lays = ti.STEPS[name]
    ti.set_env(monkeypatch, env)
    for orient, w in lays.items():
        assert ti.layout_of((CD, nx, CD, ny), orient) == dict(zip(("E", "LN", "TPL", "fast"), w)), orient
    ng = g.b2.Navier2D(nx, ny, 1e5, 1.0, 0.01, 1.0, "rbc")
    ng.update(2)
    assert_navier_padding(f"navier {name}", ng)
