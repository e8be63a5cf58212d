"""Every lane-kernel instance launch_pass dispatches to, against the numpy oracle on the GPU.

launch_pass (rustpde_mpi_b200/csrc/b200pde.cu) runs 14 compile-time-geometry instances lane_kernel<E, LN, TPL> (B2_INST) and
one generic instance lane_kernel<E, LN, 0> per (E, LN).  make_cfg picks the layout from the lane's transform size and padded
pitch, and production reaches layouts the natural test sizes do not (the pitch grows with the rank count), so each instance is
forced here on one GPU through the layout switches make_cfg reads at space creation (B2_E, B2_LN, B2_NOFAST), and every case
proves with Space2.layout() that it reached its instance before comparing with the oracle.

CPU (no GPU): every case's layout on the emulator build, and the case table against the B2_INST list of launch_pass, so
an instance added later without a case fails here.  GPU (-m gpu): field ops, derivatives and the solvers at every case,
whole Navier2D steps at forced layouts, the non-default step schedules, and the static load / store path switches."""
import json
import os
import re
import subprocess
import sys

import pytest

from tests import gpu_checks as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH, CD, CN, CDN, R2C = 0, 1, 2, 3, 4
SWITCHES = ("B2_E", "B2_LN", "B2_NOFAST")

# (id, environment, lane base (kind, n), expected (E, LN, TPL, fast))
CASES = [
    ("f4-4-8", {}, (CD, 65), (4, 4, 8, 1)),
    ("f4-4-8-r2c", {}, (R2C, 64), (4, 4, 8, 1)),
    ("f8-4-8", {}, (CD, 129), (8, 4, 8, 1)),
    ("f8-4-16", {}, (CD, 257), (8, 4, 16, 1)),
    ("f8-4-32", {}, (CD, 513), (8, 4, 32, 1)),
    ("f8-4-64", {}, (CD, 1025), (8, 4, 64, 1)),
    ("f16-4-64", {}, (CD, 2049), (16, 4, 64, 1)),
    ("f16-4-64-r2c", {}, (R2C, 2048), (16, 4, 64, 1)),
    ("f16-4-128", {}, (CD, 4097), (16, 4, 128, 1)),
    ("f16-2-256", {}, (CD, 8193), (16, 2, 256, 1)),
    ("f16-2-256-r2c", {}, (R2C, 8192), (16, 2, 256, 1)),
    ("f16-4-8", {"B2_E": "16"}, (CD, 257), (16, 4, 8, 1)),
    ("f16-4-16", {"B2_E": "16"}, (CD, 513), (16, 4, 16, 1)),
    ("f16-4-32", {"B2_E": "16"}, (CD, 1025), (16, 4, 32, 1)),
    ("f4-4-16", {"B2_E": "4"}, (CD, 129), (4, 4, 16, 1)),
    ("f4-4-32", {"B2_E": "4"}, (CD, 257), (4, 4, 32, 1)),
    ("f16-2-128", {"B2_LN": "2"}, (CD, 4097), (16, 2, 128, 1)),
    ("g16-4-cd100", {}, (CD, 100), (16, 4, 8, 0)),
    ("g16-4-nofast", {"B2_NOFAST": "1"}, (CD, 4097), (16, 4, 128, 0)),
    ("g8-4", {"B2_NOFAST": "1"}, (CD, 1025), (8, 4, 64, 0)),
    ("g4-4", {"B2_NOFAST": "1"}, (CD, 65), (4, 4, 8, 0)),
    ("g16-2", {"B2_LN": "2", "B2_NOFAST": "1"}, (CD, 4097), (16, 2, 128, 0)),
    ("g8-2", {"B2_LN": "2"}, (CD, 257), (8, 2, 16, 0)),
    ("g4-2", {"B2_LN": "2", "B2_E": "4"}, (CD, 129), (4, 2, 16, 0)),
    # rfft_fast at every (E, TPL) an r2c lane reaches, and the generic instance's FFT
    ("f8-4-8-r2c", {}, (R2C, 128), (8, 4, 8, 1)),
    ("f8-4-16-r2c", {}, (R2C, 256), (8, 4, 16, 1)),
    ("f8-4-32-r2c", {}, (R2C, 512), (8, 4, 32, 1)),
    ("f8-4-64-r2c", {}, (R2C, 1024), (8, 4, 64, 1)),
    ("f16-4-128-r2c", {}, (R2C, 4096), (16, 4, 128, 1)),
    ("f16-4-8-r2c", {"B2_E": "16"}, (R2C, 256), (16, 4, 8, 1)),
    ("f16-4-16-r2c", {"B2_E": "16"}, (R2C, 512), (16, 4, 16, 1)),
    ("f16-4-32-r2c", {"B2_E": "16"}, (R2C, 1024), (16, 4, 32, 1)),
    ("f4-4-16-r2c", {"B2_E": "4"}, (R2C, 128), (4, 4, 16, 1)),
    ("f4-4-32-r2c", {"B2_E": "4"}, (R2C, 256), (4, 4, 32, 1)),
    ("f16-2-128-r2c", {"B2_LN": "2"}, (R2C, 4096), (16, 2, 128, 1)),
    ("g8-4-r2c", {"B2_NOFAST": "1"}, (R2C, 1024), (8, 4, 64, 0)),
]
CASE = {c[0]: c for c in CASES}


def placements(case, kind=None):
    """(space, orient) of the case's lane on axis 0 (other axis cn 65) and, for Chebyshev lanes, on axis 1 (other axis cd 65);
    ``kind`` replaces the case's lane base kind (same length, so the same layout)"""
    _, _, (k, n), _ = CASE[case]
    kind = k if kind is None else kind
    out = [((kind, n, CN, 65), 1)]
    if kind != R2C:
        out.append(((CD, 65, kind, n), 0))
    return out


AXIS1 = [c for c in CASE if CASE[c][2][0] != R2C]   # cases whose lane can lie on axis 1 (a Chebyshev axis)
CDN_CASES = AXIS1
# ChebNeumann (BC_STEN_N / BC_S2_N families, LD_NEUMANN stencil-on-load) and orthonormal Chebyshev lanes at every Chebyshev case
KIND_PLACED = [(c, k, sp, orient) for c in AXIS1 for k in (CN, CH) for sp, orient in placements(c, k)]


def neumann_spaces(case):
    """(space, orient): a ChebNeumann lane of the case's length next to an orthonormal Chebyshev axis of 65 (to_ortho is the
    identity there), on axis 1 and on axis 0"""
    n = CASE[case][2][1]
    return [((CH, 65, CN, n), 0), ((CN, n, CH, 65), 1)]


# every (lane kind, layout) the GPU tests above place a lane at: each Chebyshev kind at every instance of launch_pass (the
# generic ones at the TPL of their cases), r2c at every layout an FFT-sized r2c lane reaches
GENERIC_LAYOUTS = {(16, 4, 8, 0), (16, 4, 128, 0), (8, 4, 64, 0), (4, 4, 8, 0), (16, 2, 128, 0), (8, 2, 16, 0), (4, 2, 16, 0)}
R2C_LAYOUTS = {(4, 4, 8, 1), (8, 4, 8, 1), (8, 4, 16, 1), (8, 4, 32, 1), (8, 4, 64, 1), (16, 4, 64, 1), (16, 4, 128, 1),
               (16, 2, 256, 1), (16, 4, 8, 1), (16, 4, 16, 1), (16, 4, 32, 1), (4, 4, 16, 1), (4, 4, 32, 1), (16, 2, 128, 1),
               (8, 4, 64, 0)}


def per_row_lu_spaces(case):
    """Poisson and Hholtz spaces with the case's lane on axis 1 (the per-row LU) and a 65-point GEMM axis"""
    n = CASE[case][2][1]
    return [(CN, 65, CN, n), (CD, 65, CD, n)]


def cdn_space(case):
    return (CN, 65, CDN, CASE[case][2][1])


# whole steps at forced layouts: (environment, nx, ny, {orient: expected (E, LN, TPL, fast)})
STEPS = {
    "e16-257": ({"B2_E": "16"}, 257, 257, {0: (16, 4, 8, 1), 1: (16, 4, 8, 1)}),
    "e4-257": ({"B2_E": "4"}, 257, 257, {0: (4, 4, 32, 1), 1: (4, 4, 32, 1)}),
    "ln2-257": ({"B2_LN": "2"}, 257, 257, {0: (8, 2, 16, 0), 1: (8, 2, 16, 0)}),
    "ln2e4-129": ({"B2_LN": "2", "B2_E": "4"}, 129, 129, {0: (4, 2, 16, 0), 1: (4, 2, 16, 0)}),
    "nofast-1025x129": ({"B2_NOFAST": "1"}, 1025, 129, {0: (8, 4, 8, 0), 1: (8, 4, 64, 0)}),
}


HC_C2_LAYOUT = (8, 4, 64, 1)   # the 1025-point lanes along axis 1 of the 1025^2 hc case


def want(case):
    return dict(zip(("E", "LN", "TPL", "fast"), CASE[case][3]))


def set_env(monkeypatch, env):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def layout_of(sp, orient):
    import rustpde_mpi_b200 as b2

    s = b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))
    lay = s.layout(orient)
    s.close()
    return {k: lay[k] for k in ("E", "LN", "TPL", "fast")}


# ------------------------------------------------------------------------------------------------------------------------------
# CPU: the table
# ------------------------------------------------------------------------------------------------------------------------------
LAYOUT_SCRIPT = r'''
import json, os, sys
sys.path.insert(0, %r)
from tests import emu
emu.activate()
import rustpde_mpi_b200 as b2
out = {}
for key, env, sp, orient in json.loads(sys.argv[1]):
    for k in %r:
        os.environ.pop(k, None)
    os.environ.update(env)
    s = b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))
    out[key] = s.layout(orient)
    s.close()
print(json.dumps(out))
'''


def layout_jobs():
    """(key, environment, space, orient, expected (E, LN, TPL, fast)) of every space the GPU tests below assert a layout of"""
    jobs = []
    for c in CASE:
        env, exp = CASE[c][1], list(CASE[c][3])
        jobs += [[f"{c}@{sp}", env, list(sp), orient, exp] for sp, orient in placements(c)]
        if c in AXIS1:
            jobs += [[f"{c}@{sp}", env, list(sp), 0, exp] for sp in per_row_lu_spaces(c)]
        if c in CDN_CASES:
            jobs.append([f"{c}@{cdn_space(c)}", env, list(cdn_space(c)), 0, exp])
        if c in AXIS1:
            jobs += [[f"{c}@{sp}", env, list(sp), orient, exp] for sp, orient in neumann_spaces(c)]
    jobs += [[f"{c}@{sp}", CASE[c][1], list(sp), orient, list(CASE[c][3])] for c, _, sp, orient in KIND_PLACED]
    for name, (env, nx, ny, lays) in STEPS.items():
        jobs += [[f"{name}@{orient}", env, [CD, nx, CD, ny], orient, list(w)] for orient, w in lays.items()]
    jobs.append(["hc-1025@0", {}, [CD, 1025, CD, 1025], 0, list(HC_C2_LAYOUT)])
    from tests.test_gpu_zz_any_size import SIZE_LAYOUTS
    for (nx, ny, _), lay in SIZE_LAYOUTS.items():
        jobs.append([f"size-{nx}x{ny}@1", {}, [CD, nx, CD, ny], 1, [lay[k] for k in ("E", "LN", "TPL", "fast")]])
    return jobs


def test_case_table_layouts_on_the_emulator():
    """every case reaches its (E, LN, TPL, fast) in every space a GPU test uses it in (make_cfg is host code: the emulator build
    runs it)"""
    jobs = layout_jobs()
    r = subprocess.run([sys.executable, "-c", LAYOUT_SCRIPT % (ROOT, SWITCHES), json.dumps([j[:4] for j in jobs])],
                       capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env={k: v for k, v in os.environ.items() if k not in SWITCHES})
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    bad = {}
    for key, _, _, _, exp in jobs:
        lay = [got[key][k] for k in ("E", "LN", "TPL", "fast")]
        if lay != exp:
            bad[key] = (lay, exp)
        assert got[key]["NT"] == got[key]["LN"] * got[key]["TPL"], key
    assert not bad, bad


def test_case_table_covers_every_instance_of_launch_pass():
    src = open(os.path.join(ROOT, "rustpde_mpi_b200", "csrc", "b200pde.cu")).read()
    body = src[src.index("static int launch_pass("):]
    body = body[:body.index("\n}\n")]
    fast = {tuple(int(v) for v in m) for m in re.findall(r"B2_INST\((\d+),\s*(\d+),\s*(\d+)\)", body)}
    generic = {tuple(int(v) for v in m) for m in re.findall(r"launch_ELT<(\d+),\s*(\d+),\s*0>", body)}
    assert len(fast) == 14 and len(generic) == 6, (fast, generic)
    assert {c[3][:3] for c in CASES if c[3][3]} == fast
    assert {c[3][:2] for c in CASES if not c[3][3]} == generic


def test_every_kind_reaches_every_instance():
    """the (lane kind, layout) pairs the GPU ops tests place: cd, cn, ch and cdn at all 14 compile-time instances and at the
    generic instances' layouts, r2c at every layout it reaches; a case row removed from the table fails here"""
    src = open(os.path.join(ROOT, "rustpde_mpi_b200", "csrc", "b200pde.cu")).read()
    body = src[src.index("static int launch_pass("):]
    body = body[:body.index("\n}\n")]
    fast = {tuple(int(v) for v in m) + (1,) for m in re.findall(r"B2_INST\((\d+),\s*(\d+),\s*(\d+)\)", body)}
    assert {lay[:2] for lay in GENERIC_LAYOUTS} == {tuple(int(v) for v in m) for m in re.findall(r"launch_ELT<(\d+),\s*(\d+),\s*0>", body)}
    claimed = {(k, lay) for k in (CD, CN, CH, CDN) for lay in fast | GENERIC_LAYOUTS} | {(R2C, lay) for lay in R2C_LAYOUTS}
    placed = {(CASE[c][2][0], CASE[c][3]) for c, _, _ in PLACED} | {(k, CASE[c][3]) for c, k, _, _ in KIND_PLACED}
    placed |= {(CDN, CASE[c][3]) for c in CDN_CASES}
    missing = sorted((g.KIND_NAME[k], lay) for k, lay in claimed - placed)
    assert not missing, missing
    neumann = {CASE[c][3] for c in AXIS1}
    assert neumann == fast | GENERIC_LAYOUTS, sorted((fast | GENERIC_LAYOUTS) - neumann)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------------
FIELD_OPS = ("forward", "backward", "to_ortho", "from_ortho")
DERIVS = ((1, 0), (0, 1), (2, 0), (0, 2))
PLACED = [(c, sp, orient) for c in CASE for sp, orient in placements(c)]
PLACED_IDS = [f"{c}-axis{1 - orient}" for c, _, orient in PLACED]


@pytest.mark.gpu
@pytest.mark.parametrize("case,sp,orient", PLACED, ids=PLACED_IDS)
def test_instance_ops_against_oracle(case, sp, orient, monkeypatch):
    """transforms, ortho conversions, derivatives and HholtzAdi with the forced lane on axis 0 or axis 1"""
    set_env(monkeypatch, CASE[case][1])
    assert layout_of(sp, orient) == want(case)
    errs = {op: getattr(g, "check_" + op)(*sp) for op in FIELD_OPS}
    errs.update({f"gradient{d}": g.check_gradient(*sp, d) for d in DERIVS})
    errs["hholtz_adi"] = g.check_hholtz(*sp)
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.gpu
@pytest.mark.parametrize("case", AXIS1)
def test_instance_per_row_lu_against_oracle(case, monkeypatch):
    """Poisson and Hholtz with the forced lane on axis 1: the per-row LU of the eigen-transformed system (GEMM axis 65)"""
    set_env(monkeypatch, CASE[case][1])
    errs = {}
    for name, sp in zip(("poisson", "hholtz_tensor"), per_row_lu_spaces(case)):
        assert layout_of(sp, 0) == want(case), name
        errs[name] = getattr(g, "check_" + name)(*sp)
    assert max(errs.values()) < g.TOL, errs


def report(tag, errs):
    worst = max(errs, key=errs.get)
    print(f"[instances] {tag}: worst err {errs[worst]:.2e} ({worst})")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CDN_CASES)
def test_instance_cdn_ops_against_oracle(case, monkeypatch):
    """ChebDirichletNeumann lanes (OP_STEN3, OP_PDMA in HholtzAdi) on axis 1 at every Chebyshev case"""
    set_env(monkeypatch, CASE[case][1])
    sp = cdn_space(case)
    assert layout_of(sp, 0) == want(case)
    errs, bad = g.op_errors(*sp, lane_axis=1)
    report(f"{case} cdn {sp}", errs)
    assert not bad, bad


KIND_IDS = [f"{c}-{g.KIND_NAME[k]}-axis{1 - orient}" for c, k, _, orient in KIND_PLACED]


@pytest.mark.gpu
@pytest.mark.parametrize("case,kind,sp,orient", KIND_PLACED, ids=KIND_IDS)
def test_instance_kind_ops_against_oracle(case, kind, sp, orient, monkeypatch):
    """ChebNeumann and orthonormal Chebyshev lanes of the case's length on axis 0 or axis 1"""
    set_env(monkeypatch, CASE[case][1])
    assert layout_of(sp, orient) == want(case)
    errs, bad = g.op_errors(*sp, lane_axis=1 - orient)
    report(f"{case} {g.KIND_NAME[kind]} {sp}", errs)
    assert not bad, bad


NEUMANN_PLACED = [(c, sp, orient) for c in AXIS1 for sp, orient in neumann_spaces(c)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,sp,orient", NEUMANN_PLACED, ids=[f"{c}-axis{1 - o}" for c, _, o in NEUMANN_PLACED])
def test_instance_neumann_stencil_bit_for_bit(case, sp, orient, monkeypatch):
    """the ChebNeumann stencil the lane kernel forms (BC_STEN_N on the compile-time instances, LD_NEUMANN stencil-on-load on
    the generic ones) equals the host's s_k = -(k / (k + 2))^2 in every bit"""
    set_env(monkeypatch, CASE[case][1])
    assert layout_of(sp, orient) == want(case)
    nbad, first = g.neumann_stencil_mismatches(*sp)
    assert nbad == 0, (nbad, first)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STEPS))
def test_navier_steps_at_forced_layouts(name, monkeypatch):
    env, nx, ny, lays = STEPS[name]
    set_env(monkeypatch, env)
    for orient, w in lays.items():
        assert layout_of((CD, nx, CD, ny), orient) == dict(zip(("E", "LN", "TPL", "fast"), w)), orient
    errs = g.check_navier(nx, ny, 2)
    assert max(errs.values()) < g.TOL, errs
    errs, yard = g.check_navier_white_noise(nx, ny, 2)
    tol = max(g.TOL, 10.0 * yard)
    assert max(errs.values()) < tol, (errs, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 3, 5], ids=["unfused", "fused-nograph", "fused-nobranches"])
@pytest.mark.parametrize("periodic", [False, True])
def test_navier_schedules(mode, periodic):
    """mode 0: one pass pair per reference call (the cross-check implementation); 3: fused without graph replay; 5: fused
    without parallel branches"""
    errs = g.check_navier(128 if periodic else 129, 129, 3, periodic, mode=mode)
    assert max(errs.values()) < g.TOL, errs


# bc = "hc": the temperature's axis 1 is ChebDirichletNeumann (OP_STEN3, OP_PDMA) in every step.  Its boundary field tempbc
# varies along x, and each side builds it with its own grid, cos and transforms: the coefficients differ by a transform's
# round-off, which dt ka d2/dx2 tempbc multiplies by ~k^4 in the high modes (gpu_checks.share_tempbc).  Two steps at 1025 x 129
# on the emulator build: temp differs from the oracle by 5.9e-10 when each side builds its own tempbc and by 1.0e-14 when the
# oracle takes the library's; rbc (tempbc constant along x) agrees to 2.1e-14 there.  So the step itself is checked with one
# tempbc on both sides at TOL, and the run with each side's own tempbc against the oracle's change under tempbc round-off.
def assert_hc_steps(tag, nx, ny, ra=1e5, dt=0.01, white_noise=True):
    same = g.check_navier(nx, ny, 2, ra=ra, dt=dt, bc="hc", same_tempbc=True)
    own, yard_bc = g.check_navier_tempbc_yardstick(nx, ny, 2, ra=ra, dt=dt)
    msg = f"[instances] hc {tag}: same tempbc {max(same.values()):.2e}, own tempbc {own} (tempbc yardstick {yard_bc:.2e})"
    if white_noise:
        noise, yard = g.check_navier_white_noise(nx, ny, 2, bc="hc", same_tempbc=True)
        msg += f", white noise {max(noise.values()):.2e} (yardstick {yard:.2e})"
    print(msg)
    assert max(same.values()) < g.TOL, same
    assert max(own["velx"], own["vely"], own["pres"]) < g.TOL, own
    assert own["temp"] < max(g.TOL, 10.0 * yard_bc), (own, yard_bc)
    if white_noise:
        assert max(noise.values()) < max(g.TOL, 10.0 * yard), (noise, yard)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STEPS))
def test_navier_hc_steps_at_forced_layouts(name, monkeypatch):
    env, nx, ny, lays = STEPS[name]
    set_env(monkeypatch, env)
    for orient, w in lays.items():
        assert layout_of((CD, nx, CD, ny), orient) == dict(zip(("E", "LN", "TPL", "fast"), w)), orient
    assert_hc_steps(name, nx, ny)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 3, 5], ids=["unfused", "fused-nograph", "fused-nobranches"])
@pytest.mark.parametrize("periodic", [False, True])
def test_navier_hc_schedules(mode, periodic):
    errs = g.check_navier(128 if periodic else 129, 129, 3, periodic, mode=mode, bc="hc")
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.gpu
def test_navier_hc_at_c2_lane_length(monkeypatch):
    """1025^2 confined (the lane length and Ra, dt of C2), two steps"""
    set_env(monkeypatch, {})
    assert layout_of((CD, 1025, CD, 1025), 0) == dict(zip(("E", "LN", "TPL", "fast"), HC_C2_LAYOUT))
    assert_hc_steps("1025^2", 1025, 1025, ra=1e7, dt=1e-3, white_noise=False)


SWITCH_SCRIPT = r'''
import sys
sys.path.insert(0, %r)
from tests import gpu_checks as g
e = g.check_navier(129, 129, 2); assert max(e.values()) < g.TOL, e
e = g.check_navier(257, 257, 3, False, 1e7, 1e-3, "random"); assert max(e.values()) < g.TOL, e   # test_navier_random_init_257
for op in ("forward", "backward", "to_ortho", "from_ortho"):
    e = getattr(g, "check_" + op)(1, 1025, 2, 65); assert e < g.TOL, (op, e)
print("ok")
''' % ROOT


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"B2_NOTMA": "1"}, {"B2_LDTHREADS": "1", "B2_CHW": "3"}], ids=["notma", "ldthreads-chw3"])
def test_static_path_switches(env):
    """B2_NOTMA (every load / store on the per-thread path) and B2_LDTHREADS (combining loads per thread) are read once per
    process: each runs in a process of its own (killed on timeout)"""
    r = subprocess.run([sys.executable, "-c", SWITCH_SCRIPT], capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict({k: v for k, v in os.environ.items() if k not in SWITCHES}, **env))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
