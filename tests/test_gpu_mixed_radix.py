"""Transform sizes N = 3 * 2^k and 5 * 2^k (N = n - 1 for a Chebyshev lane, n for an r2c lane) on the lane FFT: the power-of-two
Stockham passes, then one radix-3 or radix-5 pass (lane_kernel.cuh, lane_fft).  They run on the generic instances
lane_kernel<E, LN, 0> with a thread count per lane that is not a power of two.

Every case forces its layout through the switches make_cfg reads at space creation (B2_E, B2_LN) and proves it with
Space2.layout() before it compares with the numpy oracle.  tests/test_emu_mixed_radix.py runs the short lanes of this table on
the emulator build."""
import os
import subprocess
import sys

import pytest

from tests import gpu_checks as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH, CD, CN, CDN, R2C = 0, 1, 2, 3, 4
SWITCHES = ("B2_E", "B2_LN", "B2_NOFAST")

# (id, environment, lane base (kind, n), expected (E, LN, TPL, fast)): the natural layouts at every size of the two families that
# has one, then forced layouts, so that every generic (E, LN) pair runs a radix-3 and a radix-5 lane
CASES = [
    ("r3-193", {}, (CD, 193), (4, 4, 24, 0)),
    ("r3-385", {}, (CD, 385), (8, 4, 24, 0)),
    ("r3-769", {}, (CD, 769), (8, 4, 48, 0)),
    ("r3-1537", {}, (CD, 1537), (8, 4, 96, 0)),
    ("r3-3073", {}, (CD, 3073), (16, 4, 96, 0)),
    ("r3-6145", {}, (CD, 6145), (16, 2, 192, 0)),
    ("r5-321", {}, (CD, 321), (4, 4, 40, 0)),
    ("r5-641", {}, (CD, 641), (8, 4, 40, 0)),
    ("r5-1281", {}, (CD, 1281), (8, 4, 80, 0)),
    ("r5-2561", {}, (CD, 2561), (16, 4, 80, 0)),
    ("r5-5121", {}, (CD, 5121), (16, 2, 160, 0)),
    ("r3-192-r2c", {}, (R2C, 192), (4, 4, 24, 0)),
    ("r3-768-r2c", {}, (R2C, 768), (8, 4, 48, 0)),
    ("r3-3072-r2c", {}, (R2C, 3072), (16, 4, 96, 0)),
    ("r3-6144-r2c", {}, (R2C, 6144), (16, 2, 192, 0)),
    ("r5-320-r2c", {}, (R2C, 320), (4, 4, 40, 0)),
    ("r5-1280-r2c", {}, (R2C, 1280), (8, 4, 80, 0)),
    ("r5-5120-r2c", {}, (R2C, 5120), (16, 2, 160, 0)),
    ("r3-e16-769", {"B2_E": "16"}, (CD, 769), (16, 4, 24, 0)),
    ("r3-ln2-769", {"B2_LN": "2"}, (CD, 769), (8, 2, 48, 0)),
    ("r3-e16-ln2-1537", {"B2_E": "16", "B2_LN": "2"}, (CD, 1537), (16, 2, 48, 0)),
    ("r3-e4-ln2-385", {"B2_E": "4", "B2_LN": "2"}, (CD, 385), (4, 2, 48, 0)),
    ("r5-e16-1281", {"B2_E": "16"}, (CD, 1281), (16, 4, 40, 0)),
    ("r5-ln2-1281", {"B2_LN": "2"}, (CD, 1281), (8, 2, 80, 0)),
    ("r5-e16-ln2-2561", {"B2_E": "16", "B2_LN": "2"}, (CD, 2561), (16, 2, 80, 0)),
    ("r5-e4-ln2-641", {"B2_E": "4", "B2_LN": "2"}, (CD, 641), (4, 2, 80, 0)),
    ("r3-e16-768-r2c", {"B2_E": "16"}, (R2C, 768), (16, 4, 24, 0)),
    ("r5-e4-ln2-640-r2c", {"B2_LN": "2"}, (R2C, 640), (4, 2, 80, 0)),
]
CASE = {c[0]: c[1:] for c in CASES}
CROSS = 65   # the other axis: short, so that the oracle stays fast at the longest lanes


def jobs(case, cross=CROSS):
    """(space, orient) of the case's lane: an r2c lane on axis 0; a Chebyshev lane as ch, cd and cn on either axis and as cdn on
    axis 1 (orient 0 = lanes along axis 1)"""
    _, (k, n), _ = CASE[case]
    if k == R2C:
        return [((R2C, n, CD, cross), 1)]
    out = []
    for kind in (CH, CD, CN):
        out.append(((CN if kind != CH else CH, cross, kind, n), 0))
        out.append(((kind, n, CD if kind != CH else CH, cross), 1))
    out.append(((CN, cross, CDN, n), 0))
    return out


def layout(sp, orient):
    import rustpde_mpi_b200 as b2

    s = b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))
    lay = tuple(s.layout(orient)[k] for k in ("E", "LN", "TPL", "fast"))
    s.close()
    return lay


# every case in a process of its own: the layout switches are read when a space is created
SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
if sys.argv[2] == "emu":
    from tests import emu
    emu.activate()
from tests import gpu_checks as g
from tests import test_gpu_mixed_radix as t
case, cross = json.loads(sys.argv[1])
want = tuple(t.CASE[case][2])
bad = {}
for sp, orient in t.jobs(case, cross):
    lay = t.layout(sp, orient)
    assert lay == want, (sp, orient, lay, want)
    errs, fail = g.op_errors(*sp, lane_axis=1 - orient)
    if fail:
        bad[str(sp)] = fail
assert not bad, bad
print("ok")
''' % ROOT


def run_case(case, cross, where):
    import json

    env = dict({k: v for k, v in os.environ.items() if k not in SWITCHES}, **CASE[case][0])
    r = subprocess.run([sys.executable, "-c", SCRIPT, json.dumps([case, cross]), where], capture_output=True, text=True,
                       timeout=3600, cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASE))
def test_mixed_radix_operators(case):
    """forward, backward, to_ortho, from_ortho, gradients and HholtzAdi at 1e-10, the third derivative along the lane at
    max(1e-10, 10 x yardstick), on every placement of the case's lane"""
    run_case(case, CROSS, "gpu")


@pytest.mark.gpu
@pytest.mark.parametrize("sp", [(CD, 65, CD, 769), (CN, 65, CD, 1281), (R2C, 384, CD, 385), (CD, 641, CN, 193)])
def test_mixed_radix_solvers(sp):
    """Poisson and Hholtz (eigendecomposition form) with a new-size lane on axis 1, HholtzAdi on both"""
    errs = {"poisson": g.check_poisson(*sp), "hholtz": g.check_hholtz_tensor(*sp), "hholtz_adi": g.check_hholtz(*sp)}
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.gpu
@pytest.mark.parametrize("nx,ny,periodic", [(1537, 1537, False), (3073, 3073, False), (3072, 1537, True)])
def test_mixed_radix_navier_steps(nx, ny, periodic):
    """2 steps on a smooth state at 1e-10, and from white noise under the yardstick rule; padding clean after the steps"""
    errs = g.check_navier(nx, ny, 2, periodic)
    assert max(errs.values()) < g.TOL, errs
    errs, yard = g.check_navier_white_noise(nx, ny, 2, periodic)
    assert max(errs.values()) < max(g.TOL, 10.0 * yard), (errs, yard)
    import rustpde_mpi_b200 as b2

    nav = b2.Navier2D(nx, ny, 1e5, 1.0, 0.01, 1.0, periodic=periodic)
    nav.update(1)
    pad = g.check_navier_padding(nav)
    assert max(pad.values()) < 1e-13, pad


@pytest.mark.gpu
def test_mixed_radix_navier_hc():
    errs = g.check_navier(769, 769, 2, bc="hc", same_tempbc=True)
    assert max(errs.values()) < g.TOL, errs


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASE if CASE[c][1][1] <= 2561])
def test_mixed_radix_call_sequence(case):
    """the call sequences of gpu_checks (reused outputs, NaN-filled destinations, padding) at one space per layout"""
    env_before = {k: os.environ.get(k) for k in SWITCHES}
    os.environ.update(CASE[case][0])
    try:
        sp, orient = jobs(case)[0]
        assert layout(sp, orient) == tuple(CASE[case][2])
        bad = g.sequence_failures(g.run_sequences(sp))
    finally:
        for k, v in env_before.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    assert not bad, bad


@pytest.mark.gpu
def test_mixed_radix_alternates_with_power_of_two():
    """a 3073-point space and a 4097-point space (compile-time instance) in one context, step by step"""
    bad = g.sequence_failures(g.run_sequences((CN, 65, CD, 3073), (CN, 65, CD, 4097)))
    assert not bad, bad


@pytest.mark.gpu
def test_mixed_radix_full_size_properties():
    import rustpde_mpi_b200 as b2

    from tests import golden_checks as gc

    errs = {}
    for sp in ((CH, 6145, CH, 6145), (R2C, 6144, CH, 3073)):
        errs.update({f"{sp} {k}": v for k, v in gc.check_roundtrip_and_linearity(b2, sp).items()})
    errs.update({f"hholtz {k}": v for k, v in gc.check_hholtz_linearity(b2, (CD, 5121, CD, 5121)).items()})
    assert max(errs.values()) < gc.TOL, errs
