"""3 * 2^k and 5 * 2^k transform sizes (tests/test_gpu_mixed_radix.py) on the SIMT emulator of tests/emu: every layout of the
case table, the sizes that keep the dense transform or stay refused, the field operators and solvers of the cases whose lanes
hold at most 769 points against the oracle, one case per radix under the emulator's race schedule, and Navier2D steps on one
and on two ranks."""
import json
import os
import subprocess
import sys

import pytest

from tests import test_gpu_mixed_radix as mr
from tests.test_dist_gloo import run as run_ranks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH, CD, CN, CDN, R2C = 0, 1, 2, 3, 4
SMALL = [c for c in mr.CASE if mr.CASE[c][1][1] <= 769]
EMU_CROSS = 17


def emulated(code, env=None):
    """run ``code`` in a fresh process on the emulator build (the layout switches are read when a space is created)"""
    head = f"import sys\nsys.path.insert(0, {ROOT!r})\nfrom tests import emu\nemu.activate()\n"
    base = {k: v for k, v in os.environ.items() if k not in mr.SWITCHES}
    r = subprocess.run([sys.executable, "-c", head + code], capture_output=True, text=True, timeout=1800, cwd=ROOT,
                       env=dict(base, **(env or {})))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("case", list(mr.CASE))
def test_emulated_mixed_radix_layout(case):
    env, _, want = mr.CASE[case]
    emulated(f"from tests import test_gpu_mixed_radix as t\n"
             f"for sp, orient in t.jobs({case!r}, 9):\n"
             f"    lay = t.layout(sp, orient)\n"
             f"    assert lay == {tuple(want)!r}, (sp, orient, lay)\n"
             f"print('ok')\n", env)


def test_emulated_sizes_without_a_layout():
    """the short sizes of the two families keep the dense transform's layout; 3841 (= 15 * 256 + 1) is refused at its first
    transform, 10241 and 12289 when the space is created"""
    emulated("""
import rustpde_mpi_b200 as b2
from tests import gpu_checks as g
from tests import test_gpu_mixed_radix as t
CD, R2C = 1, 4
for sp, orient in [((CD, 9, CD, 97), 0), ((CD, 9, CD, 161), 0), ((R2C, 96, CD, 9), 1), ((R2C, 160, CD, 9), 1)]:
    assert t.layout(sp, orient) == (16, 4, 8, 0), sp
    assert max(g.check_forward(*sp), g.check_backward(*sp)) < g.TOL, sp
f = b2.Field2(b2.Space2((CD, 9), (CD, 3841)))
try:
    f.forward()
    raise SystemExit("3841 ran")
except b2.B2Error as e:
    assert str(e).startswith("b200pde error 3:"), e
for n in (10241, 12289):
    try:
        b2.Space2((CD, 9), (CD, n))
        raise SystemExit(f"{n} created")
    except b2.B2Error as e:
        assert str(e).startswith("b200pde error 3:") and "lane too long" in str(e), e
print("ok")
""")


@pytest.mark.parametrize("case", SMALL)
def test_emulated_mixed_radix_operators(case):
    mr.run_case(case, EMU_CROSS, "emu")


SOLVER_SPACES = [(CD, 17, CD, 193), (CN, 17, CD, 321), (R2C, 192, CD, 385), (CD, 193, CN, 161)]


@pytest.mark.parametrize("sp", SOLVER_SPACES)
def test_emulated_mixed_radix_solvers(sp):
    emulated(f"""
from tests import gpu_checks as g
sp = {sp!r}
errs = {{"poisson": g.check_poisson(*sp), "hholtz": g.check_hholtz_tensor(*sp), "hholtz_adi": g.check_hholtz(*sp)}}
assert max(errs.values()) < g.TOL, errs
print("ok")
""")


@pytest.mark.parametrize("sp", [(CD, 17, CD, 193), (R2C, 320, CD, 17)])
def test_emulated_mixed_radix_race_schedule(sp):
    """forward and backward under B2_EMU_SKEW_US (after every block barrier the warps resume in a skewed order): the odd pass
    adds a pass and its barriers to the FFT"""
    emulated(f"""
from tests import gpu_checks as g
sp = {sp!r}
errs = [g.check_forward(*sp), g.check_backward(*sp)]
assert max(errs) < g.TOL, errs
print("ok")
""", {"B2_EMU_SKEW_US": "2000,rev"})


@pytest.mark.parametrize("nx,ny,periodic,bc", [(97, 193, False, "rbc"), (192, 65, True, "rbc"), (65, 193, False, "hc")])
def test_emulated_mixed_radix_navier(nx, ny, periodic, bc):
    emulated(f"""
from tests import gpu_checks as g
errs = g.check_navier({nx}, {ny}, 1, periodic={periodic}, bc={bc!r}, same_tempbc={bc == "hc"})
assert max(errs.values()) < g.TOL, errs
print("ok")
""")


def test_emulated_mixed_radix_two_ranks():
    run_ranks(2, (65, 193, 1, 0, 1), 29631)
