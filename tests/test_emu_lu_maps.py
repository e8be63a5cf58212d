"""The banded LU solves of transform-sized lanes on the SIMT emulator of tests/emu, against the oracle to 1e-12: shared-vector
solves on their host-precomputed chunk maps (HholtzAdi, from_ortho; with the right-hand side's mat-vec folded in on E <= 8
lanes), and the per-lane solves of the Poisson per-row LU (Fourier and confined axis 0), on the E = 16 / 8 / 4 compile-time
layouts.  Every lane here ends in a partial chunk (2 (E + 1) TPL pairs cover more than the lane).

The skewed cases run the emulator's deterministic race schedule (B2_EMU_SKEW_US: after every block barrier the warps resume
one after another, milliseconds apart, lowest or highest first) on multi-warp layouts: (8,4,64) and the generic <8,4,0> on
1025-point lanes, 8 warps per lane group.  A shared-memory read after a barrier that nothing orders against another warp's
later write loses the race there every time -- e.g. the LU solve's back-substitution scan writing its warp totals over the
forward scan's entry states while a slower warp still reads them.  Says nothing about GPU results; `-m gpu` does that."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import sys
sys.path.insert(0, %r)
from tests import emu
emu.activate()
from tests import gpu_checks as g

TOL = 1e-12
FN = {"hholtz": g.check_hholtz, "from_ortho": g.check_from_ortho, "poisson": g.check_poisson, "forward": g.check_forward,
      "gradient": lambda *sp: max(g.check_gradient(*sp, d) for d in ((1, 0), (0, 1), (2, 0), (0, 2)))}
for arg in sys.argv[1:]:
    sp, names = arg.split(":")
    sp = tuple(int(v) for v in sp.split(","))
    for name in names.split(","):
        e = FN[name](*sp); assert e < TOL, (name, sp, e)
print("ok")
''' % ROOT

LU = "hholtz,from_ortho,poisson"
# B2_E caps the FFT points per thread: 257-point lanes run E = 16 (TPL = 8) under B2_E=16, 129-point lanes E = 8 (TPL = 8),
# and E = 4 (TPL = 16) under B2_E=4.
CASES = {
    "e16": ({"B2_E": "16"}, [f"1,257,2,129:{LU}", f"4,128,1,257:{LU}"]),
    "e8": ({}, [f"2,129,1,129:{LU}", f"4,64,2,129:{LU}"]),
    "e4": ({"B2_E": "4"}, [f"1,129,2,129:{LU}"]),
}
# Long lanes in one direction, 9 points (3 lane groups) in the other: HholtzAdi / from_ortho / derivatives / the forward
# transform along axis 0, and the Poisson per-row LU along axis 1.
SKEW_SPACES = ["1,1025,1,9:hholtz,from_ortho,gradient,forward", "2,9,2,1025:hholtz,from_ortho,poisson,gradient,forward"]
for geom, genv in (("fast", {}), ("nofast", {"B2_NOFAST": "1"})):
    for order in ("rev", "fwd"):
        CASES[f"skew-{geom}-{order}"] = (dict(genv, B2_EMU_SKEW_US=f"3000,{order}"), SKEW_SPACES)


@pytest.mark.parametrize("case", sorted(CASES))
def test_emulated_lu_solves(case):
    env, spaces = CASES[case]
    r = subprocess.run([sys.executable, "-c", SCRIPT, *spaces], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, **env))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
