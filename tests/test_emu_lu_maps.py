"""The banded LU solves of transform-sized lanes on the SIMT emulator of tests/emu, against the oracle to 1e-12: shared-vector
solves on their host-precomputed chunk maps (HholtzAdi, from_ortho; with the right-hand side's mat-vec folded in on E <= 8
lanes), and the per-lane solves of the Poisson per-row LU (Fourier and confined axis 0), on the E = 16 / 8 / 4 compile-time
layouts.  Every lane here ends in a partial chunk (2 (E + 1) TPL pairs cover more than the lane).  Says nothing about GPU
results; `-m gpu` does that."""
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
spaces = [tuple(int(v) for v in s.split(",")) for s in sys.argv[1:]]
for sp in spaces:
    for fn in (g.check_hholtz, g.check_from_ortho, g.check_poisson):
        e = fn(*sp); assert e < TOL, (fn.__name__, sp, e)
print("ok")
''' % ROOT

# B2_E caps the FFT points per thread: 257-point lanes run E = 16 (TPL = 8) under B2_E=16, 129-point lanes E = 8 (TPL = 8),
# and E = 4 (TPL = 16) under B2_E=4.
CASES = {
    "e16": ({"B2_E": "16"}, ["1,257,2,129", "4,128,1,257"]),
    "e8": ({}, ["2,129,1,129", "4,64,2,129"]),
    "e4": ({"B2_E": "4"}, ["1,129,2,129"]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_emulated_lu_solves(case):
    env, spaces = CASES[case]
    r = subprocess.run([sys.executable, "-c", SCRIPT, *spaces], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, **env))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
