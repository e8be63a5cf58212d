"""Edge cases of the Poisson eigen-transform GEMM (gemm_f64.cuh) on the SIMT emulator of tests/emu, against the oracle:
parity blocks whose row counts are not multiples of the 16-row MMA fragment, a last column block of a single tile (as at
4097 points), and the dense product (no parity structure) that runs as two 64-row halves.  Says nothing about GPU results;
`-m gpu` does that."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import sys
sys.path.insert(0, %r)
from tests import emu
emu.activate()
import rustpde_mpi_b200 as b2
from tests import gpu_checks as g

# 57 points: m0 = 55, parity blocks of 28 and 27 rows; 63 points: m0 = 61, the even block (31 rows) does not start on a
# tile row, so the product runs dense.  129 points on axis 1: 33 tile columns = one full column block of 32 tiles + one of 1.
for nx, blocks in ((57, 1), (63, 0)):
    info = b2.Navier2D(nx, 129, 1e5, 1.0, 0.01, 1.0, "rbc").info()
    assert info["parity_blocks"] == blocks and info["P1"] == 132, (nx, info)
for sp in [(2, 57, 2, 129), (1, 63, 1, 129)]:
    e = g.check_poisson(*sp); assert e < g.TOL, ("poisson", sp, e)
for sp in [(1, 57, 2, 129), (2, 63, 1, 129)]:
    e = g.check_hholtz_tensor(*sp); assert e < g.TOL, ("hholtz", sp, e)
print("ok")
''' % ROOT


def test_emulated_gemm_edges():
    r = subprocess.run([sys.executable, "-c", SCRIPT], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
