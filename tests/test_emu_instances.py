"""The base-kind x instance matrix of test_gpu_instances.py on the SIMT emulator of tests/emu (its CPU twin, at the cases
whose lanes hold at most 257 points): ChebNeumann lanes on either axis, ChebDirichletNeumann lanes on axis 1 and r2c lanes
on axis 0 against the oracle (gpu_checks.op_errors), and the ChebNeumann stencil bit for bit
(gpu_checks.neumann_stencil_mismatches), with each case's layout switches and its layout asserted first.  This covers the
forced E = 16 / E = 4 / LN = 2 and the generic layouts; `-m gpu` runs every case on the hardware."""
import json
import os
import subprocess
import sys

import pytest

from tests import test_gpu_instances as ti

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
from tests import emu
emu.activate()
from tests import gpu_checks as g
import rustpde_mpi_b200 as b2

bad = {}
for what, sp, orient, want in json.loads(sys.argv[1]):
    s = b2.Space2((sp[0], sp[1]), (sp[2], sp[3]))
    lay = [s.layout(orient)[k] for k in ("E", "LN", "TPL", "fast")]
    s.close()
    assert lay == want, (sp, orient, lay, want)
    if what == "ops":
        errs, fail = g.op_errors(*sp, lane_axis=1 - orient)
    else:
        nbad, first = g.neumann_stencil_mismatches(*sp)
        fail = {"neumann": (nbad, first)} if nbad else {}
    if fail:
        bad[f"{what} {sp}"] = fail
assert not bad, bad
print("ok")
''' % ROOT

SMALL = [c for c in ti.CASE if ti.CASE[c][2][1] <= 257]


def jobs(case):
    """(what, space, orient, layout) of the case: its cn / cdn / r2c placements and the Neumann stencil spaces"""
    want = list(ti.CASE[case][3])
    if ti.CASE[case][2][0] == ti.R2C:
        return [["ops", list(sp), orient, want] for sp, orient in ti.placements(case)]
    out = [["ops", list(sp), orient, want] for c, k, sp, orient in ti.KIND_PLACED if c == case and k == ti.CN]
    out.append(["ops", list(ti.cdn_space(case)), 0, want])
    return out + [["neumann", list(sp), orient, want] for sp, orient in ti.neumann_spaces(case)]


@pytest.mark.parametrize("case", SMALL)
def test_emulated_kind_instance_matrix(case):
    r = subprocess.run([sys.executable, "-c", SCRIPT, json.dumps(jobs(case))], capture_output=True, text=True, timeout=1800,
                       cwd=ROOT, env=dict({k: v for k, v in os.environ.items() if k not in ti.SWITCHES}, **ti.CASE[case][1]))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
