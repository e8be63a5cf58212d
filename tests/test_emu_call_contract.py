"""The operators as the time step and its callers use them, on the SIMT emulator of tests/emu (the CPU twin of
test_gpu_call_contract.py, on small spaces):

- call sequences on one space with every destination NaN-filled before the operator that writes it, outputs reused and all
  three solvers interleaved on the space's shared scratch; after every step the oracle at TOL and no stray value in the
  padding (the whole-array reductions norm2 / axpy / combine would see it);
- two spaces alternating step by step in one context;
- every derivative order (d0, d1) in 0..3, scaled and unscaled;
- HholtzAdi, Poisson and Hholtz at the Helmholtz coefficients of the benchmarked configurations (c ~ 1e-4 .. 1e-9),
  bounded by the oracle's own last-bit yardstick;
- the padding of a Navier2D's fields after steps in every schedule, and div_norm() against the host norm of div().

On the emulator the loads and OP_ZEROTAIL clear the lane buffer beyond the logical length, so the padding checks guard the
hardware paths (TMA box clipping, bulk copies of whole tiles) more than they find emulated defects; `-m gpu` runs them there."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
from tests import emu
emu.activate()
import numpy as np
from tests import gpu_checks as g

kind, arg = sys.argv[1], json.loads(sys.argv[2])
if kind == "seq":
    res = g.run_sequences(*[tuple(s) for s in arg])
    bad = g.sequence_failures(res)
    assert not bad, bad
elif kind == "deriv":
    for sp in arg:
        for d in [(d0, d1) for d0 in range(4) for d1 in range(4)]:
            for scale in ((1.5, 0.5), None):
                e = g.check_gradient(*sp, d, scale); assert e < g.TOL, (sp, d, scale, e)
elif kind == "solver":
    for name, sp, c in arg:
        e, yard = g.check_solver_yardstick(name, *sp, c)
        assert e < max(g.TOL, 10.0 * yard), (name, sp, c, e, yard)
elif kind == "navier":
    for nx, ny, periodic, mode, steps in arg:
        nav = g.b2.Navier2D(nx, ny, 1e5, 1.0, 0.01, 1.0, "rbc", periodic=periodic)
        nav.set_mode(mode)
        nav.update(steps)
        p = g.check_navier_padding(nav)
        assert max(p.values()) < 1e-13, (nx, ny, periodic, mode, p)
print("ok")
''' % ROOT

CD, CN, CDN, R2C, C2C, CH = 1, 2, 3, 4, 5, 0
SEQ = {
    "cd65-cn65": ({}, [(CD, 65, CN, 65)]),
    "r2c64-cd65": ({}, [(R2C, 64, CD, 65)]),
    "cn33-cd17": ({}, [(CN, 33, CD, 17)]),
    "cd17-cn33": ({}, [(CD, 17, CN, 33)]),
    "ch65-ch129": ({}, [(CH, 65, CH, 129)]),
    "cd100-cn65": ({}, [(CD, 100, CN, 65)]),          # dense transform (no FFT size)
    "r2c64-cdn65": ({}, [(R2C, 64, CDN, 65)]),
    "cn129-cdn33": ({}, [(CN, 129, CDN, 33)]),
    "c2c16-cd17": ({}, [(C2C, 16, CD, 17)]),
    "e16-cd257": ({"B2_E": "16"}, [(CD, 257, CN, 17)]),
    "nofast-cd1025": ({"B2_NOFAST": "1"}, [(CD, 1025, CN, 9)]),
    "two-spaces": ({}, [(CD, 33, CN, 17), (CD, 513, CN, 17)]),
}
DERIV = [(CD, 65, CN, 65), (R2C, 64, CD, 65), (CH, 33, CH, 65), (CN, 17, CDN, 33), (C2C, 16, CD, 17), (CD, 17, CD, 1025)]


def solver_jobs():
    """every benchmarked coefficient (C1..C5) on 1025-point lanes along either axis (E = 8 chunk maps), the other axis 9"""
    from tests import gpu_checks as g

    cs = sorted({c for ra, dt in ((1e5, 1e-2), (1e7, 1e-3), (1e9, 1e-4), (1e10, 5e-5)) for c in g.bench_coefficients(ra, dt)})
    jobs = []
    for c in cs:
        jobs += [["hholtz_adi", [CD, 1025, CD, 9], c], ["hholtz_adi", [CD, 9, CD, 1025], c], ["hholtz_adi", [CD, 9, CDN, 1025], c],
                 ["hholtz", [CN, 9, CN, 1025], c], ["poisson", [CN, 9, CN, 1025], [1.0, 1.0]]]
    return jobs


NAVIER = [[33, 33, False, m, 3] for m in (1, 0, 3, 5)] + [[32, 33, True, m, 3] for m in (1, 0)]


def run(kind, arg, env=None):
    r = subprocess.run([sys.executable, "-c", SCRIPT, kind, json.dumps(arg)], capture_output=True, text=True, timeout=900,
                       cwd=ROOT, env=dict({k: v for k, v in os.environ.items() if k not in ("B2_E", "B2_LN", "B2_NOFAST")}, **(env or {})))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("name", sorted(SEQ))
def test_emulated_call_sequence(name):
    env, spaces = SEQ[name]
    run("seq", spaces, env)


def test_emulated_third_derivatives():
    run("deriv", DERIV)


def test_emulated_solvers_at_benchmarked_coefficients():
    run("solver", solver_jobs())


def test_emulated_navier_padding():
    run("navier", NAVIER)
