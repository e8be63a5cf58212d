"""Which form every lane operator takes on each lane-kernel layout, pinned on the SIMT emulator of tests/emu.

The emulator tests elsewhere check numerics, but a banded mat-vec or solve that misses its fast form (chunk-streaming OP_BANDC,
the mat-vec folded into the LU solve, stencil-on-load) still computes the right values, only slower.  Here the per-op call
counts of the lane kernel (Context.opprof: thread 0 of every CTA, exact on the emulator) are compared with fixed histograms
for the field operators, the solvers and one Navier2D step, fused and unfused, on the E = 16 / 8 / 4 compile-time layouts and
on the generic instance.  Says nothing about GPU timing."""
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
import rustpde_mpi_b200 as b2

n = int(sys.argv[1])
ctx = b2.Context(0)
rng = np.random.default_rng(0)
CD, CN, CDN, R2C = 1, 2, 3, 4
out = {}


def run(name, fn):
    ctx.opprof(True)
    fn()
    out[name] = {k: c for k, (_, c) in ctx.opprof(False).items()}


f = b2.Field2(b2.Space2((CD, n), (CD, n), ctx=ctx))
f.vhat = rng.standard_normal(f.vhat.shape)
ortho = f.to_ortho()
run("forward", f.forward)
run("backward", f.backward)
run("to_ortho", f.to_ortho)
run("from_ortho", lambda: f.from_ortho(ortho))
run("gradient", lambda: f.gradient((1, 1), (1.0, 1.0)))
rhs = ortho.get()
h = b2.HholtzAdi(f, [0.02, 0.03])
run("hholtz", lambda: h.solve(rhs))
fc = b2.Field2(b2.Space2((CD, n), (CDN, n), ctx=ctx))
hc = b2.HholtzAdi(fc, [0.02, 0.03])
run("hholtz_cdn", lambda: hc.solve(rng.standard_normal(fc.to_ortho().get().shape)))
fp = b2.Field2(b2.Space2((CN, n), (CD, n), ctx=ctx))
pc = b2.Poisson(fp, [1.0, 1.0])
run("poisson_confined", lambda: pc.solve(rng.standard_normal(fp.to_ortho().get().shape)))
ff = b2.Field2(b2.Space2((R2C, n - 1), (CD, n), ctx=ctx))
pf = b2.Poisson(ff, [1.0, 1.0])
run("poisson_fourier", lambda: pf.solve(rng.standard_normal(ff.to_ortho().get().shape)))
nav = b2.Navier2D(n, n, 1e5, 1.0, 0.01, 1.0, "rbc", ctx=ctx)
for mode in (3, 0):
    nav.set_mode(mode)
    run(f"navier_mode{mode}", lambda: nav.update(1))
lay = f.space.layout(0)
print("HIST " + json.dumps({"layout": [lay["E"], lay["TPL"], lay["fast"]], "hist": out}))
''' % ROOT

# case: (environment, lane points, (E, TPL, fast) of the passes with lanes along axis 1)
CASES = {
    "e16": ({"B2_E": "16"}, 257, (16, 8, 1)),
    "e8": ({}, 129, (8, 8, 1)),
    "e4": ({"B2_E": "4"}, 129, (4, 16, 1)),
    "generic": ({"B2_NOFAST": "1"}, 129, (8, 8, 0)),
}

# {workload: "op=calls ..."}, recorded on the emulator
EXPECTED = {
    "e16": {
        "forward": "bandc=130 dct=130 dct.fft=130 dct.post=130 dct.pre=130 fdma=130 fdma.compose=130 fdma.fwd_apply=130 fdma.fwd_reduce=130 fdma.scan1=130 fdma.scan2=130 fdma.solve=130 ld.direct_first=130 load=130 store=130",
        "backward": "bandc=130 dct=130 dct.fft=130 dct.post=130 dct.pre=130 ld.direct_first=130 load=130 store=130",
        "to_ortho": "bandc=130 ld.direct_first=130 load=130 store=130",
        "from_ortho": "bandc=130 fdma=130 fdma.compose=130 fdma.fwd_apply=130 fdma.fwd_reduce=130 fdma.scan1=130 fdma.scan2=130 fdma.solve=130 ld.direct_first=130 load=130 store=130",
        "gradient": "bandc=130 deriv=130 ld.direct_first=130 load=130 store=130",
        "hholtz": "bandc=130 fdma=130 fdma.compose=130 fdma.fwd_apply=130 fdma.fwd_reduce=130 fdma.scan1=130 fdma.scan2=130 fdma.solve=130 ld.direct_first=130 load=130 store=130",
        "hholtz_cdn": "bandc=195 fdma=65 fdma.compose=65 fdma.fwd_apply=65 fdma.fwd_reduce=130 fdma.scan1=130 fdma.scan2=65 fdma.solve=65 ld.direct_first=260 load=260 store=260",
        "poisson_confined": "bandc=260 fdma=65 fdma.compose=65 fdma.fwd_apply=65 fdma.fwd_reduce=65 fdma.scan1=65 fdma.scan2=65 fdma.solve=65 ld.direct_first=390 load=390 store=390",
        "poisson_fourier": "bandc=130 fdma=65 fdma.compose=65 fdma.fwd_apply=65 fdma.fwd_reduce=65 fdma.scan1=65 fdma.scan2=65 fdma.solve=65 ld.direct_first=260 load=260 store=260",
        "navier_mode3": "bandc=2340 dct=1300 dct.fft=1300 dct.post=1300 dct.pre=1300 deriv=780 fdma=1105 fdma.compose=1105 fdma.fwd_apply=1105 fdma.fwd_reduce=1105 fdma.scan1=1105 fdma.scan2=1105 fdma.solve=1105 ld.combine=975 ld.direct_first=1495 ld.direct_later=910 ld.stencil=325 load=3705 store=2730 zerotail=390",
        "navier_mode0": "bandc=2990 dct=1430 dct.fft=1430 dct.post=1430 dct.pre=1430 deriv=910 fdma=715 fdma.compose=715 fdma.fwd_apply=715 fdma.fwd_reduce=715 fdma.scan1=715 fdma.scan2=715 fdma.solve=715 ld.direct_first=4810 load=4810 store=4810 zerotail=390",
    },
    "e8": {
        "forward": "dct=66 dct.fft=66 dct.post=66 dct.pre=66 fdma=66 fdma.compose=66 fdma.fwd_apply=66 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=66 fdma.solve=66 ld.direct_first=66 load=66 store=66",
        "backward": "bandc=66 dct=66 dct.fft=66 dct.post=66 dct.pre=66 ld.direct_first=66 load=66 store=66",
        "to_ortho": "bandc=66 ld.direct_first=66 load=66 store=66",
        "from_ortho": "fdma=66 fdma.compose=66 fdma.fwd_apply=66 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=66 fdma.solve=66 ld.direct_first=66 load=66 store=66",
        "gradient": "bandc=66 deriv=66 ld.direct_first=66 load=66 store=66",
        "hholtz": "fdma=66 fdma.compose=66 fdma.fwd_apply=66 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=66 fdma.solve=66 ld.direct_first=66 load=66 store=66",
        "hholtz_cdn": "bandc=66 fdma=33 fdma.compose=33 fdma.fwd_apply=33 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=33 fdma.solve=33 ld.direct_first=132 load=132 store=132",
        "poisson_confined": "bandc=132 fdma=33 fdma.compose=33 fdma.fwd_apply=33 fdma.fwd_reduce=33 fdma.scan1=33 fdma.scan2=33 fdma.solve=33 ld.direct_first=198 load=198 store=198",
        "poisson_fourier": "bandc=66 fdma=33 fdma.compose=33 fdma.fwd_apply=33 fdma.fwd_reduce=33 fdma.scan1=33 fdma.scan2=33 fdma.solve=33 ld.direct_first=132 load=132 store=132",
        "navier_mode3": "bandc=660 dct=660 dct.fft=660 dct.post=660 dct.pre=660 deriv=396 fdma=561 fdma.compose=561 fdma.fwd_apply=561 fdma.fwd_reduce=561 fdma.scan1=561 fdma.scan2=561 fdma.solve=561 ld.combine=495 ld.direct_first=759 ld.direct_later=462 ld.stencil=165 load=1881 store=1386 zerotail=198",
        "navier_mode0": "bandc=1188 dct=726 dct.fft=726 dct.post=726 dct.pre=726 deriv=462 fdma=363 fdma.compose=363 fdma.fwd_apply=363 fdma.fwd_reduce=363 fdma.scan1=363 fdma.scan2=363 fdma.solve=363 ld.direct_first=2442 load=2442 store=2442 zerotail=198",
    },
    "e4": {
        "forward": "dct=66 dct.fft=66 dct.post=66 dct.pre=66 fdma=66 fdma.compose=66 fdma.fwd_apply=66 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=66 fdma.solve=66 ld.direct_first=66 load=66 store=66",
        "backward": "bandc=66 dct=66 dct.fft=66 dct.post=66 dct.pre=66 ld.direct_first=66 load=66 store=66",
        "to_ortho": "bandc=66 ld.direct_first=66 load=66 store=66",
        "from_ortho": "fdma=66 fdma.compose=66 fdma.fwd_apply=66 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=66 fdma.solve=66 ld.direct_first=66 load=66 store=66",
        "gradient": "bandc=66 deriv=66 ld.direct_first=66 load=66 store=66",
        "hholtz": "fdma=66 fdma.compose=66 fdma.fwd_apply=66 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=66 fdma.solve=66 ld.direct_first=66 load=66 store=66",
        "hholtz_cdn": "bandc=66 fdma=33 fdma.compose=33 fdma.fwd_apply=33 fdma.fwd_reduce=66 fdma.scan1=66 fdma.scan2=33 fdma.solve=33 ld.direct_first=132 load=132 store=132",
        "poisson_confined": "bandc=132 fdma=33 fdma.compose=33 fdma.fwd_apply=33 fdma.fwd_reduce=33 fdma.scan1=33 fdma.scan2=33 fdma.solve=33 ld.direct_first=198 load=198 store=198",
        "poisson_fourier": "bandc=66 fdma=33 fdma.compose=33 fdma.fwd_apply=33 fdma.fwd_reduce=33 fdma.scan1=33 fdma.scan2=33 fdma.solve=33 ld.direct_first=132 load=132 store=132",
        "navier_mode3": "bandc=660 dct=660 dct.fft=660 dct.post=660 dct.pre=660 deriv=396 fdma=561 fdma.compose=561 fdma.fwd_apply=561 fdma.fwd_reduce=561 fdma.scan1=561 fdma.scan2=561 fdma.solve=561 ld.combine=495 ld.direct_first=759 ld.direct_later=462 ld.stencil=165 load=1881 store=1386 zerotail=198",
        "navier_mode0": "bandc=1188 dct=726 dct.fft=726 dct.post=726 dct.pre=726 deriv=462 fdma=363 fdma.compose=363 fdma.fwd_apply=363 fdma.fwd_reduce=363 fdma.scan1=363 fdma.scan2=363 fdma.solve=363 ld.direct_first=2442 load=2442 store=2442 zerotail=198",
    },
    "generic": {
        "forward": "band=66 dct=66 fdma=66 ld.direct_first=66 load=66 store=66",
        "backward": "dct=66 ld.stencil=66 load=66 store=66",
        "to_ortho": "ld.stencil=66 load=66 store=66",
        "from_ortho": "band=66 fdma=66 ld.direct_first=66 load=66 store=66",
        "gradient": "deriv=66 ld.stencil=66 load=66 store=66",
        "hholtz": "band=66 fdma=66 ld.direct_first=66 load=66 store=66",
        "hholtz_cdn": "band=66 fdma=33 fdma.fwd_reduce=33 fdma.scan1=33 ld.direct_first=99 ld.stencil=33 load=132 store=132",
        "poisson_confined": "band=66 fdma=33 ld.direct_first=132 ld.stencil=66 load=198 store=198",
        "poisson_fourier": "band=33 fdma=33 ld.direct_first=99 ld.stencil=33 load=132 store=132",
        "navier_mode3": "band=594 dct=660 deriv=396 fdma=561 ld.combine=495 ld.direct_first=297 ld.direct_later=330 ld.stencil=759 load=1881 store=1386 zerotail=198",
        "navier_mode0": "band=396 dct=726 deriv=462 fdma=363 ld.direct_first=1320 ld.stencil=1122 load=2442 store=2442 zerotail=198",
    },
}


def histograms(case):
    env, n, _ = CASES[case]
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(n)], capture_output=True, text=True, timeout=1800, cwd=ROOT,
                       env=dict(os.environ, **env))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("HIST ")][-1]
    res = json.loads(line[5:])
    assert tuple(res["layout"]) == CASES[case][2], res["layout"]
    return res["hist"]


def fmt(h):
    return " ".join(f"{k}={v}" for k, v in sorted(h.items()))


@pytest.mark.parametrize("case", sorted(CASES))
def test_lane_program_forms(case):
    got = {w: fmt(h) for w, h in histograms(case).items()}
    assert got == EXPECTED[case]


if __name__ == "__main__":   # print the histograms of one case in the form of EXPECTED
    for w, h in histograms(sys.argv[1]).items():
        print(f'        "{w}": "{fmt(h)}",')
