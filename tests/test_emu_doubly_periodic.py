"""Doubly periodic spaces (tests/test_gpu_doubly_periodic.py) on the SIMT emulator of tests/emu: the operators and the call
sequence at nx, ny in {32, 64, 96, 128} and one dense size per axis, the layout of every GPU case, the claim that the GPU cases
reach every lane-kernel instance an r2c lane can run on (on each axis), the split-lane ops under the emulator's race schedule,
and a 64 x 64 space on two ranks."""
import itertools
import os
import subprocess
import sys

import pytest

from tests import test_gpu_doubly_periodic as dp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (nx, ny): 32 and 96 run the r2c dense matrices (N < 64, no thread layout for 3 * 32), 64 and 128 the lane FFT; 48 / 100 are dense too
SIZES = [(32, 64), (64, 64), (96, 64), (128, 64), (48, 64), (64, 32), (64, 96), (64, 128), (64, 100), (128, 96)]


def emulated(code, env=None):
    """run ``code`` in a fresh process on the emulator build (the layout switches are read when a space is created)"""
    head = f"import sys\nsys.path.insert(0, {ROOT!r})\nfrom tests import emu\nemu.activate()\n"
    base = {k: v for k, v in os.environ.items() if k not in dp.SWITCHES}
    r = subprocess.run([sys.executable, "-c", head + code], capture_output=True, text=True, timeout=1800, cwd=ROOT,
                       env=dict(base, **(env or {})))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
    return r.stdout


@pytest.mark.parametrize("nx,ny", SIZES)
def test_emulated_doubly_periodic_operators(nx, ny):
    emulated(f"""
from tests import test_gpu_doubly_periodic as t
bad, worst = t.case_failures({nx}, {ny})
assert not bad, bad
print("ok")
""")


def test_emulated_doubly_periodic_layouts():
    """every GPU case's layout, with its switches"""
    by_env = {}
    for name, (env, nx, ny, axis, want) in dp.CASE.items():
        by_env.setdefault(tuple(sorted(env.items())), []).append((name, nx, ny, axis, tuple(want)))
    for env, cases in by_env.items():
        emulated(f"""
from tests import test_gpu_doubly_periodic as t
for name, nx, ny, axis, want in {cases!r}:
    lay = t.layout(nx, ny, axis)
    assert lay == want, (name, lay, want)
print("ok")
""", dict(env))


def instance(lay):
    e, ln, tpl, fast = lay
    return (e, ln, tpl) if fast else (e, ln)


def test_cases_cover_every_reachable_instance():
    """every r2c FFT size (n = f * 2^k >= 64, f = 1, 3, 5, up to 8192) under every setting of the layout switches, on each axis:
    the instances those lanes run on are exactly the ones the GPU cases run on that axis"""
    sizes = [n for n in range(64, 8193, 2) if n // (n & -n) in (1, 3, 5)]
    reached = {0: set(), 1: set()}
    for e, ln, nofast in itertools.product((None, "4", "8", "16"), (None, "2"), (None, "1")):
        env = {k: v for k, v in (("B2_E", e), ("B2_LN", ln), ("B2_NOFAST", nofast)) if v is not None}
        out = emulated(f"""
from tests import test_gpu_doubly_periodic as t
lays = {{}}
for n in {sizes!r}:
    try:
        lays[n] = (t.layout(n, 64, 0), t.layout(64, n, 1))
    except Exception:
        pass   # no thread layout for this size under these switches
print('LAYS', lays)
print('ok')
""", env)
        lays = eval([ln_ for ln_ in out.splitlines() if ln_.startswith("LAYS ")][0][5:])
        for n, per_axis in lays.items():
            for axis in (0, 1):
                lay = per_axis[axis]
                if 2 * lay[0] * lay[2] == n:   # an FFT layout (E * TPL = n / 2); other sizes run the dense matrices
                    reached[axis].add(instance(lay))
    for axis in (0, 1):
        covered = {instance(c[5]) for c in dp.CASES if c[4] == axis}
        assert reached[axis] == covered, (axis, sorted(reached[axis] - covered, key=str), sorted(covered - reached[axis], key=str))


@pytest.mark.parametrize("order", ["rev", "fwd"])
@pytest.mark.parametrize("nx,ny", [(64, 64), (128, 32)])
def test_emulated_split_ops_race_schedule(nx, ny, order):
    """OP_CPAIR (forward, backward) and OP_SDIFF (odd x derivatives swap Re and Im between the lanes of a pair) under
    B2_EMU_SKEW_US: after every block barrier the warps resume in a skewed order, so a read of the partner lane or of position
    n - k that a write overtakes shows up"""
    emulated(f"""
import numpy as np
import rustpde_mpi_b200 as b2
from tests import test_gpu_doubly_periodic as t
nx, ny = {nx}, {ny}
f = b2.Field2(b2.Space2((t.C2C, nx), (t.R2C, ny)))
rng = np.random.default_rng(4)
v = rng.uniform(-1, 1, (nx, ny))
f.v = v; f.forward()
errs = {{"forward": t.relerr(f.vhat, np.fft.rfft2(v))}}
a = t.rand_spec(nx, ny, rng)
f.vhat = a; f.backward()
errs["backward"] = t.relerr(f.v, np.fft.irfft2(a, s=(nx, ny)))
sp = t.oracle_space(nx, ny)
for d in ((1, 0), (3, 1), (2, 0)):
    errs[str(d)] = t.relerr(f.gradient(d, (1.3, 0.7)).get(), sp.gradient(a, d, (1.3, 0.7)))
assert max(errs.values()) < t.TOL, errs
print("ok")
""", {"B2_EMU_SKEW_US": f"2000,{order}"})


def test_emulated_doubly_periodic_two_ranks():
    """c2c 64 x r2c 64 on two emulated ranks: gathered forward, backward, gradient and Poisson against the serial oracle.  Like
    the other emulated multi-rank tests, a failed run is repeated once on a fresh port (the emulator's scheduling must not fail
    the suite), two failures in a row do."""
    env = dict(os.environ, B2_TEST_EMU="1", OMP_NUM_THREADS="1")
    for k in dp.SWITCHES:
        env.pop(k, None)
    for attempt in range(2):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
               "--master-port", str(29651 + 100 * attempt), os.path.join(ROOT, "tests", "dp_dist_worker.py"), "64", "64"]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT, env=env)
        if r.returncode == 0:
            break
        sys.stderr.write("first attempt failed:\n" + r.stdout[-1500:] + r.stderr[-2500:] + "\n")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert r.stdout.count("worst_rel_err") == 2, r.stdout[-2000:]
