"""FourierC2c lanes on the lane FFT (tests/test_gpu_c2c_fft.py) on the SIMT emulator of tests/emu: the layout of every case, the
claim that the cases reach every lane-kernel instance a c2c lane can run on, the lane programs (one OP_CFFT per lane group, no
OP_DENSE at FFT sizes), the operators of the cases with n <= 128 against numpy and the oracle, one radix-3 and one power-of-two
case under the emulator's race schedule, and a c2c x cd space on two ranks."""
import itertools
import json
import os
import subprocess
import sys

import pytest

from tests import test_gpu_c2c_fft as cf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = [c for c in cf.CASE if cf.CASE[c][1] <= 128]
EMU_CROSS = 17
OP_DENSE, OP_CFFT = 18, 19   # lane_kernel.cuh LaneOpCode


def emulated(code, env=None):
    """run ``code`` in a fresh process on the emulator build (the layout switches are read when a space is created)"""
    head = f"import sys\nsys.path.insert(0, {ROOT!r})\nfrom tests import emu\nemu.activate()\n"
    base = {k: v for k, v in os.environ.items() if k not in cf.SWITCHES}
    r = subprocess.run([sys.executable, "-c", head + code], capture_output=True, text=True, timeout=1800, cwd=ROOT,
                       env=dict(base, **(env or {})))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
    return r.stdout


@pytest.mark.parametrize("case", list(cf.CASE))
def test_emulated_c2c_layout(case):
    env, n, want = cf.CASE[case]
    emulated(f"from tests import test_gpu_c2c_fft as t\n"
             f"for kind1 in (t.CD, t.CN, t.CH):\n"
             f"    lay = t.layout((t.C2C, {n}, kind1, {EMU_CROSS}))\n"
             f"    assert lay == {tuple(want)!r}, (kind1, lay)\n"
             f"print('ok')\n", env)


def instance(lay):
    """the lane-kernel instance a layout runs: (E, LN, TPL) compile-time geometry, or (E, LN) generic"""
    e, ln, tpl, fast = lay
    return (e, ln, tpl) if fast else (e, ln)


def test_cases_cover_every_reachable_instance():
    """every c2c FFT size (2n = f * 2^k >= 64, f = 1, 3, 5, n <= 1024) under every setting of the layout switches: the
    instances those lanes run on are exactly the ones the case table runs"""
    sizes = [n for n in range(32, 1025) if (2 * n) // ((2 * n) & -(2 * n)) in (1, 3, 5)]
    reached = set()
    for e, ln, nofast in itertools.product((None, "4", "8", "16"), (None, "2"), (None, "1")):
        env = {k: v for k, v in (("B2_E", e), ("B2_LN", ln), ("B2_NOFAST", nofast)) if v is not None}
        out = emulated(f"from tests import test_gpu_c2c_fft as t\n"
                       f"print('LAYS', [t.layout((t.C2C, n, t.CD, {EMU_CROSS})) for n in {sizes!r}])\n"
                       f"print('ok')\n", env)
        lays = eval([l for l in out.splitlines() if l.startswith("LAYS ")][0][5:])
        # an FFT layout has E * TPL = n; sizes without one run the dense transform on the banded-only layout (16, 4, TPL, 0)
        reached |= {instance(lay) for n, lay in zip(sizes, lays) if lay[0] * lay[2] == n}
    covered = {instance(c[3]) for c in cf.CASES}
    assert reached == covered, (sorted(reached - covered, key=str), sorted(covered - reached, key=str))


OPCOUNT = r'''
import ctypes as C
import json
import numpy as np
import rustpde_mpi_b200 as b2
from rustpde_mpi_b200._lib import check, lib
ctx = b2.Context(0)
out = {}
for n in (32, 96, 128, 1024, 100, 48):
    # axis 1 orthonormal Chebyshev: its passes run OP_DCT only, so the slots of OP_DENSE and OP_CFFT count the c2c lanes' transforms alone (the
    # compile-time LU solve also records phases in slots 16 .. 21)
    f = b2.Field2(b2.Space2((5, n), (0, 65), ctx=ctx))
    f.v = np.ones((n, 65)) + 0j
    for name, fn in (("forward", f.forward), ("backward", f.backward)):
        ctx.opprof(True)
        fn()
        buf = (C.c_ulonglong * 64)()
        check(lib().b2_ctx_opprof(ctx._h, 0, buf))
        out[f"{n} {name}"] = [buf[32 + %d], buf[32 + %d]]
print("COUNTS " + json.dumps(out))
print("ok")
''' % (OP_DENSE, OP_CFFT)


def test_c2c_lane_programs():
    """calls of OP_DENSE and OP_CFFT (Context.opprof's counters, thread 0 of every CTA: exact on the emulator) in a forward and a
    backward of c2c n x ch 65: one OP_CFFT per lane group (65 columns = 17 groups of 4 lanes, one CTA each) and no OP_DENSE at
    the FFT sizes; OP_DENSE and no OP_CFFT at 100 and 48 (no factorisation / no thread layout)"""
    out = emulated(OPCOUNT)
    got = json.loads([l for l in out.splitlines() if l.startswith("COUNTS ")][0][7:])
    want = {}
    for n in (32, 96, 128, 1024, 100, 48):
        fft = n not in (100, 48)
        for name in ("forward", "backward"):
            want[f"{n} {name}"] = [0, 17] if fft else [17, 0]
    assert got == want


@pytest.mark.parametrize("case", SMALL)
def test_emulated_c2c_operators(case):
    cf.run_case(case, "emu", cross=EMU_CROSS, sequences=False)


@pytest.mark.parametrize("case", ["r3-96", "n64"])
def test_emulated_c2c_race_schedule(case):
    """forward and backward against numpy under B2_EMU_SKEW_US (after every block barrier the warps resume in a skewed order):
    the backward's conjugation runs without a barrier in front of the FFT"""
    env, n, want = cf.CASE[case]
    emulated(f"""
from tests import test_gpu_c2c_fft as t
assert t.layout((t.C2C, {n}, t.CD, {EMU_CROSS})) == {tuple(want)!r}
errs = t.numpy_errors(t.CD, {n}, {EMU_CROSS})
assert max(errs.values()) < t.TOL, errs
print("ok")
""", dict(env, B2_EMU_SKEW_US="2000,rev"))


def run_ranks(world, args, port):
    """tests/c2c_dist_worker.py on ``world`` emulated ranks.  Like tests.test_dist_gloo.run (which runs its own worker), a failed
    run is reported and repeated once on a fresh port: the emulator's scheduling (one OS thread per CUDA thread, ranks as
    processes on a few cores) must not fail the suite, two failures in a row do."""
    env = dict(os.environ, B2_TEST_EMU="1", OMP_NUM_THREADS="1")
    for k in cf.SWITCHES:
        env.pop(k, None)
    for attempt in range(2):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
               "127.0.0.1", "--master-port", str(port + 100 * attempt), os.path.join(ROOT, "tests", "c2c_dist_worker.py")]
        r = subprocess.run(cmd + [str(a) for a in args], capture_output=True, text=True, timeout=1500, cwd=ROOT, env=env)
        if r.returncode == 0:
            break
        sys.stderr.write("first attempt failed:\n" + r.stdout[-1500:] + r.stderr[-2500:] + "\n")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert r.stdout.count("worst_rel_err") == world, r.stdout[-2000:]


def test_emulated_c2c_two_ranks():
    """c2c 64 x cd 33 on two emulated ranks (slabs of 64 rows each, cfft_fast): forward, backward and Poisson against the serial
    oracle"""
    run_ranks(2, (64, 33, 1), 29641)


def test_emulated_c2c_seven_ranks_keep_the_dense_transform():
    """c2c 32 on 7 ranks: the pitch (84 = 64 rounded up to 4 x 7) exceeds the 80 elements of the only FFT layout (E = 4, TPL = 8),
    so the lanes keep the dense transform on the banded-only layout (16, 4, 8, 0) instead of refusing the space; forward,
    backward and Poisson on 7 emulated ranks against the serial oracle"""
    emulated(f"""
import rustpde_mpi_b200 as b2
ctx = b2.Context(0, 0, 7, heap_bytes=64 << 20)
for kind1 in (1, 2):
    s = b2.Space2((5, 32), (kind1, {EMU_CROSS}), ctx=ctx)
    lay = s.layout(1)
    assert (lay["E"], lay["LN"], lay["TPL"], lay["fast"]) == (16, 4, 8, 0), lay
    s.close()
print("ok")
""")
    run_ranks(7, (32, 17, 0), 29642)
