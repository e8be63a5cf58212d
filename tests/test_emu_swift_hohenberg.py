"""SwiftHohenberg2D (tests/test_gpu_swift_hohenberg.py) on the SIMT emulator of tests/emu: 30 steps against numpy at small sizes
(lane FFT and dense transforms), the new lane ops under the emulator's race schedule, two emulated ranks, and the behaviour of the
Python surface (update, time, snapshots, exit, integrate, refused arguments)."""
import os
import subprocess
import sys

import pytest

from tests import test_gpu_doubly_periodic as dp
from tests.test_emu_doubly_periodic import emulated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("nx,ny", [(64, 64), (128, 32), (32, 128), (48, 48)])
def test_emulated_swift_hohenberg_steps(nx, ny):
    """30 steps against sh_numpy within max(1e-10, 10 x yardstick); 32 and 48 run the dense transforms"""
    emulated(f"""
from tests import test_gpu_swift_hohenberg as t
err, bound, sh = t.sh_errors({nx}, {ny}, 30)
assert err < bound, (err, bound)
assert sh.launches_per_step() == 4
print("ok")
""")


@pytest.mark.parametrize("order", ["rev", "fwd"])
@pytest.mark.parametrize("nx,ny", [(64, 64), (128, 32)])
def test_emulated_swift_hohenberg_race_schedule(nx, ny, order):
    """OP_CUBE, the SH division and the mode fix (reads of elements 1 .. (n-1)/2, writes of n - i) under B2_EMU_SKEW_US: after
    every block barrier the warps resume in a skewed order, so a read that a write overtakes shows up"""
    emulated(f"""
from tests import test_gpu_swift_hohenberg as t
err, bound, _ = t.sh_errors({nx}, {ny}, 3)
assert err < bound, (err, bound)
print("ok")
""", {"B2_EMU_SKEW_US": f"2000,{order}"})


def test_emulated_swift_hohenberg_two_ranks():
    """64 x 64 on two emulated ranks: the gathered theta_hat after 20 steps against serial numpy, and the global norm.  Like the
    other emulated multi-rank tests, a failed run is repeated once on a fresh port; two failures in a row fail."""
    env = dict(os.environ, B2_TEST_EMU="1", OMP_NUM_THREADS="1")
    for k in dp.SWITCHES:
        env.pop(k, None)
    for attempt in range(2):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
               "--master-port", str(29671 + 100 * attempt), os.path.join(ROOT, "tests", "sh_dist_worker.py"), "64", "64", "20"]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT, env=env)
        if r.returncode == 0:
            break
        sys.stderr.write("first attempt failed:\n" + r.stdout[-1500:] + r.stderr[-2500:] + "\n")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert r.stdout.count("worst_rel_err") == 2, r.stdout[-2000:]


def test_emulated_swift_hohenberg_update_and_time():
    """update(0) changes nothing, update(5) is bit-identical to five update(1), get_time() = n dt, 4 lane passes per step"""
    emulated("""
import numpy as np
import rustpde_mpi_b200 as b2
from tests import test_gpu_doubly_periodic as t
a = b2.SwiftHohenberg2D(64, 64, t.SH_R, t.SH_DT, t.SH_L, seed=3)
b = b2.SwiftHohenberg2D(64, 64, t.SH_R, t.SH_DT, (t.SH_L, t.SH_L), seed=3)
v0 = a.theta.vhat
a.update(0)
assert np.array_equal(a.theta.vhat, v0) and a.get_time() == 0.0
a.update(5)
for _ in range(5):
    b.update(1)
assert np.array_equal(a.theta.vhat, b.theta.vhat)
assert abs(a.get_time() - 5 * t.SH_DT) < 1e-14 and a.get_time() == b.get_time()
assert a.get_dt() == t.SH_DT and a.launches_per_step() == 4
print("ok")
""")


def test_emulated_swift_hohenberg_snapshot_and_exit(tmp_path):
    """write then read into a fresh object restores theta_hat bitwise and the time; exit() is False on a normal state and True
    once a NaN is in theta_hat; a snapshot of another grid is refused"""
    emulated(f"""
import numpy as np
import rustpde_mpi_b200 as b2
from rustpde_mpi_b200 import snapshot as sn
from tests import test_gpu_doubly_periodic as t
a = b2.SwiftHohenberg2D(64, 32, t.SH_R, t.SH_DT, t.SH_L)
a.update(3)
fn = {str(tmp_path / "snap.npz")!r}
a.write(fn)
d = sn.load_datasets(fn)
assert d["temp/v"].shape == (64, 32) and d["temp/vhat_re"].shape == (64, 17)
assert float(d["dt"]) == t.SH_DT and float(d["r"]) == t.SH_R and float(d["time"]) == a.get_time()
assert np.allclose(d["temp/v"], np.fft.irfft2(a.theta.vhat, s=(64, 32)), atol=1e-14)
b = b2.SwiftHohenberg2D(64, 32, t.SH_R, t.SH_DT, t.SH_L, init_random=False)
b.read(fn)
assert np.array_equal(b.theta.vhat, a.theta.vhat) and b.get_time() == a.get_time()
assert not a.exit()
vh = a.theta.vhat
vh[5, 3] = np.nan
a.theta.vhat = vh
assert a.exit()
c = b2.SwiftHohenberg2D(32, 32, t.SH_R, t.SH_DT, t.SH_L, init_random=False)
try:
    c.read(fn)
    raise SystemExit("a snapshot of another grid was accepted")
except b2.B2Error:
    pass
print("ok")
""")


def test_emulated_swift_hohenberg_integrate(tmp_path):
    """integrate(pde, 0.2, 0.1) at dt = 0.02 with io_dir set writes the two flow files with the datasets of _write"""
    out = emulated(f"""
import os
import numpy as np
import rustpde_mpi_b200 as b2
from rustpde_mpi_b200 import snapshot as sn
from tests import test_gpu_doubly_periodic as t
sh = b2.SwiftHohenberg2D(64, 64, t.SH_R, t.SH_DT, t.SH_L)
sh.io_dir = {str(tmp_path)!r}
b2.integrate(sh, 0.2, 0.1)
files = sorted(os.listdir(sh.io_dir))
assert files == ["flow00000.10.npz", "flow00000.20.npz"], files
for f in files:
    d = sn.load_datasets(os.path.join(sh.io_dir, f))
    for k in ("temp/v", "temp/vhat_re", "temp/vhat_im", "time", "dt", "r"):
        assert k in d, (f, k, sorted(d))
assert abs(sh.get_time() - 0.2) < 1e-12
print("ok")
""")
    assert out.count("Time = ") == 2 and out.count("|F| = ") == 2, out


def test_emulated_swift_hohenberg_refusals():
    """spaces other than fourier_c2c x fourier_r2c, non-finite r / dt, a non-positive length and update(-1) raise B2Error"""
    emulated("""
import rustpde_mpi_b200 as b2
from rustpde_mpi_b200._lib import B2Error, check, lib
import ctypes as C
from tests import test_gpu_doubly_periodic as t

def refused(fn):
    try:
        fn()
    except B2Error:
        return True
    return False

for bases in ((b2.fourier_r2c(64), b2.cheb_dirichlet(65)), (b2.fourier_c2c(64), b2.cheb_dirichlet(65))):
    f = b2.Field2(b2.Space2(*bases))
    h = C.c_void_p()
    sc = (C.c_double * 2)(20.0, 20.0)
    assert refused(lambda: check(lib().b2_sh2d_create(f._h, 0.35, 0.02, sc, C.byref(h)))), bases
assert refused(lambda: b2.SwiftHohenberg2D(64, 64, t.SH_R, float("nan"), t.SH_L))
assert refused(lambda: b2.SwiftHohenberg2D(64, 64, float("inf"), t.SH_DT, t.SH_L))
assert refused(lambda: b2.SwiftHohenberg2D(64, 64, t.SH_R, t.SH_DT, 0.0))
assert refused(lambda: b2.SwiftHohenberg2D(64, 64, t.SH_R, t.SH_DT, (20.0, -1.0)))
sh = b2.SwiftHohenberg2D(64, 64, t.SH_R, t.SH_DT, t.SH_L, init_random=False)
assert refused(lambda: sh.update(-1))
print("ok")
""")
