"""SwiftHohenberg2D (examples/swift_hohenberg_2d.rs) on the GPU: the 4-pass step against the same implicit steps in numpy
(sh_numpy of tests/test_gpu_doubly_periodic.py) at the example's parameters r = 0.35, dt = 0.02, L = 20.  The model is a gradient
flow, so rounding differences do not grow exponentially: long runs are held to max(1e-10, 10 x the numpy run's own change when the
start moves in the last bit).  tests/test_emu_swift_hohenberg.py runs the small sizes on the emulator."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import test_gpu_doubly_periodic as dp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sh_errors(nx, ny, steps, seed=0):
    """(relative error of theta_hat after ``steps`` updates against sh_numpy, its bound, the model object)"""
    import rustpde_mpi_b200 as b2

    sh = b2.SwiftHohenberg2D(nx, ny, dp.SH_R, dp.SH_DT, dp.SH_L, seed=seed)
    theta0 = sh.theta.v
    sh.update(steps)
    ref = dp.sh_numpy(theta0, steps)
    yard = dp.relerr(dp.sh_numpy(dp.perturbed(theta0, 3), steps), ref)
    return dp.relerr(sh.theta.vhat, ref), max(dp.TOL, 10.0 * yard), sh


# every layout case of the doubly periodic spaces in a process of its own (the layout switches are read when a space is created)
SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
if sys.argv[2] == "emu":
    from tests import emu
    emu.activate()
from tests import test_gpu_doubly_periodic as dp
from tests import test_gpu_swift_hohenberg as t
case = json.loads(sys.argv[1])
_, nx, ny, axis, want = dp.CASE[case]
lay = dp.layout(nx, ny, axis)
assert lay == tuple(want), (case, lay, want)
err, bound, sh = t.sh_errors(nx, ny, 20)
assert sh.launches_per_step() == 4, sh.launches_per_step()
print("err", err, "bound", bound)
assert err < bound, (err, bound)
print("ok")
''' % ROOT


def run_case(case, where):
    env = dict({k: v for k, v in os.environ.items() if k not in dp.SWITCHES}, **dp.CASE[case][0])
    r = subprocess.run([sys.executable, "-c", SCRIPT, json.dumps(case), where], capture_output=True, text=True, timeout=3600,
                       cwd=ROOT, env=env)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(dp.CASE))
def test_swift_hohenberg_case(case):
    """the layout of the case, then 20 steps against numpy: every lane-kernel instance OP_CUBE (y lanes) and the SH division and
    mode fix (x lanes) run on"""
    run_case(case, "gpu")


@pytest.mark.gpu
def test_swift_hohenberg_2000_steps_512():
    err, bound, sh = sh_errors(512, 512, 2000)
    print(f"[swift-hohenberg 512^2] 2000 steps: relative error {err:.2e}, bound {bound:.2e}")
    assert err < bound, (err, bound)
    assert abs(sh.get_time() - 2000 * dp.SH_DT) < 1e-9


@pytest.mark.gpu
def test_swift_hohenberg_4096():
    err, bound, _ = sh_errors(4096, 4096, 10)
    print(f"[swift-hohenberg 4096^2] 10 steps: relative error {err:.2e}, bound {bound:.2e}")
    assert err < bound, (err, bound)


@pytest.mark.gpu
def test_swift_hohenberg_integrate(tmp_path, capsys):
    """integrate() over the example's setup (512^2) to t = 1 with save_intervall 0.5: both callbacks print and write their flow
    file, and the final state matches numpy"""
    import rustpde_mpi_b200 as b2

    sh = b2.SwiftHohenberg2D(512, 512, dp.SH_R, dp.SH_DT, dp.SH_L)
    theta0 = sh.theta.v
    sh.io_dir = str(tmp_path)
    b2.integrate(sh, 1.0, 0.5)
    out = capsys.readouterr().out
    assert out.count("Time = ") == 2 and out.count("|F| = ") == 2, out
    files = sorted(os.path.basename(f) for f in glob.glob(os.path.join(str(tmp_path), "flow*")))
    assert [f.split(".npz")[0].split(".h5")[0] for f in files] == ["flow00000.50", "flow00001.00"], files
    ref = dp.sh_numpy(theta0, 50)
    yard = dp.relerr(dp.sh_numpy(dp.perturbed(theta0, 3), 50), ref)
    assert dp.relerr(sh.theta.vhat, ref) < max(dp.TOL, 10.0 * yard)
    assert abs(sh.get_time() - 1.0) < 1e-9


@pytest.mark.gpu
@pytest.mark.multigpu
def test_swift_hohenberg_two_ranks():
    """two GPUs, slabs with peer-store transposes: the gathered theta_hat after 20 steps at 256 x 256 against serial numpy"""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    env = dict(os.environ, B2_TEST_EMU="0")
    for k in dp.SWITCHES:
        env.pop(k, None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29731", os.path.join(ROOT, "tests", "sh_dist_worker.py"), "256", "256", "20"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert r.stdout.count("worst_rel_err") == 2, r.stdout[-2000:]
