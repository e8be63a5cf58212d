"""bench.py's repo arm cannot run without a GPU; its control flow and JSON contract can: tests/bench_dry_run.py runs main() on the
SIMT-emulator build with the CUDA-only torch calls stubbed (timings are meaningless and not checked)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_main_dry_run_prints_the_contract_line(tmp_path):
    from tests.emu import build_emu

    build_emu.build()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "bench_dry_run.py"), "T0", "--steps", "2", "--warmup", "3", "--no-parity",
                        "--no-cpu-baseline", "--ops-calls", "1", "--dump-outputs", str(tmp_path / "out")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline", "ops"):
        assert k in line, k
    assert line["metric"] == "Navier2D timesteps/sec" and line["unit"] == "steps/s" and line["dtype"] == "f64" and line["n_gpus"] == 1
    assert line["steps"] == 2 and line["warmup"] == 3 and line["gpu_launches"] == 2 * line["run"]["launches_per_step"]
    assert line["e2e_error"] is None and line["e2e"]["h2d_bytes_per_step"] == line["e2e"]["d2h_bytes_per_step"] > 0
    assert line["ops_error"] is None
    assert set(line["ops"]["ms_per_transform"]) == {"forward", "backward"} and set(line["ops"]["ms_per_solve"]) == {"hholtz_adi", "poisson"}
    assert line["ops"]["alg_bytes"]["forward"] == 32.0 * 65 * 65
    for key in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert key in line["roofline"], key
    import numpy as np

    for name, shape in (("temp", (63, 63)), ("velx", (63, 63)), ("vely", (63, 63)), ("pres", (65, 65))):
        a = np.load(tmp_path / "out" / f"{name}.npy")
        assert a.dtype == np.float64 and a.shape == shape and np.isfinite(a).all() and np.abs(a).max() > 0, name


def test_dump_outputs_samples_large_arrays_at_fixed_indices(tmp_path):
    """--dump-outputs: float64 files, complex as [..., 2], arrays above the cap cut to the same seeded sample on every call"""
    import numpy as np

    sys.path.insert(0, ROOT)
    import bench

    rng = np.random.default_rng(7)
    big = rng.standard_normal((1100, 1000))
    cx = rng.standard_normal((1100, 600)) + 1j * rng.standard_normal((1100, 600))
    for d in ("a", "b"):
        bench.dump_outputs({"big": big, "cx": cx, "small": big[:10, :10]}, str(tmp_path / d), 0)
    bench.dump_outputs({"big": big}, str(tmp_path / "rank1"), 1)
    assert not (tmp_path / "rank1").exists()
    got = {k: np.load(tmp_path / "a" / f"{k}.npy") for k in ("big", "cx", "small")}
    assert got["big"].shape == (bench.DUMP_VALUES_PER_ARRAY,) and got["cx"].shape == (bench.DUMP_VALUES_PER_ARRAY // 2, 2)
    assert np.array_equal(got["small"], big[:10, :10])
    assert np.isin(got["big"], big).all() and np.isin(got["cx"][:, 0], cx.real).all()
    for k, v in got.items():
        assert v.dtype == np.float64 and np.array_equal(v, np.load(tmp_path / "b" / f"{k}.npy")), k


import pytest  # noqa: E402


@pytest.mark.skipif(os.environ.get("B2_SLOW_TESTS") != "1", reason="opt-in (B2_SLOW_TESTS=1): ~1 min on 2 emulated ranks")
def test_bench_main_dry_run_two_ranks():
    """the N > 1 control flow under torchrun: distributed context, all-reduced timings, identical burst counts on every rank,
    standalone operators on slabs (--ops-multi), rank 0 alone prints"""
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29617", os.path.join(ROOT, "tests", "bench_dry_run.py"), "T0", "--gpus", "2", "--steps", "2", "--warmup", "3",
                        "--no-parity", "--no-cpu-baseline", "--ops-calls", "1", "--ops-multi"], capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    line = json.loads(lines[0])
    assert line["n_gpus"] == 2 and line["ops_error"] is None and line["e2e_error"] is None and line["gpu_launches"] == 2 * line["run"]["launches_per_step"]
