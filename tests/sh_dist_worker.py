"""Worker of the multi-rank SwiftHohenberg2D tests: one process per rank (torch.distributed), the model on slabs of a fourier_c2c x
fourier_r2c space; the gathered theta_hat after some steps against the serial numpy steps on every rank.

  CPU (tests/test_emu_swift_hohenberg.py):  B2_TEST_EMU=1, backend gloo, library = SIMT-emulator build
  GPU (tests/test_gpu_swift_hohenberg.py):  backend nccl/gloo, library = CUDA build, one GPU per rank

  sh_dist_worker.py nx ny steps"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    use_emu = os.environ.get("B2_TEST_EMU", "0") == "1"
    if use_emu:
        from tests import emu

        emu.activate()
    import numpy as np
    import torch
    import torch.distributed as dist

    import rustpde_mpi_b200 as b2
    from tests import test_gpu_doubly_periodic as t

    dist.init_process_group(backend="gloo" if use_emu else "cpu:gloo,cuda:nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    device = 0 if use_emu else int(os.environ.get("LOCAL_RANK", rank))
    if not use_emu:
        torch.cuda.set_device(device)
    nx, ny, steps = (int(v) for v in sys.argv[1:4])
    ctx = b2.Context.distributed(device, heap_bytes=(40 * (nx + 16) * (ny + 16) * 8) // world + (8 << 20))
    sh = b2.SwiftHohenberg2D(nx, ny, t.SH_R, t.SH_DT, t.SH_L, ctx=ctx, seed=7)
    theta0 = sh.theta.all_gather_physical()
    sh.update(steps)
    got = sh.theta.all_gather_spectral()
    ref = t.sh_numpy(theta0, steps)
    yard = t.relerr(t.sh_numpy(t.perturbed(theta0, 3), steps), ref)
    err = t.relerr(got, ref)
    bound = max(t.TOL, 10.0 * yard)
    print(f"rank {rank}/{world}: SwiftHohenberg2D c2c {nx} x r2c {ny}, {steps} steps, {sh.launches_per_step()} passes per step, "
          f"yardstick {yard:.2e} worst_rel_err={err:.3e}", flush=True)
    assert err < bound, (err, bound)
    nref = np.sqrt(np.sum(np.abs(ref) ** 2)) / ref.size   # norm_l2_c64, a collective over the ranks
    assert abs(sh.norm() - nref) < 1e-10 * nref, (sh.norm(), nref)
    sh.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
