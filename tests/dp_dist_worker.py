"""Worker of the multi-rank test of tests/test_emu_doubly_periodic.py: one process per rank (torch.distributed, gloo, emulator
build), a fourier_c2c x fourier_r2c space on slabs; gathered forward, backward, gradient and Poisson against the serial oracle on
every rank.

  dp_dist_worker.py nx ny"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import emu

    emu.activate()
    import numpy as np
    import torch.distributed as dist

    import rustpde_mpi_b200 as b2
    from tests import test_gpu_doubly_periodic as t

    dist.init_process_group(backend="gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    nx, ny = int(sys.argv[1]), int(sys.argv[2])
    ctx = b2.Context.distributed(0, heap_bytes=(200 * (nx + 16) * (ny + 16) * 8) // world + (8 << 20))
    fg = b2.Field2(b2.Space2(b2.fourier_c2c(nx), b2.fourier_r2c(ny), ctx=ctx))
    space = t.oracle_space(nx, ny)
    rng = np.random.default_rng(9)
    v = rng.uniform(-1, 1, (nx, ny))
    errs = {}
    fg.v = v[fg.local_slice(b2.PHYSICAL)]
    fg.forward()
    errs["forward"] = t.relerr(fg.all_gather_spectral(), np.fft.rfft2(v))
    a = t.rand_spec(nx, ny, rng)
    fg.vhat = a[fg.local_slice(b2.SPECTRAL)]
    fg.backward()
    errs["backward"] = t.relerr(fg.all_gather_physical(), np.fft.irfft2(a, s=(nx, ny)))
    for d in ((1, 0), (0, 1), (3, 2)):
        errs[f"gradient{d}"] = t.relerr(ctx.all_gather_rows(fg.gradient(d, (1.3, 0.7)).get()), space.gradient(a, d, (1.3, 0.7)))
    _, _, so, _ = t.solver_refs(nx, ny)[1]
    inp = b2.DeviceArray(fg.space, b2.ORTHO)
    r0, cnt = inp.local_rows()
    inp.set(a[r0:r0 + cnt])
    errs["poisson"] = t.solve_err("poisson", ctx.all_gather_rows(b2.Poisson(fg, [1.0, 1.0]).solve(inp).get()), so.solve(a))
    worst = max(errs.values())
    print(f"rank {rank}/{world}: c2c {nx} x r2c {ny}, layouts {fg.space.layout(0)} {fg.space.layout(1)}, {errs} "
          f"worst_rel_err={worst:.3e}", flush=True)
    assert worst < t.TOL, errs
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
