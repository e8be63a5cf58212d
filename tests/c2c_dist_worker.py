"""Worker of the multi-rank tests of tests/test_emu_c2c_fft.py: one process per rank (torch.distributed, gloo, emulator build), a
FourierC2c x ChebDirichlet space on slabs; forward, backward and Poisson against the serial oracle on every rank.

  c2c_dist_worker.py n ny fast    fast = the expected PassCfg::fast of the c2c lanes (1: cfft_fast, 0: a generic instance)"""
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
    from oracle import rustpde_oracle as o

    dist.init_process_group(backend="gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    n, ny, fast = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
    ctx = b2.Context.distributed(0, heap_bytes=(200 * (2 * n + 16) * (ny + 16) * 8) // world + (8 << 20))
    fo = o.Field2(o.Space2(o.fourier_c2c(n), o.cheb_dirichlet(ny)))
    fg = b2.Field2(b2.Space2(b2.fourier_c2c(n), b2.cheb_dirichlet(ny), ctx=ctx))
    lay = fg.space.layout(1)
    rng = np.random.default_rng(9)
    vg = rng.standard_normal((n, ny)) + 1j * rng.standard_normal((n, ny))
    errs = {}
    fg.v = vg[fg.local_slice(b2.PHYSICAL)]
    fg.forward()
    fo.v = vg; fo.forward()
    got = fg.all_gather_spectral()
    errs["forward"] = float(np.abs(got - fo.vhat).max() / np.abs(fo.vhat).max())
    fg.backward(); fo.backward()
    errs["backward"] = float(np.abs(fg.all_gather_physical() - fo.v).max() / np.abs(fo.v).max())
    so, sg = o.Poisson(fo, [1.0, 1.0]), b2.Poisson(fg, [1.0, 1.0])
    sh = fo.space.to_ortho(fo.vhat).shape
    rhs = rng.standard_normal(sh) + 1j * rng.standard_normal(sh)
    inp = b2.DeviceArray(fg.space, b2.ORTHO)
    r0, cnt = inp.local_rows()
    inp.set(rhs[r0:r0 + cnt])
    x, xo = ctx.all_gather_rows(sg.solve(inp).get()), so.solve(rhs)
    x[0, 0] = 0; xo[0, 0] = 0   # the shifted-singular mode is removed by the caller (navier_eq.rs:161)
    errs["poisson"] = float(np.abs(x - xo).max() / np.abs(xo).max())
    worst = max(errs.values())
    print(f"rank {rank}/{world}: c2c {n} x cd {ny}, layout {lay}, {errs} worst_rel_err={worst:.3e}", flush=True)
    assert worst < 1e-10, errs
    assert lay["fast"] == fast, lay
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
