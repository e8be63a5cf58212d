"""Standalone operators of doubly periodic spaces: ms per call on c2c n x r2c n, one GPU, CUDA events, with r2c n x cd (n + 1)
forward / backward as the yardstick (the Navier2D periodic transforms: two lane passes each).

  python tools/dp_timing.py [--root TREE] [--calls K] [--warmup W]

--root imports rustpde_mpi_b200 from another checkout, so that two builds can be timed alternately on the same card.  Prints the
card's name and power limit, then per size the lane layouts (along y, along x), ms per call and the achieved rate over the passes'
algorithmic bytes: each lane pass reads and writes the whole padded array once (2 x 8 x P0 x P1 bytes per pass; forward,
gradient, HholtzAdi and Poisson run 2 passes, the doubly periodic backward 3).
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (512, 1024, 2048, 4096)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e!r})"
    return q


def timed(ctx, call, calls):
    ctx.timer_start()
    for _ in range(calls):
        call()
    return ctx.timer_stop() / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np

    import rustpde_mpi_b200 as b2

    ctx = b2.Context(0)
    print(f"card: {card()}", flush=True)
    print(f"library: {b2.LIB_PATH}", flush=True)
    runs = []
    for n in SIZES:   # build and warm every shape first
        rng = np.random.default_rng(n)
        dp = b2.Field2(b2.Space2((b2.FOURIER_C2C, n), (b2.FOURIER_R2C, n), ctx=ctx))
        dp.v = rng.uniform(-1.0, 1.0, (n, n))
        ortho, spec = b2.DeviceArray(dp.space, b2.ORTHO), b2.DeviceArray(dp.space, b2.SPECTRAL)
        adi, pois = b2.HholtzAdi(dp, [0.02, 0.03]), b2.Poisson(dp, [1.0, 1.0])
        ref = b2.Field2(b2.Space2((b2.FOURIER_R2C, n), (b2.CHEB_DIRICHLET, n + 1), ctx=ctx))
        ref.v = rng.uniform(-1.0, 1.0, (n, n + 1))
        ops = {
            "forward": dp.forward, "backward": dp.backward,
            "gradient(1,0)": lambda f=dp, o=ortho: f.gradient((1, 0), out=o),
            "gradient(0,1)": lambda f=dp, o=ortho: f.gradient((0, 1), out=o),
            "hholtz_adi": lambda s=adi, i=ortho, o=spec: s.solve(i, out=o),
            "poisson": lambda s=pois, i=ortho, o=spec: s.solve(i, out=o),
            "r2c x cd forward": ref.forward, "r2c x cd backward": ref.backward,
        }
        for _ in range(args.warmup):
            for call in ops.values():
                call()
        lay = tuple(tuple(dp.space.layout(o)[k] for k in ("E", "LN", "TPL", "fast")) for o in (0, 1))
        runs.append((n, lay, ops, (dp, ref, ortho, spec, adi, pois)))
    ctx.sync()
    for n, lay, ops, _ in runs:
        p0, p1 = -(-(n + 2) // 4) * 4, -(-(n + 2) // 4) * 4   # padded rows: the half spectra of n + 2 reals on both axes
        pass_gb = 2 * 8 * p0 * p1 / 1e9
        ref_gb = 2 * 8 * (-(-(n + 2) // 4) * 4) * (-(-(n + 1) // 4) * 4) / 1e9
        print(f"c2c {n} x r2c {n}  layouts (y, x) {lay}", flush=True)
        for name, call in ops.items():
            ms = timed(ctx, call, args.calls)
            gb = ref_gb * 2 if name.startswith("r2c") else pass_gb * (3 if name == "backward" else 2)
            print(f"  {name:18s} {ms:8.4f} ms  {gb / ms * 1e3:7.1f} GB/s  ({gb * 1e3:.1f} MB)", flush=True)
    for _, _, _, objs in runs:
        for o in objs:
            o.close()


if __name__ == "__main__":
    main()
