"""Standalone FourierC2c transforms: ms per forward and backward on c2c n x cd 1025, one GPU, CUDA events.

  python tools/c2c_timing.py [--root TREE] [--calls K] [--warmup W]

--root imports rustpde_mpi_b200 from another checkout (e.g. a build of an older commit), so that two builds can be timed
alternately on the same card.  Prints the card's name and power limit, then per size the lane layout along axis 0, ms per call
and the achieved rate over the algorithmic bytes of a transform: its two lane passes each read and write the whole padded
array once (4 x 8 x rows x columns bytes).
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (256, 512, 640, 768, 1024)
NY = 1025


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e!r})"
    return q


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
    fields = {}
    for n in SIZES:   # warm every shape first
        f = b2.Field2(b2.Space2((b2.FOURIER_C2C, n), (b2.CHEB_DIRICHLET, NY), ctx=ctx))
        rng = np.random.default_rng(n)
        f.v = rng.uniform(-1.0, 1.0, (n, NY)) + 1j * rng.uniform(-1.0, 1.0, (n, NY))
        for _ in range(args.warmup):
            f.forward()
            f.backward()
        fields[n] = f
    ctx.sync()
    for n, f in fields.items():
        lay = tuple(f.space.layout(1)[k] for k in ("E", "LN", "TPL", "fast"))
        rows, cols = 2 * n, -(-NY // 4) * 4
        gbytes = 4 * 8 * rows * cols / 1e9
        out = {}
        for op in ("forward", "backward"):
            call = getattr(f, op)
            ctx.timer_start()
            for _ in range(args.calls):
                call()
            out[op] = ctx.timer_stop() / args.calls
        print(f"c2c {n:5d} x cd {NY}  layout {lay}  forward {out['forward']:8.4f} ms ({gbytes / out['forward'] * 1e3:7.1f} GB/s)  "
              f"backward {out['backward']:8.4f} ms ({gbytes / out['backward'] * 1e3:7.1f} GB/s)  bytes/transform {gbytes * 1e9:.4g}",
              flush=True)
    for f in fields.values():
        f.close()


if __name__ == "__main__":
    main()
