"""Transform sizes 3 * 2^k + 1 against the power-of-two sizes around them, on one GPU in one process.

  python tools/size_sweep.py [--steps K]

Prints, with the card's name and power limit:
  - ms per step of confined rbc (Ra 1e7, dt 1e-3) at 2049^2, 3073^2 and 4097^2, split into lane passes and the Poisson GEMMs;
  - the same at 4097^2 under B2_NOFAST=1: the generic lane-kernel instances that 3073^2 runs on, so that the cost per point of
    the two sizes compares the same code;
  - periodic 3072 x 1537 next to 4096 x 2049;
  - ms per standalone forward and backward on ch x ch at 3073^2 and 4097^2.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import rustpde_mpi_b200 as b2  # noqa: E402

STEPS = [  # (name, nx, ny, periodic, environment at space creation)
    ("confined 2049x2049", 2049, 2049, False, {}),
    ("confined 3073x3073", 3073, 3073, False, {}),
    ("confined 4097x4097", 4097, 4097, False, {}),
    ("confined 4097x4097 B2_NOFAST=1", 4097, 4097, False, {"B2_NOFAST": "1"}),
    ("periodic 3072x1537", 3072, 1537, True, {}),
    ("periodic 4096x2049", 4096, 2049, True, {}),
]
TRANSFORMS = [("ch x ch 3073x3073", 3073), ("ch x ch 4097x4097", 4097)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e!r})"
    return q


def with_env(env, make):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return make()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    ctx = b2.Context(0)
    print(f"card: {card()}", flush=True)
    for name, nx, ny, per, env in STEPS:
        eig = None if per else b2.poisson_eig(b2.CHEB_NEUMANN, nx, 1.0)
        nav = with_env(env, lambda: b2.Navier2D(nx, ny, 1e7, 1.0, 1e-3, 1.0, "rbc", periodic=per, ctx=ctx, pois_eig=eig))
        sp = with_env(env, lambda: b2.Space2((b2.FOURIER_R2C if per else b2.CHEB_DIRICHLET, nx), (b2.CHEB_DIRICHLET, ny), ctx=ctx))
        lay = [tuple(sp.layout(o)[k] for k in ("E", "LN", "TPL", "fast")) for o in (0, 1)]
        sp.close()
        nav.set_mode(1)
        nav.update(args.warmup)
        ctx.sync()
        ctx.timer_start()
        nav.update(args.steps)
        ms = ctx.timer_stop() / args.steps
        ctx.profile(True)
        nav.update(3)
        gemm = ctx.profile(False) / 3
        print(f"{name:34s} {ms:8.3f} ms/step  lane {ms - gemm:8.3f}  gemm {gemm:7.3f}  ns/point {ms * 1e6 / (nx * ny):6.3f}  "
              f"layouts (E, LN, TPL, fast) {lay}  div {nav.div_norm():.3e}", flush=True)
        nav.close()
    for name, n in TRANSFORMS:
        f = b2.Field2(b2.Space2((b2.CHEBYSHEV, n), (b2.CHEBYSHEV, n), ctx=ctx))
        f.v = np.random.default_rng(0).uniform(-1.0, 1.0, (n, n))
        out = {}
        for op in ("forward", "backward"):
            call = getattr(f, op)
            for _ in range(args.warmup):
                call()
            ctx.sync()
            ctx.timer_start()
            for _ in range(args.calls):
                call()
            out[op] = ctx.timer_stop() / args.calls
        print(f"{name:34s} forward {out['forward']:7.3f} ms  backward {out['backward']:7.3f} ms", flush=True)
        f.close()


if __name__ == "__main__":
    main()
