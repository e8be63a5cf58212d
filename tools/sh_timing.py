"""SwiftHohenberg2D.update: ms per step on c2c n x r2c n, one GPU, CUDA events, alternated in the same process with the same
step composed from existing C-ABI calls (copy, 3-pass backward, two pointwise products, 2-pass forward, axpy, pointwise
division: 9 kernels), once with the Hermitian fix of the ky = 0 column done on the host (a full theta_hat download and upload per
step, as a user of the plain field operators has to) and once without it.

  python tools/sh_timing.py [--root TREE] [--warmup W] [--seconds S] [--sizes 512,2048,4096]

Each variant is warmed up, then timed over at least S seconds of steps (default 1), three times in alternation; the median is
printed.  The achieved rate is over the step's algorithmic bytes: nine array transfers of the padded spectrum (8 x P0 x P1 bytes
each): pass 1 read + write, pass 2 read + write, pass 3 read + write, pass 4 reads two arrays and writes one.  The card's name,
power limit and maximum SM clock are printed first.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R, DT, L = 0.35, 0.02, 20.0   # examples/swift_hohenberg_2d.rs main()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e!r})"
    return q


class Composed:
    """update_implicit from the field operators and array calls of the C ABI (the step of tests/test_gpu_doubly_periodic.py)"""

    def __init__(self, b2, ctx, theta0, host_fix):
        import numpy as np

        from rustpde_mpi_b200._lib import check, lib

        self.np, self.check, self.lib, self.host_fix = np, check, lib, host_fix
        nx, ny = theta0.shape
        self.f = b2.Field2(b2.Space2((b2.FOURIER_C2C, nx), (b2.FOURIER_R2C, ny), ctx=ctx))
        self.v, self.vhat = (self._borrow(b2, w) for w in (0, 1))
        self.sq = b2.DeviceArray(self.f.space, b2.PHYSICAL)
        self.rhs = b2.DeviceArray(self.f.space, b2.SPECTRAL)
        kx = np.fft.fftfreq(nx, 1.0 / nx)[:, None] / L
        ky = np.arange(ny // 2 + 1)[None, :] / L
        q = 1.0 - kx ** 2 - ky ** 2
        inv = 1.0 / (1.0 - R * DT + DT * q * q)
        self.minv = b2.DeviceArray(self.f.space, b2.SPECTRAL).set(inv + 1j * inv)
        self.f.v = theta0
        self.f.forward()

    def _borrow(self, b2, which):
        h = C.c_void_p()
        self.check(self.lib().b2_field_array(self.f._h, which, C.byref(h)))
        return b2.DeviceArray(self.f.space, b2.PHYSICAL if which == 0 else b2.SPECTRAL, handle=h, owner=False)

    def step(self):
        check, lib = self.check, self.lib
        check(lib().b2_array_copy(self.rhs._h, self.vhat._h))
        self.f.backward()
        check(lib().b2_array_combine(self.sq._h, self.v._h, self.v._h, 0, C.c_double(1.0)))
        check(lib().b2_array_combine(self.v._h, self.v._h, self.sq._h, 0, C.c_double(1.0)))
        self.f.forward()
        self.rhs.axpy(-DT, self.vhat)
        check(lib().b2_array_combine(self.vhat._h, self.rhs._h, self.minv._h, 0, C.c_double(1.0)))
        if self.host_fix:
            vh = self.f.vhat
            vh[0, 0] = 0
            n = vh.shape[0]
            i = self.np.arange(1, (n - 1) // 2 + 1)
            vh[n - i, 0] = self.np.conj(vh[i, 0])
            self.f.vhat = vh


def timed(ctx, step, k):
    ctx.timer_start()
    for _ in range(k):
        step()
    return ctx.timer_stop() / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--sizes", default="512,2048,4096")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np

    import rustpde_mpi_b200 as b2

    ctx = b2.Context(0)
    print(f"card (name, power limit, max SM clock): {card()}", flush=True)
    print(f"library: {b2.LIB_PATH}", flush=True)
    for n in (int(s) for s in args.sizes.split(",")):
        sh = b2.SwiftHohenberg2D(n, n, R, DT, L, ctx=ctx)
        theta0 = sh.theta.v
        variants = {"SwiftHohenberg2D.update": lambda s=sh: s.update(1)}
        objs = []
        for fix in (False, True):
            c = Composed(b2, ctx, theta0, fix)
            objs.append(c)
            variants[f"composed, {'host fix' if fix else 'no fix'}"] = c.step
        reps = {}
        for name, step in variants.items():
            for _ in range(args.warmup):
                step()
            ms = timed(ctx, step, 3)
            reps[name] = max(3, int(np.ceil(args.seconds * 1e3 / ms)))
        ms = {name: [] for name in variants}
        for _ in range(3):   # alternate the variants
            for name, step in variants.items():
                ms[name].append(timed(ctx, step, reps[name]))
        p = -(-(n + 2) // 4) * 4
        gb = 9 * 8 * p * p / 1e9
        lay = tuple(tuple(sh.space.layout(o)[k] for k in ("E", "LN", "TPL", "fast")) for o in (0, 1))
        print(f"c2c {n} x r2c {n}  layouts (y, x) {lay}  launches per step {sh.launches_per_step()}  "
              f"algorithmic bytes per step {gb * 1e3:.1f} MB", flush=True)
        for name in variants:
            med = float(np.median(ms[name]))
            runs = ", ".join(f"{m:.4f}" for m in ms[name])
            print(f"  {name:26s} {med:9.4f} ms/step  ({reps[name]} steps x 3: {runs})  {gb / med * 1e3:7.1f} GB/s over the 4-pass bytes",
                  flush=True)
        sh.close()
        for c in objs:
            for o in (c.minv, c.rhs, c.sq, c.f):
                o.close()
            c.f.space.close()


if __name__ == "__main__":
    main()
