"""Run every parity check and print the errors (no early abort) -- first-light tool on a new GPU."""
import sys
import time
import traceback

import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import gpu_checks as g  # noqa: E402

SPACES = [(1, 65, 1, 65), (2, 129, 1, 65), (0, 65, 0, 129), (2, 129, 2, 129), (4, 64, 1, 65), (4, 128, 0, 129), (4, 256, 2, 65), (1, 257, 1, 513)]


def run(name, fn, *a, **k):
    t = time.time()
    try:
        r = fn(*a, **k)
        flag = ""
        if isinstance(r, dict):
            flag = "" if max(r.values()) < g.TOL else "  <-- FAIL"
        else:
            flag = "" if r < g.TOL else "  <-- FAIL"
        print(f"{name:60s} {r}  ({time.time()-t:.1f}s){flag}", flush=True)
    except Exception as e:  # noqa: BLE001
        print(f"{name:60s} EXC {type(e).__name__}: {e}", flush=True)
        traceback.print_exc()


if __name__ == "__main__":
    quick = "--quick" in sys.argv
    for sp in SPACES[: 3 if quick else None]:
        tag = f"{g.KIND_NAME[sp[0]]}{sp[1]}x{g.KIND_NAME[sp[2]]}{sp[3]}"
        run(f"layout    {tag}", g.check_roundtrip_layout, *sp)
        run(f"to_ortho  {tag}", g.check_to_ortho, *sp)
        run(f"from_ortho {tag}", g.check_from_ortho, *sp)
        run(f"backward  {tag}", g.check_backward, *sp)
        run(f"forward   {tag}", g.check_forward, *sp)
        for d in ((1, 0), (0, 1), (2, 0), (0, 2)):
            run(f"gradient{d} {tag}", g.check_gradient, *sp, d)
        if sp[0] != 0 and sp[2] != 0:
            run(f"hholtz    {tag}", g.check_hholtz, *sp)
    for sp in [(2, 65, 2, 65), (2, 129, 2, 65), (4, 64, 2, 65), (4, 128, 2, 129)]:
        tag = f"{g.KIND_NAME[sp[0]]}{sp[1]}x{g.KIND_NAME[sp[2]]}{sp[3]}"
        run(f"poisson   {tag}", g.check_poisson, *sp)
    run("navier confined 65x65 1 step", g.check_navier, 65, 65, 1)
    run("navier confined 65x65 10 steps", g.check_navier, 65, 65, 10)
    run("navier periodic 64x65 1 step", g.check_navier, 64, 65, 1, True)
    run("navier periodic 64x65 10 steps", g.check_navier, 64, 65, 10, True)
    if not quick:
        run("navier confined 129x129 100 steps (C1)", g.check_navier, 129, 129, 100)
        run("navier confined 257x257 random 3 steps", g.check_navier, 257, 257, 3, False, 1e7, 1e-3, "random")
