"""The banded lane operators form their coefficients in the kernel (csrc/band_coef.cuh) instead of reading uploaded vectors.

- The device functions, compiled as for the emulator (the device's Newton steps from a coarser seed), against the host's s2 and
  Base1::pv that the LU setup uses, bit for bit, for every n = 2^k + 1 from 9 to 8193 and both composite kinds: every family at
  every element, and the MatVecFdma triple as the chunk loops ask for it (pv0 carried along a chunk as pv4 of the element
  before); the reciprocal and the quotient against correctly rounded division for every index below 2^20.
- to_ortho, from_ortho, HholtzAdi and Poisson (whose solve runs the MatVecFdma) on the E = 16 / 8 / 4 compile-time layouts and
  the generic instance against the oracle.  Every transform-sized lane ends in a partial chunk (n = 2 E TPL + 1 elements,
  E + 1 pairs per thread), and the composite lengths n - 2 end inside one.
"""
import json
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")

HARNESS = r'''
#include "b200pde.cu"
#include <cstdio>
#include <cstring>

static bool same(double a, double b) { return std::memcmp(&a, &b, sizeof a) == 0; }

int main() {
  long bad = 0, checked = 0;
  auto check = [&](double got, double want, const char* what, int kind, int n, int i) {
    checked++;
    if (!same(got, want) && bad++ < 20) std::printf("MISMATCH %s kind=%d n=%d i=%d got=%.17g want=%.17g\n", what, kind, n, i, got, want);
  };
  for (int n = 9; n <= 8193; n = 2 * n - 1) {
    for (int kind : {B2_CHEB_DIRICHLET, B2_CHEB_NEUMANN}) {
      Base1 b;
      if (b.init_host(kind, n) != B2_OK) { std::printf("init_host failed\n"); return 1; }
      const int m = b.m;
      for (int i = 0; i < n + 8; i++) {
        check(band_coef(b.sten_family(), i, n), (i >= 2 && i < n) ? b.s2[i - 2] : 0.0, "sten", kind, n, i);
        check(band_coef(b.s2_family(), i, n), i < m ? b.s2[i] : 0.0, "s2", kind, n, i);
        check(band_coef(BC_PV0, i, n), i < m ? b.pv(i, 0) : 0.0, "pv0", kind, n, i);
        check(band_coef(BC_PV2, i, n), i < m - 2 ? b.pv(i, 2) : 0.0, "pv2", kind, n, i);
        check(band_coef(BC_PV4, i, n), i < m - 4 ? b.pv(i, 4) : 0.0, "pv4", kind, n, i);
        check(band_coef(BC_UNIT, i, n), 1.0, "unit", kind, n, i);
      }
      // the chunk loops: pairs p0, p0 + 1, ... of one thread, for chunk starts all along the lane
      for (int cp : {5, 9, 17})
        for (int p0 = 0; 2 * p0 < n + 4; p0 += cp) {
          BandPairs<BC_PV0, BC_PV2, BC_PV4> pv(n, 2 * p0);
          for (int t = 0; t < cp; t++) {
            const int e = 2 * (p0 + t);
            double2 k0, k1, k2;
            pv.at(e, k0, k1, k2);
            for (int h = 0; h < 2; h++) {
              const int i = e + h;
              check(h ? k0.y : k0.x, i < m ? b.pv(i, 0) : 0.0, "pair pv0", kind, n, i);
              check(h ? k1.y : k1.x, i < m - 2 ? b.pv(i, 2) : 0.0, "pair pv2", kind, n, i);
              check(h ? k2.y : k2.x, i < m - 4 ? b.pv(i, 4) : 0.0, "pair pv4", kind, n, i);
            }
          }
        }
    }
  }
  // the branch-free reciprocal and quotient against correctly rounded division for every index below 2^20 (lanes hold <= 8193)
  for (int i = 1; i < (1 << 20); i++) {
    const double r = i + 2;
    for (double d : {4.0 * r * (r - 1.0), 2.0 * (r * r - 1.0), 4.0 * r * (r + 1.0)}) check(bc_rcp(d), 1.0 / d, "rcp", 0, 0, i);
    check(bc_div((double)i, i + 2.0), (double)i / (i + 2.0), "div", 0, 0, i);
  }
  std::printf("checked %ld bad %ld\n", checked, bad);
  return bad != 0;
}
'''


def test_device_coefficients_match_host_bit_for_bit():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "harness.cpp"), os.path.join(d, "harness")
        with open(src, "w") as f:
            f.write(HARNESS)
        cc = subprocess.run(["g++", "-x", "c++", "-std=c++17", "-O2", "-DB2_EMU", "-I", EMU, "-I",
                             os.path.join(ROOT, "rustpde_mpi_b200", "csrc"), "-pthread", "-Wno-unused-function", "-o", exe, src],
                            capture_output=True, text=True)
        assert cc.returncode == 0, cc.stderr[-4000:]
        r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-4000:]
        assert " bad 0" in r.stdout and "checked 0 " not in r.stdout, r.stdout


SCRIPT = r'''
import json, sys
sys.path.insert(0, %r)
from tests import emu
emu.activate()
from tests import gpu_checks as g

out = []
for k0, n0, k1, n1 in json.loads(sys.argv[1]):
    sp = (k0, n0, k1, n1)
    out.append({"space": sp, "to_ortho": g.check_to_ortho(*sp), "from_ortho": g.check_from_ortho(*sp),
                "hholtz_adi": g.check_hholtz(*sp), "poisson": g.check_poisson(*sp)})
print("RES " + json.dumps(out))
''' % ROOT

CD, CN = 1, 2
# (environment, spaces): the lanes along axis 1 run the layout named by the case; both kinds along both axes
CASES = {
    "e16": ({"B2_E": "16"}, [(CD, 17, CD, 257), (CN, 17, CN, 257), (CN, 9, CD, 257)]),
    "e8": ({}, [(CD, 65, CD, 129), (CN, 65, CN, 129), (CD, 33, CN, 129)]),
    "e4": ({"B2_E": "4"}, [(CD, 65, CD, 129), (CN, 33, CN, 129)]),
    "generic": ({"B2_NOFAST": "1"}, [(CD, 65, CD, 129), (CN, 33, CN, 129), (CN, 17, CD, 100)]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_band_operators_against_oracle(case):
    env, spaces = CASES[case]
    r = subprocess.run([sys.executable, "-c", SCRIPT, json.dumps(spaces)], capture_output=True, text=True, timeout=1800, cwd=ROOT,
                       env=dict({k: v for k, v in os.environ.items() if k not in ("B2_E", "B2_LN", "B2_NOFAST")}, **env))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RES ")][-1][4:])
    bad = [(x["space"], k, v) for x in res for k, v in x.items() if k != "space" and not v < 1e-12]
    assert not bad, bad
