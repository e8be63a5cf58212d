// Coefficients of the banded lane operators, formed where they are used (included by lane_kernel.cuh).
//
// Every coefficient of the composite bases' banded mat-vecs is a closed-form function of the element index and the base size n
// (m = n - 2 composite coefficients), so the lane kernel computes it instead of streaming a coefficient vector:
//   to_ortho stencil   y_j = x_j + s_{j-2} x_{j-2}                   BC_STEN_*: s_{j-2} for 2 <= j < n, else 0
//   S^T of from_ortho  y_k = x_k + s_k x_{k+2}                       BC_S2_*:   s_k for k < m, else 0
//   MatVecFdma of the preconditioner pinv (Base1::pv, r = i + 2)
//     y_i = pv0_i x_i + pv2_i x_{i+2} + pv4_i x_{i+4}
//     pv0_i = 1 / (4 r (r - 1)) (0.25 at r = 2), i < m;  pv2_i = -1 / (2 (r^2 - 1)), i < m - 2;  pv4_i = 1 / (4 r (r + 1)), i < m - 4
// with s = -1 (ChebDirichlet) or s_k = -(k / (k + 2))^2 (ChebNeumann).  Every denominator is an integer below 2^53, so it is exact in
// double, and the correctly rounded reciprocal (quotient) is the value the host computes with 1.0 / x (k / (k + 2.0)): the kernel
// reproduces the host's coefficients bit for bit.  The reciprocal is branch-free (bc_rcp): the library's __drcp_rn and double
// division branch to a slow path, which puts every reciprocal of an unrolled chunk loop into a block of its own and serialises
// their latencies (the folded E = 8 solve of C2 took 1.8x as long in its forward pass); and its seed is the one MUFU operation
// of the hardware's double approximation, not a single-precision reciprocal with two conversions, which share MUFU's
// quarter-rate pipe (C4 band ops 9.1k -> 11.7k cycles with them).
#pragma once

// family of one term of a banded op (4 bits per term in LaneOp::i2, see band_fams)
enum BandCoefFamily {
  BC_ABSENT = 0,   // no term
  BC_UNIT = 1,     // coefficient 1
  BC_STEN_D = 2, BC_STEN_N = 3,   // to_ortho stencil at output element j (Dirichlet / Neumann)
  BC_S2_D = 4, BC_S2_N = 5,       // s_k at element k (S^T)
  BC_PV0 = 6, BC_PV2 = 7, BC_PV4 = 8
};
// LaneOp::i2 of OP_BAND / OP_BANDC / OP_PREBAND: families of terms 0..2 in bits 0..11, base size n from bit 12
static inline __host__ __device__ int band_fams(int f0, int f1, int f2, int n) { return f0 | (f1 << 4) | (f2 << 8) | (n << 12); }
#define B2_BAND_TERMS(f0, f1, f2) ((f0) | ((f1) << 4) | ((f2) << 8))
__device__ __forceinline__ int band_terms(int i2) { return i2 & 0xfff; }
__device__ __forceinline__ int band_fam(int i2, int m) { return (i2 >> (4 * m)) & 15; }
__device__ __forceinline__ int band_n(int i2) { return i2 >> 12; }

// 1 / x, correctly rounded for the integer denominators x < 2^53 of the families below: an approximate reciprocal and two Newton
// steps, whose residuals fma(-x, y, 1) are exact; no branch.  The emulator build's seed keeps only 20 significant bits of 1 / x,
// coarser than the hardware's rcp.approx, and with it bc_rcp equals 1.0 / x for every index below 2^20
// (tests/test_emu_band_coefficients.py; lanes hold at most 8193 elements)
__device__ __forceinline__ double bc_rcp_seed(double x) {
#ifdef B2_EMU
  int e;
  const double m = std::frexp(1.0 / x, &e);
  return std::ldexp(std::floor(std::ldexp(m, 20)), e - 20);
#else
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  return y;
#endif
}
__device__ __forceinline__ double bc_rcp(double x) {
  double y = bc_rcp_seed(x);
  y = fma(y, fma(-x, y, 1.0), y);
  return fma(y, fma(-x, y, 1.0), y);
}
// a / b correctly rounded from the correctly rounded reciprocal: one correction of the quotient with its exact residual
__device__ __forceinline__ double bc_div(double a, double b) {
  const double y = bc_rcp(b), q = a * y;
  return fma(fma(-q, b, a), y, q);
}
__device__ __forceinline__ double bc_s2n(int k) { const double a = bc_div((double)k, k + 2.0); return -a * a; }
// pv0 without its range: i == 0 (r = 2) is the one end rule
__device__ __forceinline__ double bc_pv0(int i) { const double r = i + 2; return i == 0 ? 0.25 : bc_rcp(4.0 * r * (r - 1.0)); }
__device__ __forceinline__ double bc_pv2(int i) { const double r = i + 2; return -bc_rcp(2.0 * (r * r - 1.0)); }

// coefficient of family f at element i of a base of size n
__device__ __forceinline__ double band_coef(int f, int i, int n) {
  switch (f) {
    case BC_UNIT: return 1.0;
    case BC_STEN_D: return (i >= 2 && i < n) ? -1.0 : 0.0;
    case BC_STEN_N: return (i >= 2 && i < n) ? bc_s2n(i - 2) : 0.0;
    case BC_S2_D: return (i < n - 2) ? -1.0 : 0.0;
    case BC_S2_N: return (i < n - 2) ? bc_s2n(i) : 0.0;
    case BC_PV0: return (i < n - 2) ? bc_pv0(i) : 0.0;
    case BC_PV2: return (i < n - 4) ? bc_pv2(i) : 0.0;
    case BC_PV4: return (i < n - 6) ? bc_pv0(i + 1) : 0.0;   // 1 / (4 r (r + 1)) = pv0 of the next element
  }
  return 0.0;
}

// Coefficients (k0, k1, k2) of the term families F0, F1, F2 for the element pairs (e, e + 1), e = 2p, asked for with increasing p
// starting at e0.  The MatVecFdma triple carries pv0 of the next element along the chunk (pv4_i = pv0_{i+1}): two reciprocals per
// element instead of three.
template <int F0, int F1, int F2> struct BandPairs {
  int n;
  __device__ __forceinline__ BandPairs(int n_, int) : n(n_) {}
  __device__ __forceinline__ void at(int e, double2& k0, double2& k1, double2& k2) {
    k0 = make_double2(band_coef(F0, e, n), band_coef(F0, e + 1, n));
    k1 = make_double2(band_coef(F1, e, n), band_coef(F1, e + 1, n));
    k2 = make_double2(band_coef(F2, e, n), band_coef(F2, e + 1, n));
  }
};
template <> struct BandPairs<BC_PV0, BC_PV2, BC_PV4> {
  int n;
  double c;   // pv0 of element e (no range applied)
  __device__ __forceinline__ BandPairs(int n_, int e0) : n(n_), c(bc_pv0(e0)) {}
  __device__ __forceinline__ void at(int e, double2& k0, double2& k1, double2& k2) {
    const double a = bc_pv0(e + 1), b = bc_pv0(e + 2);
    k0 = make_double2(e < n - 2 ? c : 0.0, e + 1 < n - 2 ? a : 0.0);
    k1 = make_double2(e < n - 4 ? bc_pv2(e) : 0.0, e + 1 < n - 4 ? bc_pv2(e + 1) : 0.0);
    k2 = make_double2(e < n - 6 ? a : 0.0, e + 1 < n - 6 ? b : 0.0);
    c = b;
  }
};
