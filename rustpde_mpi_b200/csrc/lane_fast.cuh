// Compile-time-geometry versions of the hot lane operators (included by lane_kernel.cuh).
//
// The lane operators are issue-bound: in the generic versions two thirds of the instructions are integer
// index arithmetic (tile-layout address of element i, range clamps).  For transform-sized lanes the
// geometry is fixed by (E, TPL): N = 2*E*TPL, so every shared-memory address here is ONE runtime base per
// thread plus a compile-time offset that folds into the LDS/STS immediate, loops have constant trip counts,
// and the only predicates left are the ones the mathematics needs (first / last element of a lane).
//   pairs:    pix(a + K) = pix(a) + (K/2) * 2^LSH       for even K
//   elements: eix(a + K) = eix(a) + (K/4) * 2^(LSH+1)   for K a multiple of 4
#pragma once

template <int LN, int K> struct POff { static_assert(K % 2 == 0, "even pair offsets only"); static constexpr int v = (K / 2) * (1 << Lay<LN>::LSH); };
template <int LN, int K> struct EOff { static_assert(K % 4 == 0, "element offsets in tiles only"); static constexpr int v = (K / 4) * (1 << (Lay<LN>::LSH + 1)); };

// ---------------------------------------------------------------------------------------------
// FFT: one Stockham pass with compile-time radix R, stride Ns and swizzle handling (see fft_stage).
// ---------------------------------------------------------------------------------------------
template <int E, int R, int Ns, int LN, int TPL, bool SWZI, bool SWZO>
__device__ __forceinline__ void fstage(double2* __restrict__ wl, int q, const cplx* __restrict__ tw) {
  constexpr int NB = E / R, LE = Log2<E>::v, Nc = E * TPL, stride = Nc / R, LSH = Lay<LN>::LSH;
  constexpr int RS = POff<LN, stride>::v;
  static_assert(!SWZI || stride % (1 << LE) == 0, "swizzled reads need stride to be a multiple of E");
  cplx v[E];
  cplx w1[NB];
#pragma unroll
  for (int b = 0; b < NB; b++) {
    const int j = q + b * TPL;
    if (Ns > 1) w1[b] = ldg(tw + (j & (Ns - 1)) * (stride / Ns));   // issued ahead of the barrier
    if (!SWZI) {
      const int base = Lay<LN>::pix(j);
#pragma unroll
      for (int r = 0; r < R; r++) v[b * R + r] = wl[base + r * RS];
    } else {   // point i = j + r*stride was written at i ^ ((i >> LE) & 1)
      const int s0 = (j >> LE) & 1;
      const int b0 = Lay<LN>::pix(j ^ s0), b1 = Lay<LN>::pix(j ^ (s0 ^ 1));
#pragma unroll
      for (int r = 0; r < R; r++) v[b * R + r] = wl[(((r * (stride >> LE)) & 1) ? b1 : b0) + r * RS];
    }
  }
  __syncthreads();
#pragma unroll
  for (int b = 0; b < NB; b++) {
    const int j = q + b * TPL;
    if (Ns > 1) Twid<R>::run(v + b * R, w1[b]);
    Dft<R>::run(v + b * R);
    if (Ns == 1) {          // results go to points j*R + r (R consecutive points)
      const int hb = (j * (R / 2)) << LSH;
      if (SWZO) {
        const int s = j & 1, be = hb + s, bo = hb + 1 - s;
#pragma unroll
        for (int r = 0; r < R; r++) wl[((r & 1) ? bo : be) + ((r >> 1) << LSH)] = v[b * R + r];
      } else {
#pragma unroll
        for (int r = 0; r < R; r++) wl[hb + ((r >> 1) << LSH) + (r & 1)] = v[b * R + r];
      }
    } else {                // points j0 + r*Ns, j0 = (j - k) * R + k, k = j mod Ns
      const int k = j & (Ns - 1);
      const int base = Lay<LN>::pix((j - k) * R + k);
#pragma unroll
      for (int r = 0; r < R; r++) wl[base + r * POff<LN, (Ns > 1 ? Ns : 2)>::v] = v[b * R + r];
    }
  }
  __syncthreads();
}

template <int E, int LN, int TPL, int Ns, bool SWZ> struct FftRest {   // the passes after the first one
  static __device__ __forceinline__ void run(double2* __restrict__ wl, int q, const cplx* __restrict__ tw) {
    constexpr int rem = (E * TPL) / Ns;
    if constexpr (rem >= E) {
      fstage<E, E, Ns, LN, TPL, SWZ, false>(wl, q, tw);
      FftRest<E, LN, TPL, Ns * E, false>::run(wl, q, tw);
    } else if constexpr (rem > 1) {
      fstage<E, rem, Ns, LN, TPL, SWZ, false>(wl, q, tw);
    }
  }
};
template <int E, int LN, int TPL>
__device__ __forceinline__ void lane_fft_fast(double* __restrict__ W, int l, int q, const cplx* __restrict__ tw) {
  double2* wl = reinterpret_cast<double2*>(W) + 2 * l;
  fstage<E, E, 1, LN, TPL, false, true>(wl, q, tw);
  FftRest<E, LN, TPL, E, true>::run(wl, q, tw);
}

// ---------------------------------------------------------------------------------------------
// Chebyshev transform (see op_dct for the algorithm), N = 2*E*TPL.
// ---------------------------------------------------------------------------------------------
template <int E, int LN, int TPL>
__device__ __noinline__ void dct_fast(const LaneOp& op, double* __restrict__ W, double* scratch, unsigned long long* prof) {
  PhaseClock pc(prof);
  constexpr int M = E * TPL, N = 2 * M, PS = POff<LN, TPL>::v, ES = EOff<LN, TPL>::v;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int mode = op.i1;
  const cplx* tw = (const cplx*)op.p0; const cplx* tw2 = (const cplx*)op.p1; const double* isin = (const double*)op.p2;
  double* w = W + 4 * l;
  cplx* w2 = reinterpret_cast<cplx*>(W) + 2 * l;
  const bool q0 = (q == 0);
  // ---- pre: x -> g (N/2 complex), pairs (j, M-j), j = q + pi*TPL < M/2; thread q = 0 also does j = M/2 ----
  const int bj = Lay<LN>::pix(q), bjl = Lay<LN>::pix(q - 1), bm = Lay<LN>::pix(M - q), bml = Lay<LN>::pix(M - q - 1);
  cplx gj[E / 2], gm[E / 2];
  double r0 = 0.0;
  const double sg = (mode == 1) ? -1.0 : 1.0, endf = (mode == 1) ? 2.0 : 1.0;   // backward: y_k = (-1)^k c_k, ends doubled
#pragma unroll
  for (int pi = 0; pi < E / 2; pi++) {
    const bool first = (pi == 0) && q0;   // j == 0, M - j == M
    const cplx pj = w2[bj + pi * PS], pjl = w2[first ? bj : bjl + pi * PS], pm = w2[bm - pi * PS], pml = w2[bml - pi * PS];
    const double xo_p = sg * pj.y;                              // x_{2j+1}
    const double xo_m = first ? xo_p : sg * pjl.y;              // x_{2j-1}, x_{-1} = x_1
    const double xm_m = sg * pml.y;                             // x_{2jm-1}
    const double xm_p = first ? xm_m : sg * pm.y;               // x_{2jm+1}, x_{N+1} = x_{N-1}
    const cplx zj = make_double2(pj.x * (first ? endf : 1.0), xo_p - xo_m);
    const cplx zmc = make_double2(pm.x * (first ? endf : 1.0), -(xm_p - xm_m));   // conj(z_{M-j})
    const cplx e = cadd(zj, zmc), d = cmul(csub(zj, zmc), ldg(tw2 + q + pi * TPL));
    gj[pi] = make_double2(e.x - d.y, e.y + d.x);           // e + i d
    gm[pi] = make_double2(e.x + d.y, -e.y + d.x);          // conj(e) + i conj(d)
    r0 += xo_p + xm_m;
  }
  cplx gmid = make_double2(0.0, 0.0);
  if (q0) {   // j = M - j = M/2
    const cplx pj = w2[Lay<LN>::pix(M / 2)], pjl = w2[Lay<LN>::pix(M / 2 - 1)];
    const double xo_p = sg * pj.y, xo_m = sg * pjl.y;
    const cplx zj = make_double2(pj.x, xo_p - xo_m), zmc = make_double2(pj.x, -(xo_p - xo_m));
    const cplx e = cadd(zj, zmc), d = cmul(csub(zj, zmc), ldg(tw2 + M / 2));
    gmid = make_double2(e.x - d.y, e.y + d.x);
  }
  r0 = 2.0 * lane_sum<LN>(r0, TPL, scratch);   // R_0 = 2 * sum of odd samples
  __syncthreads();
#pragma unroll
  for (int pi = 0; pi < E / 2; pi++) {
    w2[bj + pi * PS] = gj[pi];
    if (!((pi == 0) && q0)) w2[bm - pi * PS] = gm[pi];
  }
  if (q0) w2[Lay<LN>::pix(M / 2)] = gmid;
  __syncthreads();
  pc.mark(22);
  lane_fft_fast<E, LN, TPL>(W, l, q, tw);
  pc.mark(23);
  // ---- post: Z (N reals) -> X (N+1), pairs (k, N-k), k = q + pi*TPL in [1, M-1] ----
  const double fs = (mode == 0) ? 1.0 / N : 0.5;
  const double sk = (mode == 0 && (q & 1)) ? -fs : fs;      // TPL and N are even: k, N-k and q have the same parity
  const int be = Lay<LN>::eix(q), bn = Lay<LN>::eix(N - q);
#pragma unroll
  for (int pi = 0; pi < E; pi++) {
    const bool skip = (pi == 0) && q0;
    const double zk = w[be + pi * ES], zn = w[skip ? be : bn - pi * ES];
    const double A = 0.5 * (zk + zn), R = (zn - zk) * ldg(isin + q + pi * TPL);
    if (!skip) { w[be + pi * ES] = (A + R) * sk; w[bn - pi * ES] = (A - R) * sk; }
  }
  if (q0) {   // k = 0 (and N), k = M: untouched by the loop above
    const double z0 = w[0], e0 = (mode == 0) ? 0.5 * fs : fs;
    w[0] = (z0 + r0) * e0;
    w[Lay<LN>::eix(N)] = (z0 - r0) * e0;
    w[Lay<LN>::eix(M)] = w[Lay<LN>::eix(M)] * ((mode == 0 && (M & 1)) ? -fs : fs);
  }
  __syncthreads();
  pc.mark(24);
}

// Real FFT (see op_rfft), n = 2*E*TPL.
template <int E, int LN, int TPL>
__device__ __noinline__ void rfft_fast(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  constexpr int M = E * TPL, n = 2 * M, PS = POff<LN, TPL>::v, ES = EOff<LN, TPL>::v;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int mode = op.i1;
  const cplx* tw = (const cplx*)op.p0; const cplx* tw2 = (const cplx*)op.p1;
  double* w = W + 4 * l;
  cplx* w2 = reinterpret_cast<cplx*>(W) + 2 * l;
  const bool q0 = (q == 0);
  const int bk = Lay<LN>::pix(q), bm = Lay<LN>::pix(M - q);
  if (mode == 0) {
    lane_fft_fast<E, LN, TPL>(W, l, q, tw);
    // X_k = (S - i wD)/2 ; X_{M-k} = conj((S + i wD)/2),  S = z_k + conj(z_{M-k}), D = z_k - conj(z_{M-k}), k = q + pi*TPL < M/2
#pragma unroll
    for (int pi = 0; pi < E / 2; pi++) {
      const bool first = (pi == 0) && q0;
      const cplx zk = w2[bk + pi * PS], zm = cconj(w2[first ? bk : bm - pi * PS]);
      const cplx S = cadd(zk, zm), D = cmul(ldg(tw2 + q + pi * TPL), csub(zk, zm));
      if (first) {
        w2[0] = make_double2(zk.x + zk.y, 0.0);
        w2[Lay<LN>::pix(M)] = make_double2(zk.x - zk.y, 0.0);
      } else {
        w2[bk + pi * PS] = make_double2(0.5 * (S.x + D.y), 0.5 * (S.y - D.x));
        w2[bm - pi * PS] = make_double2(0.5 * (S.x - D.y), -0.5 * (S.y + D.x));
      }
    }
    if (q0) {   // k = M/2 = M - k
      const cplx zk = w2[Lay<LN>::pix(M / 2)], zm = cconj(zk);
      const cplx S = cadd(zk, zm), D = cmul(ldg(tw2 + M / 2), csub(zk, zm));
      w2[Lay<LN>::pix(M / 2)] = make_double2(0.5 * (S.x + D.y), 0.5 * (S.y - D.x));
    }
    __syncthreads();
  } else {
#pragma unroll
    for (int pi = 0; pi < E / 2; pi++) {
      const bool first = (pi == 0) && q0;
      const cplx xk = w2[bk + pi * PS], xm = cconj(w2[first ? bk : bm - pi * PS]);
      const cplx S = cadd(xk, xm), D = cmul(cconj(ldg(tw2 + q + pi * TPL)), csub(xk, xm));
      if (first) {
        const double x0 = xk.x, xM = w[Lay<LN>::eix(2 * M)];
        w2[0] = make_double2(0.5 * (x0 + xM), -0.5 * (x0 - xM));   // Zc_0 = ((x0+xm) + i(x0-xm))/2, stored conjugated
      } else {
        w2[bk + pi * PS] = make_double2(0.5 * (S.x - D.y), -0.5 * (S.y + D.x));
        w2[bm - pi * PS] = make_double2(0.5 * (S.x + D.y), 0.5 * (S.y - D.x));
      }
    }
    if (q0) {
      const cplx xk = w2[Lay<LN>::pix(M / 2)], xm = cconj(xk);
      const cplx S = cadd(xk, xm), D = cmul(cconj(ldg(tw2 + M / 2)), csub(xk, xm));
      w2[Lay<LN>::pix(M / 2)] = make_double2(0.5 * (S.x - D.y), -0.5 * (S.y + D.x));
    }
    __syncthreads();
    lane_fft_fast<E, LN, TPL>(W, l, q, tw);
    const double s = (q & 1) ? -1.0 / M : 1.0 / M;   // conjugate back (odd elements = imaginary parts) and scale
    const int be = Lay<LN>::eix(q);
#pragma unroll
    for (int i = 0; i < 2 * E; i++) w[be + i * ES] *= s;
    for (int e = n + q; e < P.LP; e += TPL) w[Lay<LN>::eix(e)] = 0.0;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// banded mat-vec (see op_band): pairs p = q + t*TPL, t = 0..E; only t = 0 (first pair) and t = E (the pairs
// beyond N/2) need range predicates.
// ---------------------------------------------------------------------------------------------
template <int E, int LN, int TPL>
__device__ __noinline__ void band_fast(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  constexpr int CP = E + 1, PS = POff<LN, TPL>::v, M = E * TPL;
  const int HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int len_out = op.i0;
  const int h0 = (int)(signed char)(op.i1 & 0xff), h1 = (int)(signed char)((op.i1 >> 8) & 0xff), h2 = (int)(signed char)((op.i1 >> 16) & 0xff);
  const double2* __restrict__ c0 = (const double2*)op.p0;
  const double2* __restrict__ c1 = (const double2*)op.p1;
  const double2* __restrict__ c2 = (const double2*)op.p2;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  const double2 zero = d2(0.0, 0.0), one = d2(1.0, 1.0);
  double2 y[CP];
#pragma unroll
  for (int t = 0; t < CP; t++) y[t] = zero;
  auto term = [&](int h, const double2* __restrict__ c) {
    const int hp = h >> 1;                 // -1 .. 2
    const int bx = Lay<LN>::pix(q + hp);   // (q + hp = -1 gives a base that is only valid from t = 1 on)
    const bool neg = (q + hp) < 0;
    const int pl = q + M;
    const bool okl = pl < HP && pl + hp < HP;
    const double2 x0 = w2[neg ? 0 : bx], xl = w2[okl ? bx + E * PS : 0];
    if (c) {
      const double2 c0v = ldg(c + q), clv = ldg(c + (okl ? pl : 0));
      if (!neg) y[0] = d2fma(c0v, x0, y[0]);
#pragma unroll
      for (int t = 1; t < E; t++) y[t] = d2fma(ldg(c + q + t * TPL), w2[bx + t * PS], y[t]);   // p + hp <= M + 1 < HP: in range
      if (okl) y[E] = d2fma(clv, xl, y[E]);
    } else {
      if (!neg) { y[0].x += x0.x; y[0].y += x0.y; }
#pragma unroll
      for (int t = 1; t < E; t++) { const double2 x = w2[bx + t * PS]; y[t].x += x.x; y[t].y += x.y; }
      if (okl) { y[E].x += xl.x; y[E].y += xl.y; }
    }
  };
  if (h0 != 127) term(h0, c0);
  if (h1 != 127) term(h1, c1);
  if (h2 != 127) term(h2, c2);
  __syncthreads();
  const int bq = Lay<LN>::pix(q);
  if (len_out >= 2 * M) {     // the usual case: only the pairs of t = E can reach len_out
#pragma unroll
    for (int t = 0; t < E; t++) w2[bq + t * PS] = y[t];
  } else {
#pragma unroll
    for (int t = 0; t < E; t++) {
      const int p = q + t * TPL;
      double2 v = y[t];
      if (2 * p >= len_out) v.x = 0.0;
      if (2 * p + 1 >= len_out) v.y = 0.0;
      w2[bq + t * PS] = v;
    }
  }
  {
    const int p = q + M;
    double2 v = y[E];
    if (2 * p >= len_out) v.x = 0.0;
    if (2 * p + 1 >= len_out) v.y = 0.0;
    if (p < HP) w2[bq + E * PS] = v;
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// chunked recurrences: thread q owns pairs p0 + t, p0 = q*CP, t < CP (CP = E + 1 odd).  pix(p0 + t) is
// base_even + c(t) for even t and base_odd + c(t) for odd t with compile-time c: two runtime bases per thread.
// ---------------------------------------------------------------------------------------------
template <int LN> struct ChunkAddr {
  int be, bo;
  __device__ __forceinline__ ChunkAddr(int p0) {
    const int par = p0 & 1, pe = Lay<LN>::pix(p0 - par);
    be = pe + par; bo = pe + par * ((1 << Lay<LN>::LSH) - 1);
  }
  template <int T> __device__ __forceinline__ int at() const { return ((T & 1) ? bo : be) + Lay<LN>::pix(T); }
  __device__ __forceinline__ int at(int t) const { return ((t & 1) ? bo : be) + Lay<LN>::pix(t); }
};

// Banded mat-vec with chunk ownership, streamed in place (OP_BANDC, set by the launcher): thread q owns the pairs
// p0 + t like the recurrences below, reads every pair of W once and writes it once -- one read and one write traversal
// of the lane group instead of one read per term plus the write of band_fast (the lane operators are bound by
// shared-memory bandwidth, 128 B/clk: ~1k cycles per traversal of a 131 KB group).
//   forward type  (i1 bit 0 = 0): y_p = k0 x_p + k1 x_{p+1} + k2 x_{p+2}   (pair offsets 0, +1, +2: S^T, MatVecFdma)
//   backward type (i1 bit 0 = 1): y_p = k0 x_p + k1 x_{p-1}                (to_ortho stencil)
// term flags, 2 bits each from bit 2: 0 absent, 1 unit coefficient, 2 scan-layout vector ([t][q]) in p0 / p1 / p2.
template <int E, int LN, int TPL>
__device__ __noinline__ void band_chunk(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  constexpr int CP = E + 1;
  const int HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  const int p0 = q * CP;
  const ChunkAddr<LN> ca(p0);
  const int tmax = HP - p0;                                     // t < tmax: the pair exists in W
  const int len_out = op.i0;
  const int tx = (len_out - 2 * p0 + 1) >> 1, ty = (len_out - 2 * p0) >> 1;   // t < tx: element 2p < len_out; t < ty: 2p+1 < len_out
  const double2 zero = d2(0.0, 0.0);
  const double2* cp[3] = {(const double2*)op.p0, (const double2*)op.p1, (const double2*)op.p2};
  const double2* any = cp[0] ? cp[0] : (cp[1] ? cp[1] : cp[2]);
  double wl[3], ad[3];                                          // coefficient = loaded * wl + ad (loads stay unconditional)
#pragma unroll
  for (int m = 0; m < 3; m++) {
    const int f = (op.i1 >> (2 + 2 * m)) & 3;
    wl[m] = (f == 2) ? 1.0 : 0.0; ad[m] = (f == 1) ? 1.0 : 0.0;
    cp[m] = ((f == 2) ? cp[m] : any) + q;
  }
  if (!(op.i1 & 1)) {
    const double2 hA = (CP < tmax) ? w2[ca.at(CP)] : zero, hB = (CP + 1 < tmax) ? w2[ca.at(CP + 1)] : zero;
    __syncthreads();
    double2 x0 = (0 < tmax) ? w2[ca.at(0)] : zero, x1 = (1 < tmax) ? w2[ca.at(1)] : zero;
#pragma unroll
    for (int t = 0; t < CP; t++) {
      const double2 x2 = (t + 2 < CP) ? ((t + 2 < tmax) ? w2[ca.at(t + 2 < CP ? t + 2 : 0)] : zero) : (t + 2 == CP ? hA : hB);
      const double2 l0 = ldg(cp[0] + t * TPL), l1 = ldg(cp[1] + t * TPL), l2 = ldg(cp[2] + t * TPL);
      const double2 k0 = d2(fma(l0.x, wl[0], ad[0]), fma(l0.y, wl[0], ad[0]));
      const double2 k1 = d2(fma(l1.x, wl[1], ad[1]), fma(l1.y, wl[1], ad[1]));
      const double2 k2 = d2(fma(l2.x, wl[2], ad[2]), fma(l2.y, wl[2], ad[2]));
      double2 b = d2fma(k0, x0, d2fma(k1, x1, d2(k2.x * x2.x, k2.y * x2.y)));
      if (t >= tx) b.x = 0.0;
      if (t >= ty) b.y = 0.0;
      if (t < tmax) w2[ca.at(t)] = b;
      x0 = x1; x1 = x2;
    }
  } else {
    const double2 hP = (q > 0 && 0 <= tmax) ? w2[Lay<LN>::pix(p0 - 1)] : zero;   // the pair in front of the chunk
    __syncthreads();
    double2 x0 = (CP - 1 < tmax) ? w2[ca.at(CP - 1)] : zero;
#pragma unroll
    for (int t = CP - 1; t >= 0; t--) {
      const double2 xm = (t > 0) ? ((t - 1 < tmax) ? w2[ca.at(t > 0 ? t - 1 : 0)] : zero) : hP;
      const double2 l0 = ldg(cp[0] + t * TPL), l1 = ldg(cp[1] + t * TPL);
      const double2 k0 = d2(fma(l0.x, wl[0], ad[0]), fma(l0.y, wl[0], ad[0]));
      const double2 k1 = d2(fma(l1.x, wl[1], ad[1]), fma(l1.y, wl[1], ad[1]));
      double2 b = d2fma(k0, x0, d2(k1.x * xm.x, k1.y * xm.y));
      if (t >= tx) b.x = 0.0;
      if (t >= ty) b.y = 0.0;
      if (t < tmax) w2[ca.at(t)] = b;
      x0 = xm;
    }
  }
  __syncthreads();
}

template <int E, int LN, int TPL>
__device__ __noinline__ void deriv_fast(const LaneProg& P, const LaneOp& op, double* __restrict__ W, void* scratch) {
  constexpr int CP = E + 1;
  const int HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  const int p0 = q * CP;
  const ChunkAddr<LN> ca(p0);
  const int tmax = HP - p0;   // pairs of this chunk that exist (may be <= 0 or >= CP)
  for (int rep = 0; rep < op.i1; rep++) {
    double2 tp[CP];
    double2 tot = d2(0.0, 0.0);
#pragma unroll
    for (int t = 0; t < CP; t++) {
      const bool ok = t < tmax;
      const double2 a = ok ? w2[ca.at(t)] : d2(0.0, 0.0);
      const double f = 4.0 * (p0 + t);
      tp[t] = d2(f * a.x, (f + 2.0) * a.y);
      tot.x += tp[t].x; tot.y += tp[t].y;
    }
    Aff1::V m; m.d[0] = 1; m.d[1] = tot.x; m.d[2] = 1; m.d[3] = tot.y;
    Aff1::S in = lane_scan_state<Aff1, true, LN>(m, TPL, scratch);
    double2 S = d2(in.d[0], in.d[1]);   // S of the first pair of the next chunk
    const double sc = (rep == op.i1 - 1) ? op.a : 1.0;
#pragma unroll
    for (int t = CP - 1; t >= 0; t--) {
      const double nx = S.x;
      S.x += tp[t].x; S.y += tp[t].y;
      double2 o = d2(S.y * sc, nx * sc);
      if (t == 0 && q == 0) o.x *= 0.5;
      if (t < tmax) w2[ca.at(t)] = o;
    }
    __syncthreads();
  }
}

// LU solve (see op_fdma).  PERLANE: coefficient arrays [group][t][q][lane of 4] instead of shared [t][q].  Shared vectors come
// as the chunk-map table (LM_*): the forward chunk map needs no product of coefficients, the back-substitution chunk map is a
// weighted sum of the chunk's y (2 FMA per pair and parity instead of composing a 2x2 affine map per pair), and the solve does
// not multiply by id.  The per-lane arrays stream from HBM (one set per lane), where a table of 6 vectors instead of 4 would
// cost more traffic than the arithmetic it saves, so they keep the composing form.
template <int E, int LN, int TPL, bool PERLANE, bool PREBAND>
__device__ __forceinline__ void fdma_fast_body(const LaneProg& P, const LaneOp& op, double* __restrict__ W, int gl, int lb, void* scratch) {
  constexpr int CP = E + 1, CS = PERLANE ? 4 * TPL : TPL;
  constexpr bool MAPS = !PERLANE;
  const int HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int n = op.i0;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  const size_t cb = PERLANE ? ((size_t)gl * CP * TPL + q) * 4 + lb + l : (size_t)q;
  const double2* __restrict__ cfl = (const double2*)op.p0 + cb;   // MAPS: the table, slot LM_FL = 0
  const double2* __restrict__ cid = MAPS ? cfl + LM_ID * CP * TPL : (const double2*)op.p1 + cb;
  const double2* __restrict__ cu1 = MAPS ? cfl + LM_U1 * CP * TPL : (const double2*)op.p2 + cb;
  const double2* __restrict__ cu2 = MAPS ? cfl + LM_U2 * CP * TPL : (const double2*)op.p3 + cb;
  const bool nou2 = op.i2 & FD_NOU2;
  const double2 zero = d2(0.0, 0.0);
  const int p0 = q * CP;
  const ChunkAddr<LN> ca(p0);
  const int tmax = HP - p0;                                    // t < tmax: the pair exists in W
  const int tx = (n - 2 * p0 + 1) >> 1, ty = (n - 2 * p0) >> 1; // t < tx: element 2p < n;  t < ty: element 2p+1 < n
  // Chunks that lie completely inside [0, n) (all but the last one or two of a lane) run without any masks.
  const bool interior = (tmax >= CP) && (ty >= CP);
  auto rdm = [&](int t) -> double2 {   // right-hand side / intermediate at pair p0+t, zero outside [0, n)
    double2 v = (t < tmax) ? w2[ca.at(t)] : zero;
    if (t >= tx) v.x = 0.0;
    if (t >= ty) v.y = 0.0;
    return v;
  };
  PhaseClock pc(P.prof);
  // MAPS: translation of the back-substitution chunk map = the weighted sums of the chunk's y, accumulated as the forward pass
  // produces y (no separate pass over the chunk)
  double2 ta = zero, tb = zero;
  const double2* __restrict__ cwa = cfl + LM_WA * CP * TPL;
  const double2* __restrict__ cwb = cfl + LM_WB * CP * TPL;
  // ---- forward elimination: y_p = b_p - fl_p y_{p-1} ----
  {
    double2 A = d2(1.0, 1.0), B = zero;
    if constexpr (PREBAND) {
      // The right-hand side is a banded mat-vec of what is in W: b_p = c0_p x_p + c1_p x_{p+1} + c2_p x_{p+2}
      // (pair offsets 0, +1, +2; a null coefficient vector = 1; scan-layout vectors [t][q]).  It is formed here, on the
      // fly, and written back in place; the two pairs after the chunk are read before anybody writes.
      const LaneOp& bop = *(&op - 1);
      // every term loads unconditionally (absent / unit coefficients read the LU vector instead and are blended
      // to 0 / 1 afterwards), so that the 3 x CP coefficient loads can all be in flight at once
      const double2* cf[3] = {cfl, cfl, cfl};
      double wl[3] = {0.0, 0.0, 0.0}, ad[3] = {0.0, 0.0, 0.0};   // coefficient = loaded * wl + ad
#pragma unroll
      for (int m = 0; m < 3; m++) {
        const int h = (int)(signed char)((bop.i1 >> (8 * m)) & 0xff);
        const double2* cp = (const double2*)(m == 0 ? bop.p0 : (m == 1 ? bop.p1 : bop.p2));
#pragma unroll
        for (int k = 0; k < 3; k++)
          if (h == 2 * k) { if (cp) { cf[k] = cp + q; wl[k] = 1.0; } else ad[k] = 1.0; }
      }
      const double2 hA = (CP < tmax) ? w2[ca.at(CP)] : zero, hB = (CP + 1 < tmax) ? w2[ca.at(CP + 1)] : zero;
      __syncthreads();
      double2 x0 = (0 < tmax) ? w2[ca.at(0)] : zero, x1 = (1 < tmax) ? w2[ca.at(1)] : zero;
#pragma unroll
      for (int t = 0; t < CP; t++) {
        const double2 x2 = (t + 2 < CP) ? ((t + 2 < tmax) ? w2[ca.at(t + 2 < CP ? t + 2 : 0)] : zero) : (t + 2 == CP ? hA : hB);
        double2 b = zero;
        const double2 l0 = ldg(cf[0] + t * TPL), l1 = ldg(cf[1] + t * TPL), l2 = ldg(cf[2] + t * TPL);
        const double2 k0 = d2(fma(l0.x, wl[0], ad[0]), fma(l0.y, wl[0], ad[0]));
        const double2 k1 = d2(fma(l1.x, wl[1], ad[1]), fma(l1.y, wl[1], ad[1]));
        const double2 k2 = d2(fma(l2.x, wl[2], ad[2]), fma(l2.y, wl[2], ad[2]));
        b = d2fma(k0, x0, d2fma(k1, x1, d2(k2.x * x2.x, k2.y * x2.y)));
        if (t >= tx) b.x = 0.0;
        if (t >= ty) b.y = 0.0;
        if (t < tmax) w2[ca.at(t)] = b;
        const double2 f = ldg(cfl + t * CS);
        B = d2(fma(-f.x, B.x, b.x), fma(-f.y, B.y, b.y));
        if constexpr (!MAPS) A = d2(-f.x * A.x, -f.y * A.y);
        x0 = x1; x1 = x2;
      }
    } else if (interior) {
#pragma unroll
      for (int t = 0; t < CP; t++) {
        const double2 f = ldg(cfl + t * CS), b = w2[ca.at(t)];
        B = d2(fma(-f.x, B.x, b.x), fma(-f.y, B.y, b.y));
        if constexpr (!MAPS) A = d2(-f.x * A.x, -f.y * A.y);
      }
    } else {
#pragma unroll
      for (int t = 0; t < CP; t++) {
        const double2 f = ldg(cfl + t * CS), b = rdm(t);
        B = d2(fma(-f.x, B.x, b.x), fma(-f.y, B.y, b.y));
        if constexpr (!MAPS) A = d2(-f.x * A.x, -f.y * A.y);
      }
    }
    if constexpr (MAPS) A = ldg(cfl + (LM_CHUNK * CP + LMC_A) * TPL);
    pc.mark(16);
    Aff1::V m; m.d[0] = A.x; m.d[1] = B.x; m.d[2] = A.y; m.d[3] = B.y;
    Aff1::S in = lane_scan_state<Aff1, false, LN>(m, TPL, scratch);
    pc.mark(17);
    double2 y = d2(in.d[0], in.d[1]);   // y of the last pair before this chunk (the start state is 0)
    if (interior) {
#pragma unroll
      for (int t = 0; t < CP; t++) {
        const double2 f = ldg(cfl + t * CS), b = w2[ca.at(t)];
        y = d2(fma(-f.x, y.x, b.x), fma(-f.y, y.y, b.y));
        w2[ca.at(t)] = y;
        if constexpr (MAPS) { ta = d2fma(ldg(cwa + t * TPL), y, ta); tb = d2fma(ldg(cwb + t * TPL), y, tb); }
      }
    } else {
#pragma unroll
      for (int t = 0; t < CP; t++) {
        const double2 f = ldg(cfl + t * CS), b = rdm(t);
        y = d2(fma(-f.x, y.x, b.x), fma(-f.y, y.y, b.y));
        if (t < tmax) w2[ca.at(t)] = y;
        if constexpr (MAPS) {   // the y the back substitution reads: zero outside [0, n) and beyond the lane
          double2 v = (t < tmax) ? y : zero;
          if (t >= tx) v.x = 0.0;
          if (t >= ty) v.y = 0.0;
          ta = d2fma(ldg(cwa + t * TPL), v, ta); tb = d2fma(ldg(cwb + t * TPL), v, tb);
        }
      }
    }
  }
  pc.mark(18);
  // every thread only touched its own chunk of W: no barrier needed before the back substitution.  The scan scratch needs none
  // either: the back substitution's warp totals never overlap the entry states a slower warp may still be reading from the
  // forward scan (lane_scan_state)
  // ---- back substitution: x_p = (y_p - u1_p x_{p+1} - u2_p x_{p+2}) id_p ----
  {
    Aff2::V m = Aff2::identity();
    if constexpr (MAPS) {   // linear part of the chunk map from the table, translation from the forward pass
      const double2* __restrict__ cP = cfl + (LM_CHUNK * CP + LMC_P) * TPL;
      const double2 P00 = ldg(cP), P01 = ldg(cP + TPL), P10 = ldg(cP + 2 * TPL), P11 = ldg(cP + 3 * TPL);
      m.d[0] = P00.x; m.d[1] = P01.x; m.d[2] = P10.x; m.d[3] = P11.x; m.d[4] = ta.x; m.d[5] = tb.x;
      m.d[6] = P00.y; m.d[7] = P01.y; m.d[8] = P10.y; m.d[9] = P11.y; m.d[10] = ta.y; m.d[11] = tb.y;
    } else {
      auto compose = [&](int t, double2 y) {   // compose pair t onto the chunk map; state = (x_{p+1}, x_{p+2}) per component
        const double2 idv = ldg(cid + t * CS), u1 = ldg(cu1 + t * CS), u2 = nou2 ? zero : ldg(cu2 + t * CS);
        const double2 m0 = d2(-u1.x * idv.x, -u1.y * idv.y), m1 = d2(-u2.x * idv.x, -u2.y * idv.y), g0 = d2(y.x * idv.x, y.y * idv.y);
        double* Mx = m.d;
        double r0 = m0.x * Mx[0] + m1.x * Mx[2], r1 = m0.x * Mx[1] + m1.x * Mx[3], rp = m0.x * Mx[4] + m1.x * Mx[5] + g0.x;
        Mx[2] = Mx[0]; Mx[3] = Mx[1]; Mx[5] = Mx[4]; Mx[0] = r0; Mx[1] = r1; Mx[4] = rp;
        Mx = m.d + 6;
        r0 = m0.y * Mx[0] + m1.y * Mx[2]; r1 = m0.y * Mx[1] + m1.y * Mx[3]; rp = m0.y * Mx[4] + m1.y * Mx[5] + g0.y;
        Mx[2] = Mx[0]; Mx[3] = Mx[1]; Mx[5] = Mx[4]; Mx[0] = r0; Mx[1] = r1; Mx[4] = rp;
      };
      if (interior) {
#pragma unroll
        for (int t = CP - 1; t >= 0; t--) compose(t, w2[ca.at(t)]);
      } else {
#pragma unroll
        for (int t = CP - 1; t >= 0; t--) compose(t, rdm(t));
      }
    }
    pc.mark(19);
    Aff2::S in = lane_scan_state<Aff2, true, LN>(m, TPL, scratch);
    pc.mark(20);
    double2 s1 = d2(in.d[0], in.d[2]), s2 = d2(in.d[1], in.d[3]);   // x_{p+1}, x_{p+2} entering the chunk
    auto solve = [&](int t, double2 y) -> double2 {
      const double2 idv = ldg(cid + t * CS), u1 = ldg(cu1 + t * CS), u2 = nou2 ? zero : ldg(cu2 + t * CS);
      const double2 x = MAPS ? d2(fma(-u1.x, s1.x, fma(-u2.x, s2.x, idv.x * y.x)), fma(-u1.y, s1.y, fma(-u2.y, s2.y, idv.y * y.y)))   // u1, u2 times id
                             : d2((y.x - u1.x * s1.x - u2.x * s2.x) * idv.x, (y.y - u1.y * s1.y - u2.y * s2.y) * idv.y);
      s2 = s1; s1 = x;
      return x;
    };
    if (interior) {
#pragma unroll
      for (int t = CP - 1; t >= 0; t--) w2[ca.at(t)] = solve(t, w2[ca.at(t)]);
    } else {
#pragma unroll
      for (int t = CP - 1; t >= 0; t--) { const double2 x = solve(t, rdm(t)); if (t < tmax) w2[ca.at(t)] = x; }
    }
  }
  __syncthreads();
  pc.mark(21);
}
template <int E, int LN, int TPL>
__device__ __noinline__ void fdma_fast(const LaneProg& P, const LaneOp& op, double* __restrict__ W, int gl, int lb, void* scratch) {
  if (op.i2 & FD_PERLANE) fdma_fast_body<E, LN, TPL, true, false>(P, op, W, gl, lb, scratch);
  else if (op.i2 & FD_PREBAND) fdma_fast_body<E, LN, TPL, false, true>(P, op, W, gl, lb, scratch);
  else fdma_fast_body<E, LN, TPL, false, false>(P, op, W, gl, lb, scratch);
}
