// Lane-program kernel: the one CUDA kernel family behind every per-axis operator
// of the Navier2D spectral hot path (SURVEY.md 8a rows A-L).
//
// A CTA owns one "lane group" = 4 neighbouring 1-D lanes (pencils) of a 2-D array (or half a group for
// very long lanes) and keeps them resident in shared memory while it interprets a short program of
// 1-D operators (load / banded mat-vec / Chebyshev recurrence / banded LU solve / DCT-I / real FFT /
// masks / store).  Arrays live in HBM in a 4x4 micro-tiled layout (128-byte tiles), so a lane group is ONE
// contiguous slab, and shared memory keeps exactly that layout (tile J of the group = [lane][4 positions]):
//   * a plain load is a zero-copy bulk tensor copy (TMA) of the slab into shared memory, a plain store the
//     reverse; loads that combine with the resident operand (accumulate, multiply, composite->orthonormal
//     stencil) stream through a small TMA ring that thread 0 keeps full across op boundaries;
//   * a transposing store (the x<->y pencil switch: every pass of a 2-D operator ends in one) transposes
//     each 4x4 tile on its way into a staging slot and leaves as ONE 4-D tensor store per chunk -- full
//     128-byte lines into the transposed array (or, multi-GPU, per-thread stores into the peer's slab);
//   * threads map lane-fastest (tid -> lane = tid % LN, q = tid / LN), which makes every shared-memory
//     access of every operator bank-conflict free in this layout and lets the 4 lanes of a group share
//     each coefficient / twiddle load (one broadcast request instead of four).
//
// sm_90a (H100) only.  No CPU fallback, no library calls in here.
#pragma once
#ifdef B2_EMU   // tests/emu: the same source compiled for the CPU SIMT emulator (test infrastructure only)
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#define B2_DYN_SMEM(type, name) extern __shared__ __align__(1024) type name[]
#define B2_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif
#include <stdint.h>
#include <stddef.h>
#include "async_ops.cuh"

#define B2_MAXOPS 24
#define B2_MAXPEERS 8
#define B2_MAXPST 6     // transposing stores per program that can go to peer GPUs through tensor maps
#define B2_BARBYTES 512  // mbarriers at the start of dynamic shared memory: dfull + 2 per warp
#define B2_SCRATCH 8192  // bytes of scan scratch: 16 warps x 4 lanes x (Aff2 map + Aff2 state); entry states at one fixed offset
                         // behind the largest warp totals (see lane_scan_state)
#define B2_PROGCOPY 2048 // shared-memory copy of the program header + ops (everything of LaneProg in front of tm[])

enum LaneOpCode {
  OP_LOAD = 1,     // W = [W +|*] a * src           i0=len  i2=flags(LD_*)       p0=src (p1 = stencil coefficients)
  OP_STORE = 2,    // dst = [dst +] a * W            i0=len  i2=flags(ST_*)       p0=dst  (p1=peer table)
  OP_BAND = 3,     // y_i = sum_m c_m[i] x_{i+o_m}   i0=len_out i1=packed offs i2=len_in  p0..p2 coef (null = 1, i1 byte=127: unused)
  OP_DERIV = 4,    // Chebyshev d/dx of i0 coeffs, i1 times, times a
  OP_FDMA = 5,     // banded LU solve (fwd elim + back subst)  i0=len i2=flags(FD_*) p0=fl p1=inv_dia p2=u1 p3=u2 (fast geometry,
                   //   shared vectors: p0 = chunk-map table, LM_*)
  OP_DCT = 6,      // Chebyshev transform, i0=n (=N+1), i1: 0 fwd (values->coeffs) 1 bwd   p0=tw p1=tw2 p2=isin
  OP_RFFT = 7,     // Fourier r2c/c2r, i0=n, i1: 0 fwd 1 bwd                              p0=tw p1=tw2
  OP_FDIFF = 8,    // interleaved complex modes: c_k *= (i k)^{i1} * a,  i0 = number of modes, i2 = n for FFT-ordered modes (c2c) else 0
  OP_SCALEVEC = 9, // W[e] *= p0[e >> i1] for e < i0
  OP_ZEROTAIL = 10,// W[e] = 0 for e >= i0
  OP_LANEMASK = 11,// lanes >= i0 zeroed
  OP_ZEROELEM = 12,// W[lane i0][pos i1] = 0 (global lane index)
  OP_SCALE = 13,   // W *= a
  OP_PREBAND = 14, // an OP_BAND folded into the OP_FDMA that follows it (set by the launcher, fast geometry only): no-op here
  OP_BANDC = 15,   // an OP_BAND in chunk-streaming form (set by the launcher, fast geometry only): see band_chunk
  OP_STEN3 = 16,   // ChebDirichletNeumann stencil (odd offsets): i1 = 0: y_j = x_j + a_{j-1} x_{j-1} + b_{j-2} x_{j-2} (to_ortho, S);
                   //   i1 = 1: y_k = x_k + a_k x_{k+1} + b_k x_{k+2} (S^T);  i0 = len_out, p0 = a, p1 = b (natural order)
  OP_DENSE = 18,   // dense mat-vec along the lane: y_k = sum_j M[k][j] x_j, i0 = n_out, i1 = n_in, p0 = M (row-major): the transforms
                   //   of sizes the FFT core does not handle (n - 1 / n not a power of two): O(n^2) per lane, small grids only
  OP_PDMA = 17,    // PdmaPlus2 solve (7 diagonals -2..+4, src/solver/pdma_plus2.rs:123-157): i0 = n, i1 = pitch L of the packed LU
                   //   p0 = [l2 shifted | ka | 1/mu | al | be | ga | de], each L doubles
};
enum { LD_ACC = 1, LD_PLAIN = 2, LD_MUL = 4, LD_STENCIL = 8,   // LD_STENCIL: value = src[j] + p1[j] * src[j-2]
       LD_TMA = 16,          // set by the launcher: the slab streams through the warps' staging slots (load_warps)
       LD_AFTER_STORE = 32,  // set by the launcher: the source was stored earlier in this program (flush stores first)
       LD_DIRECT = 64,       // set by the launcher: zero-copy TMA straight into W (plain load, a == 1)
       LD_PSPLIT = 128,      // plain sources: rows are stored parity-split (row r < i1 lives at r/2, odd rows after the even ones)
       LD_PSPLITC = 256 };   // plain sources: the positions along the lane (columns) are stored parity-split, i1 = m0
enum { ST_ACC = 1, ST_PLAIN = 2, ST_TRANS = 8, ST_PEER = 16,
       ST_TMA = 32,          // set by the launcher: staged, bulk tensor store / reduction
       ST_DIRECT = 64,       // set by the launcher: zero-copy TMA straight from W (same orientation, a == 1, no accumulate)
       ST_PSPLIT = 128,      // plain destinations, same orientation: store row r < i1 at r/2 (even) or ceil(i1/2) + r/2 (odd)
       ST_PSPLITC = 256,     // plain transposing stores: lane index (= column) c <= i1 goes to c/2 (even) or ceil(i1/2) + c/2 (odd)
       ST_COLSPLIT = 512 };  // several GPUs, same orientation: the positions along the lane are distributed over the ranks -- tile J of global
                             // lane group g goes to rank J / groups_per_rank, tile (g, J mod groups_per_rank) of its [all rows][local columns] array
                             // (operand of the eigen-transform GEMM, whose contraction runs over the rows); p1 = peer table
enum { FD_PERLANE = 1, FD_NOU2 = 2,
       FD_PREBAND = 4 };   // the right-hand side is the banded mat-vec described by the preceding OP_PREBAND op
// Chunk maps of an LU solve with shared coefficient vectors (set by the launcher on transform-sized lanes: OP_FDMA p0 = the
// table, see fdma_fast_body).  Everything in it depends on the coefficients only, so the host computes it once.  double2 slot
// [s][q] of the thread that owns pairs q*CP + t (both parities), s = LM_x * CP + t for the per-pair entries:
//   LM_FL: fl   LM_ID: id   LM_U1: u1 * id   LM_U2: u2 * id
//   LM_WA, LM_WB: weight of y_t in x_{p0} and x_{p0+1} of the chunk's back-substitution map (entered with zero state)
// and LM_CHUNK * CP + LMC_x for the per-chunk entries: LMC_A = product of -fl over the chunk (linear part of the forward map),
// LMC_P .. LMC_P + 3 = P00 P01 P10 P11 (linear part of the back-substitution map, Aff2 order).
enum { LM_FL = 0, LM_ID, LM_U1, LM_U2, LM_WA, LM_WB, LM_CHUNK };
enum { LMC_A = 0, LMC_P = 1, LMC_N = 5 };

struct LaneOp {
  int code, i0, i1, i2;
  double a, b;
  const void* p0;
  const void* p1;
  const void* p2;
  const void* p3;
};

struct LaneProg {
  int nops;
  int LP;         // lane pitch in doubles = 4 * in_tiles (>= every length used)
  int in_tiles;   // 4x4 tiles per lane of arrays in the orientation being read
  int out_tiles;  // tiles per row of the transposed orientation (= number of lane groups)
  int TPL;        // threads per lane
  int C;          // pairs per thread per lane (= E+1 of the kernel instance), 2*C*TPL >= LP
  int group0;     // first lane group of this launch (multi-GPU slabs)
  int groups_per_rank;  // for ST_PEER: owner(J) = J / groups_per_rank (destination orientation)
  int rank;       // this GPU's rank (peer table index)
  int LN;         // lanes per CTA: 4 (a whole lane group) or 2 (half a group; grid = 2 x groups)
  int NT;         // threads per CTA = LN*TPL (multiple of 32)
  // copy-pipeline geometry
  int CHW, nsc;               // per-warp sub-chunks: tiles per sub-chunk, sub-chunks per lane (warp w takes w, w + nwarps, ...)
  int wslot_bytes;            // pitch of a warp's staging slot: (CHW + 1) tiles (one halo tile in front), multiple of 128
  int CHD, nchd;              // direct copies: tiles per box (<= 256), boxes per lane
  int w_off, st_off;          // byte offsets inside dynamic shared memory (128-aligned)
  int bulk1d;                 // LN == 4: the slab is contiguous, so slab-shaped copies are plain 1-D bulk copies (no tensor map)
  unsigned long long* prof;   // optional per-op cycle counters (64 entries), null in production
  LaneOp ops[B2_MAXOPS];
  B2TMap tm[B2_MAXOPS];       // tensor map of op i (3-D slab view, or 4-D transposed view for transposing stores)
  B2TMap tmp[B2_MAXPST][B2_MAXPEERS];   // multi-GPU transposing store k (op.i1 = k): the transposed view of the destination in every owner's slab
};

// sub-phase cycle marks of the per-op profiler (thread 0; slots 16..31 of LaneProg::prof, counts at +32): only active
// while b2_ctx_opprof is on
__device__ __forceinline__ long long b2_clock() {
#if defined(__CUDA_ARCH__) || defined(B2_EMU)
  return clock64();
#else
  return 0;
#endif
}
struct PhaseClock {
  unsigned long long* prof; long long t;
  __device__ __forceinline__ explicit PhaseClock(unsigned long long* p) : prof(p), t(p ? b2_clock() : 0) {}
  __device__ __forceinline__ void mark(int slot) {
    if (prof && threadIdx.x == 0) {
      const long long n = b2_clock();
      atomicAdd(prof + slot, (unsigned long long)(n - t));
      atomicAdd(prof + 32 + slot, 1ull);
      t = n;
    }
  }
};
#ifdef B2_EMU
template <class T> static inline T ldg(const T* p) { return *p; }
#else
template <class T> __device__ __forceinline__ T ldg(const T* p) { return __ldg(p); }   // LDG.CONSTANT: read-only tables / coefficients
#endif
typedef double2 cplx;
__device__ __forceinline__ cplx cmul(cplx a, cplx b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ cplx cadd(cplx a, cplx b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ cplx csub(cplx a, cplx b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ cplx cconj(cplx a) { return make_double2(a.x, -a.y); }
__device__ __forceinline__ cplx cmulmi(cplx a) { return make_double2(a.y, -a.x); }  // a * (-i)
__device__ __forceinline__ cplx csq(cplx a) { return make_double2(fma(a.x, a.x, -a.y * a.y), (a.x + a.x) * a.y); }
__device__ __forceinline__ double2 d2(double x, double y) { return make_double2(x, y); }
__device__ __forceinline__ double2 d2fma(double2 a, double2 b, double2 c) { return make_double2(fma(a.x, b.x, c.x), fma(a.y, b.y, c.y)); }

// ---------------------------------------------------------------------------------------------
// Shared-memory layout of the resident lanes = the slab layout: tile J holds [lane][4 positions].
// ---------------------------------------------------------------------------------------------
template <int LN> struct Lay {
  static constexpr int LOG = (LN == 4) ? 2 : 1;   // log2 LN
  static constexpr int LSH = LOG + 1;             // log2 (16-byte pieces per tile)
  // pair p = elements (2p, 2p+1) of a lane, in double2 units relative to the lane's base (W2 + 2*lane)
  static __device__ __forceinline__ int pix(int p) { return (p >> 1) * (1 << LSH) + (p & 1); }
  // element e of a lane, in double units relative to the lane's base (W + 4*lane)
  static __device__ __forceinline__ int eix(int e) { return (e >> 2) * (1 << (LSH + 1)) + (e & 3); }
};

// ---------------------------------------------------------------------------------------------
// Radix-R DFT in registers (forward, e^{-2 pi i jk/R}), natural order in and out.
// ---------------------------------------------------------------------------------------------
template <int R> struct Dft;
template <> struct Dft<1> { static __device__ __forceinline__ void run(cplx*) {} };
template <> struct Dft<2> {
  static __device__ __forceinline__ void run(cplx* v) {
    cplx a = v[0], b = v[1];
    v[0] = cadd(a, b);
    v[1] = csub(a, b);
  }
};
template <> struct Dft<4> {
  static __device__ __forceinline__ void run(cplx* v) {
    cplx t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
    cplx t2 = cadd(v[1], v[3]), t3 = cmulmi(csub(v[1], v[3]));
    v[0] = cadd(t0, t2);
    v[1] = cadd(t1, t3);
    v[2] = csub(t0, t2);
    v[3] = csub(t1, t3);
  }
};
template <> struct Dft<8> {
  static __device__ __forceinline__ void run(cplx* v) {
    cplx e[4] = {v[0], v[2], v[4], v[6]}, o[4] = {v[1], v[3], v[5], v[7]};
    Dft<4>::run(e);
    Dft<4>::run(o);
    const double h = 0.70710678118654752440;
    cplx t1 = make_double2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));   // * e^{-i pi/4}
    cplx t2 = cmulmi(o[2]);                                                 // * (-i)
    cplx t3 = make_double2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));  // * e^{-3i pi/4}
    v[0] = cadd(e[0], o[0]); v[4] = csub(e[0], o[0]);
    v[1] = cadd(e[1], t1);   v[5] = csub(e[1], t1);
    v[2] = cadd(e[2], t2);   v[6] = csub(e[2], t2);
    v[3] = cadd(e[3], t3);   v[7] = csub(e[3], t3);
  }
};
template <> struct Dft<16> {
  static __device__ __forceinline__ void run(cplx* v) {
    cplx e[8], o[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { e[i] = v[2 * i]; o[i] = v[2 * i + 1]; }
    Dft<8>::run(e);
    Dft<8>::run(o);
    const double c1 = 0.92387953251128675613, s1 = 0.38268343236508977173, h = 0.70710678118654752440;
    const cplx w[8] = {{1, 0}, {c1, -s1}, {h, -h}, {s1, -c1}, {0, -1}, {-s1, -c1}, {-h, -h}, {-c1, -s1}};
    v[0] = cadd(e[0], o[0]); v[8] = csub(e[0], o[0]);
#pragma unroll
    for (int k = 1; k < 8; k++) {
      cplx t = (k == 4) ? cmulmi(o[4]) : cmul(w[k], o[k]);
      v[k] = cadd(e[k], t);
      v[k + 8] = csub(e[k], t);
    }
  }
};

// v[r] *= w1^r for r = 1..R-1.  The powers are generated in registers from the one loaded twiddle (chain
// depth <= 4 multiplications, error a few ulp) instead of R-1 dependent table loads per butterfly.
template <int R> struct Twid;
template <> struct Twid<2> { static __device__ __forceinline__ void run(cplx* v, cplx w1) { v[1] = cmul(v[1], w1); } };
template <> struct Twid<4> {
  static __device__ __forceinline__ void run(cplx* v, cplx w1) {
    const cplx w2 = csq(w1);
    v[1] = cmul(v[1], w1); v[2] = cmul(v[2], w2); v[3] = cmul(v[3], cmul(w2, w1));
  }
};
template <> struct Twid<8> {
  static __device__ __forceinline__ void run(cplx* v, cplx w1) {
    const cplx w2 = csq(w1), w3 = cmul(w2, w1), w4 = csq(w2);
    v[1] = cmul(v[1], w1); v[2] = cmul(v[2], w2); v[3] = cmul(v[3], w3); v[4] = cmul(v[4], w4);
    v[5] = cmul(v[5], cmul(w4, w1)); v[6] = cmul(v[6], csq(w3)); v[7] = cmul(v[7], cmul(w4, w3));
  }
};
template <> struct Twid<16> {
  static __device__ __forceinline__ void run(cplx* v, cplx w1) {
    const cplx w2 = csq(w1), w3 = cmul(w2, w1), w4 = csq(w2);
    v[1] = cmul(v[1], w1); v[2] = cmul(v[2], w2); v[3] = cmul(v[3], w3); v[4] = cmul(v[4], w4);
    const cplx w5 = cmul(w4, w1), w7 = cmul(w4, w3), w8 = csq(w4);
    v[5] = cmul(v[5], w5); v[6] = cmul(v[6], csq(w3)); v[7] = cmul(v[7], w7); v[8] = cmul(v[8], w8);
    v[9] = cmul(v[9], cmul(w8, w1)); v[10] = cmul(v[10], csq(w5)); v[11] = cmul(v[11], cmul(w8, w3));
    v[12] = cmul(v[12], cmul(w8, w4)); v[13] = cmul(v[13], cmul(w8, w5)); v[14] = cmul(v[14], csq(w7));
    v[15] = cmul(v[15], cmul(w8, w7));
  }
};
template <int V> struct Log2 { static constexpr int v = 1 + Log2<V / 2>::v; };
template <> struct Log2<1> { static constexpr int v = 0; };

// ---------------------------------------------------------------------------------------------
// shuffle helpers for small structs of doubles
// ---------------------------------------------------------------------------------------------
template <int K> struct DVec { double d[K]; };
template <int K> __device__ __forceinline__ DVec<K> shfl_up(const DVec<K>& m, int delta) {
  DVec<K> r;
#pragma unroll
  for (int i = 0; i < K; i++) r.d[i] = __shfl_up_sync(0xffffffffu, m.d[i], delta, 32);
  return r;
}
template <int K> __device__ __forceinline__ DVec<K> shfl_down(const DVec<K>& m, int delta) {
  DVec<K> r;
#pragma unroll
  for (int i = 0; i < K; i++) r.d[i] = __shfl_down_sync(0xffffffffu, m.d[i], delta, 32);
  return r;
}

// Affine maps used by the lane recurrences.  "then(f, s)" = apply f first, then s; "apply(m, v)" = m(v).
// First order, two independent parities:  y -> A y + B.      d = {A0,B0,A1,B1};  state = {y0, y1}
struct Aff1 {
  typedef DVec<4> V;
  typedef DVec<2> S;
  static __device__ __forceinline__ V identity() { V v; v.d[0] = 1; v.d[1] = 0; v.d[2] = 1; v.d[3] = 0; return v; }
  static __device__ __forceinline__ S zero() { S s; s.d[0] = 0; s.d[1] = 0; return s; }
  static __device__ __forceinline__ V then(const V& f, const V& s) {
    V r;
    r.d[0] = s.d[0] * f.d[0]; r.d[1] = fma(s.d[0], f.d[1], s.d[1]);
    r.d[2] = s.d[2] * f.d[2]; r.d[3] = fma(s.d[2], f.d[3], s.d[3]);
    return r;
  }
  static __device__ __forceinline__ S apply(const V& m, const S& v) {
    S r; r.d[0] = fma(m.d[0], v.d[0], m.d[1]); r.d[1] = fma(m.d[2], v.d[1], m.d[3]); return r;
  }
};
// Second order, two parities: state (u,w) -> P (u,w) + p.   d = {P00,P01,P10,P11,p0,p1} x 2;  state = {u0,w0,u1,w1}
struct Aff2 {
  typedef DVec<12> V;
  typedef DVec<4> S;
  static __device__ __forceinline__ V identity() {
    V v;
#pragma unroll
    for (int h = 0; h < 2; h++) { v.d[6*h+0] = 1; v.d[6*h+1] = 0; v.d[6*h+2] = 0; v.d[6*h+3] = 1; v.d[6*h+4] = 0; v.d[6*h+5] = 0; }
    return v;
  }
  static __device__ __forceinline__ S zero() { S s; s.d[0] = s.d[1] = s.d[2] = s.d[3] = 0; return s; }
  static __device__ __forceinline__ V then(const V& f, const V& s) {
    V r;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const double* F = f.d + 6 * h; const double* S_ = s.d + 6 * h; double* R = r.d + 6 * h;
      R[0] = S_[0] * F[0] + S_[1] * F[2]; R[1] = S_[0] * F[1] + S_[1] * F[3];
      R[2] = S_[2] * F[0] + S_[3] * F[2]; R[3] = S_[2] * F[1] + S_[3] * F[3];
      R[4] = S_[0] * F[4] + S_[1] * F[5] + S_[4];
      R[5] = S_[2] * F[4] + S_[3] * F[5] + S_[5];
    }
    return r;
  }
  static __device__ __forceinline__ S apply(const V& m, const S& v) {
    S r;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const double* M = m.d + 6 * h;
      r.d[2*h+0] = M[0] * v.d[2*h] + M[1] * v.d[2*h+1] + M[4];
      r.d[2*h+1] = M[2] * v.d[2*h] + M[3] * v.d[2*h+1] + M[5];
    }
    return r;
  }
};

// State entering each thread's chunk: the maps of the threads before it (PREFIX: q' < q, lowest applied first;
// SUFFIX: q' > q, highest applied first) applied to the zero state.  Threads of a lane sit LN apart in a warp
// (32/LN of them per warp); warp totals go through shared memory and ONE thread per lane runs the short
// serial recurrence over the warps (vector recurrence only -- no matrix products on the critical path).
// scratch: [warp totals tot: 16 warps * LN lanes * V][entry states ent at 16 * LN * sizeof(Aff2::V), the same offset for
// every map type: 16 * LN * S].  All threads of the CTA must call.
// Scratch invariant (callers run scans back to back without a barrier in between, e.g. the two scans of an LU solve):
// no scan's tot overlaps any scan's ent.  A warp reads its ent[w] after the scan's last barrier and nothing waits for that
// read, so a fast warp may already be writing the NEXT scan's tot while a slow one still reads ent.  ent itself is only
// written between the two barriers of a scan (by tid < LN), and every thread has read the previous scan's ent before it
// arrives at the first of them.
template <class M, bool SUFFIX, int LN>
__device__ __forceinline__ typename M::S lane_scan_state(typename M::V mine, int TPL, void* scratch) {
  typedef typename M::V V;
  typedef typename M::S S;
  static_assert(sizeof(V) <= sizeof(Aff2::V), "warp totals would overlap the entry states of another scan");
  static_assert(sizeof(S) <= sizeof(Aff2::S), "entry states would run past the scan scratch");
  static_assert(16 * 4 * (sizeof(Aff2::V) + sizeof(Aff2::S)) <= B2_SCRATCH, "scan scratch too small");
  constexpr int QW = 32 / LN;                    // threads of one lane inside a warp
  const int tid = threadIdx.x, l = tid & (LN - 1);
  const int qi = (tid & 31) >> Lay<LN>::LOG;     // position inside the warp's segment of the lane
  const int width = TPL < QW ? TPL : QW;
  V inc = mine;
#pragma unroll
  for (int d = 1; d < QW; d <<= 1) {
    if (d < width) {
      V o = SUFFIX ? shfl_down(inc, d * LN) : shfl_up(inc, d * LN);
      bool take = SUFFIX ? (qi + d < width) : (qi >= d);
      if (take) inc = M::then(o, inc);
    }
  }
  V exc = SUFFIX ? shfl_down(inc, LN) : shfl_up(inc, LN);
  if (SUFFIX ? (qi == width - 1) : (qi == 0)) exc = M::identity();
  if (TPL <= QW) return M::apply(exc, M::zero());
  const int nw = TPL / QW, w = tid >> 5;
  V* tot = reinterpret_cast<V*>(scratch);                  // [warp][lane] warp totals
  S* ent = reinterpret_cast<S*>(static_cast<char*>(scratch) + 16 * LN * sizeof(Aff2::V));   // [warp][lane] state entering the warp
  if (SUFFIX ? (qi == 0) : (qi == QW - 1)) tot[w * LN + l] = inc;
  __syncthreads();
  if (tid < LN) {
    S s = M::zero();
    if (SUFFIX) { for (int k = nw - 1; k >= 0; k--) { ent[k * LN + l] = s; s = M::apply(tot[k * LN + l], s); } }
    else        { for (int k = 0; k < nw; k++) { ent[k * LN + l] = s; s = M::apply(tot[k * LN + l], s); } }
  }
  __syncthreads();
  return M::apply(exc, ent[w * LN + l]);
}

// sum over the TPL threads of a lane (result valid in every thread of the lane)
template <int LN>
__device__ __forceinline__ double lane_sum(double v, int TPL, double* scratch) {
  constexpr int QW = 32 / LN;
  const int tid = threadIdx.x, l = tid & (LN - 1);
  const int width = TPL < QW ? TPL : QW;
  for (int d = width >> 1; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d * LN, 32);
  if (TPL > QW) {
    const int nw = TPL / QW, w = tid >> 5;
    if ((tid & 31) < LN) scratch[w * LN + l] = v;
    __syncthreads();
    double s = 0;
    for (int k = 0; k < nw; k++) s += scratch[k * LN + l];
    __syncthreads();
    v = s;
  }
  return v;
}

// ---------------------------------------------------------------------------------------------
// Shared memory: [mbarriers 512 B][program copy][scan scratch][W = LN lanes, slab layout][per-warp staging]
//   dfull          : a direct (zero-copy) load has landed in W
//   wbar[warp][s]  : sub-chunk slot s of a warp has been filled by the copy engine (combining loads)
// Every warp owns two staging slots of CHW (+1 halo) tiles and runs its OWN copy pipeline: the lane is cut into
// sub-chunks of CHW tiles, warp w takes sub-chunks w, w + nwarps, ...; lane 0 of the warp issues the bulk copies
// (async-group / mbarrier accounting is per thread), the other lanes only see __syncwarp.  16 independent pipelines keep
// ~80 KB in flight per SM without a single CTA barrier inside a load or a store (measured: the CTA-wide chunk loop
// with one issuing thread spent as long in its per-chunk barriers and slot waits as in the copies themselves).
// ---------------------------------------------------------------------------------------------
struct SmemView {
  uint64_t* dfull; uint64_t* wbar;
  void* scratch; double* W; char* st;
};
__device__ __forceinline__ SmemView smem_view(const LaneProg& P, char* base) {
  SmemView v;
  v.dfull = reinterpret_cast<uint64_t*>(base); v.wbar = v.dfull + 2;
  v.scratch = base + B2_BARBYTES + B2_PROGCOPY; v.W = reinterpret_cast<double*>(base + P.w_off); v.st = base + P.st_off;
  return v;
}
struct Prefetch {             // per-thread pipeline state
  int gl, lb;                 // this CTA's lane group / first lane
  unsigned dphase;            // parity of the direct-load barrier
  unsigned wph;               // parities of this warp's two slot barriers (bits 0, 1)
  int ws;                     // the staging slot this warp's next store sub-chunk goes to (slots alternate across ops as well)
};

// every thread that issues bulk stores waits for its own groups (whole CTA must call)
__device__ __forceinline__ void wait_all_stores_complete() {
  if ((threadIdx.x & 31) == 0) bulk_wait<0>();
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// loads
// ---------------------------------------------------------------------------------------------
// W = src: the slab lands in W as it is (zero-copy); elements at and beyond len are cleared afterwards.
template <int LN>
__device__ __noinline__ void load_direct(const LaneProg& P, const LaneOp& op, const B2TMap* tm, const SmemView& sv, Prefetch& pf) {
  if (op.i2 & LD_AFTER_STORE) wait_all_stores_complete();   // the source was stored by this CTA earlier in the program
  if (threadIdx.x == 0) {
    if (P.bulk1d) {
      const char* src = static_cast<const char*>(op.p0) + (size_t)pf.gl * P.in_tiles * 128;
      mbar_arrive_expect_tx(sv.dfull, (uint32_t)P.in_tiles * 128u);
      for (int t0 = 0; t0 < P.in_tiles; t0 += P.CHD) {
        const int t1 = min(t0 + P.CHD, P.in_tiles);
        bulk_load_1d(reinterpret_cast<char*>(sv.W) + (size_t)t0 * 128, src + (size_t)t0 * 128, (uint32_t)(t1 - t0) * 128u, sv.dfull);
      }
    } else {
      mbar_arrive_expect_tx(sv.dfull, (uint32_t)(P.nchd * P.CHD * LN * 32));
      for (int c = 0; c < P.nchd; c++)
        tma_load_3d(reinterpret_cast<char*>(sv.W) + (size_t)c * P.CHD * LN * 32, tm, pf.lb * 4, c * P.CHD, pf.gl, sv.dfull);
    }
  }
  mbar_wait(sv.dfull, pf.dphase);
  pf.dphase ^= 1u;
  const int len = op.i0, ntail = P.LP - len;
  for (int i = threadIdx.x; i < ntail * LN; i += P.NT) {
    const int l = i & (LN - 1), e = len + (i >> Lay<LN>::LOG);
    sv.W[4 * l + Lay<LN>::eix(e)] = 0.0;
  }
  __syncthreads();
}

// W = [W +|*] a * src (tiled source, same orientation), optionally with the composite -> orthonormal stencil applied on
// the way in (value_j = src_j + p1_j * src_{j-2}).  Per-warp pipeline: sub-chunk slot layout [tile t = 0..CHW][lane][4],
// t = 0 being the halo tile in front of the sub-chunk (the stencil reaches two elements back).
template <int LN>
__device__ __noinline__ void load_warps(const LaneProg& P, const LaneOp& op, const B2TMap* tm, const SmemView& sv, Prefetch& pf) {
  constexpr int LSH = Lay<LN>::LSH;
  const int len = op.i0, in_tiles = P.in_tiles, CHW = P.CHW, nsc = P.nsc, nw = P.NT >> 5;
  const int w = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const double a = op.a;
  const bool acc = op.i2 & LD_ACC, mul = op.i2 & LD_MUL, sten = op.i2 & LD_STENCIL;
  const double* sc = reinterpret_cast<const double*>(op.p1);
  double2* W2 = reinterpret_cast<double2*>(sv.W);
  char* slot0 = sv.st + (size_t)w * 2 * P.wslot_bytes;
  uint64_t* bar = sv.wbar + 2 * w;
  if (op.i2 & LD_AFTER_STORE) wait_all_stores_complete();
  else if (ln == 0) bulk_wait_read<0>();   // this warp's earlier stores may still be reading the slots
  auto request = [&](int c, int s) {       // lane 0: sub-chunk c -> slot s
    const int J0 = c * CHW;
    char* dst = slot0 + (size_t)s * P.wslot_bytes;
    if (P.bulk1d) {   // contiguous slab: tiles [J0-1, J0+CHW) clipped to the lane
      const int t0 = J0 > 0 ? J0 - 1 : 0, t1 = min(J0 + CHW, in_tiles);
      const uint32_t bytes = (uint32_t)(t1 - t0) * 128u;
      mbar_arrive_expect_tx(bar + s, bytes);
      bulk_load_1d(dst + (size_t)(t0 - (J0 - 1)) * 128, static_cast<const char*>(op.p0) + ((size_t)pf.gl * in_tiles + t0) * 128, bytes, bar + s);
    } else {
      mbar_arrive_expect_tx(bar + s, (uint32_t)((CHW + 1) * LN * 32));
      tma_load_3d(dst, tm, pf.lb * 4, J0 - 1, pf.gl, bar + s);
    }
  };
  __syncwarp();
  if (ln == 0) { if (w < nsc) request(w, 0); if (w + nw < nsc) request(w + nw, 1); }
  const int npc = CHW << LSH;
  int s = 0;
  for (int c = w; c < nsc; c += nw, s ^= 1) {
    mbar_wait(bar + s, (pf.wph >> s) & 1u);
    pf.wph ^= 1u << s;
    const double2* st = reinterpret_cast<const double2*>(slot0 + (size_t)s * P.wslot_bytes) + (1 << LSH);
    const int J0 = c * CHW;
#pragma unroll 3
    for (int pc = ln; pc < npc; pc += 32) {
      const int J = J0 + (pc >> LSH), j0 = 4 * J + 2 * (pc & 1);
      if (J >= in_tiles) break;
      double2 v = st[pc];
      if (sten && j0 >= 2) {
        const double2 u = (pc & 1) ? st[pc - 1] : st[pc - (1 << LSH) + 1];
        const double2 cf = ldg(reinterpret_cast<const double2*>(sc + j0));
        v.x = fma(cf.x, u.x, v.x); v.y = fma(cf.y, u.y, v.y);
      }
      v.x = (j0 < len) ? v.x * a : 0.0;
      v.y = (j0 + 1 < len) ? v.y * a : 0.0;
      double2* wp = W2 + ((size_t)J0 << LSH) + pc;
      if (acc) { const double2 ov = *wp; v.x += ov.x; v.y += ov.y; }
      else if (mul) { const double2 ov = *wp; v.x *= ov.x; v.y *= ov.y; }
      *wp = v;
    }
    __syncwarp();
    if (ln == 0 && c + 2 * nw < nsc) request(c + 2 * nw, s);
  }
  __syncthreads();
}

// Per-thread path (row-major "plain" sources written by the GEMM; everything when TMA is switched off).
template <int LN, int U>   // U = 16-byte global loads in flight per thread
__device__ __noinline__ void load_threads(const LaneProg& P, const LaneOp& op, const SmemView& sv, int gl, int lb) {
  constexpr int LSH = Lay<LN>::LSH;
  const int T = P.NT, len = op.i0;
  const int npieces = P.in_tiles << LSH;
  const double a = op.a;
  const bool acc = op.i2 & LD_ACC, mul = op.i2 & LD_MUL, plain = op.i2 & LD_PLAIN, sten = op.i2 & LD_STENCIL;
  const double2* src = reinterpret_cast<const double2*>(op.p0);
  const size_t slab = (size_t)gl * P.in_tiles * 8;  // in double2 units
  const double* sc = reinterpret_cast<const double*>(op.p1);
  double2* W2 = reinterpret_cast<double2*>(sv.W);
  const int psplit = (op.i2 & LD_PSPLIT) ? op.i1 : 0;   // rows < psplit of a plain source are stored parity-split
  if (op.i2 & LD_AFTER_STORE) wait_all_stores_complete();   // the source was written by this CTA's bulk stores
  for (int p0 = threadIdx.x; p0 < npieces; p0 += U * T) {
    double2 v[U], u[U];
#pragma unroll
    for (int k = 0; k < U; k++) {
      const int pc = p0 + k * T;
      const int J = pc >> LSH, l = (pc >> 1) & (LN - 1), j0 = 4 * J + (pc & 1) * 2;
      v[k] = make_double2(0.0, 0.0); u[k] = make_double2(0.0, 0.0);
      if (pc < npieces && j0 < len) {
        int row = 4 * gl + lb + l;
        if (row < psplit) row = (row & 1) ? ((psplit + 1) >> 1) + (row >> 1) : (row >> 1);
        if (plain && (op.i2 & LD_PSPLITC) && j0 <= op.i1) {   // elements j0 (even) and j0+1 (odd) live in the two parity halves
          const double* sd = reinterpret_cast<const double*>(op.p0) + (size_t)row * P.in_tiles * 4;
          v[k] = make_double2(sd[j0 >> 1], sd[((op.i1 + 1) >> 1) + (j0 >> 1)]);
        } else
        v[k] = plain ? src[((size_t)row * P.in_tiles * 4 + j0) >> 1]
                     : src[slab + (size_t)J * 8 + (lb + l) * 2 + (pc & 1)];
        if (sten && j0 >= 2) {   // composite -> orthonormal on the fly: + p1[j] * src[j-2]  (tiled sources only)
          const int jm = j0 - 2;
          u[k] = src[slab + ((size_t)(jm >> 2) * 16 + (lb + l) * 4 + (jm & 3)) / 2];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < U; k++) {
      const int pc = p0 + k * T;
      if (pc >= npieces) break;
      const int j0 = 4 * (pc >> LSH) + (pc & 1) * 2;
      double2 x = v[k];
      if (sten && j0 >= 2 && j0 < len) { x.x = fma(sc[j0], u[k].x, x.x); x.y = fma(sc[j0 + 1], u[k].y, x.y); }
      x.x *= a;
      x.y = (j0 + 1 < len) ? x.y * a : 0.0;
      double2* w = W2 + pc;
      if (acc) { double2 ov = *w; x.x += ov.x; x.y += ov.y; }
      else if (mul) { double2 ov = *w; x.x *= ov.x; x.y *= ov.y; }
      *w = x;
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// stores
// ---------------------------------------------------------------------------------------------
// dst = W, same orientation: W leaves as it is (zero-copy) once its tail (>= len) is cleared.
template <int LN>
__device__ __noinline__ void store_direct(const LaneProg& P, const LaneOp& op, const B2TMap* tm, const SmemView& sv, int g, int gl, int lb) {
  const int len = op.i0, ntail = P.LP - len;
  for (int i = threadIdx.x; i < ntail * LN; i += P.NT) {
    const int l = i & (LN - 1), e = len + (i >> Lay<LN>::LOG);
    sv.W[4 * l + Lay<LN>::eix(e)] = 0.0;
  }
  fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) {
    if (op.i2 & ST_COLSPLIT) {   // (bulk1d only) one run of tiles per owner, straight from W into the owner's array
      const int tpr = P.groups_per_rank;
      char* const* peers = reinterpret_cast<char* const*>(op.p1);
      const size_t off = static_cast<const char*>(op.p0) - peers[P.rank];
      for (int o = 0; o * tpr < P.in_tiles; o++)
        for (int t0 = o * tpr; t0 < (o + 1) * tpr; t0 += P.CHD) {
          const int t1 = min(t0 + P.CHD, (o + 1) * tpr);
          bulk_store_1d(peers[o] + off + ((size_t)g * tpr + (t0 - o * tpr)) * 128, reinterpret_cast<const char*>(sv.W) + (size_t)t0 * 128, (uint32_t)(t1 - t0) * 128u);
        }
    } else if (P.bulk1d) {
      char* dst = static_cast<char*>(const_cast<void*>(op.p0)) + (size_t)gl * P.in_tiles * 128;
      for (int c = 0; c < P.nchd; c++) {
        const int t0 = c * P.CHD, t1 = min(t0 + P.CHD, P.in_tiles);
        bulk_store_1d(dst + (size_t)t0 * 128, reinterpret_cast<const char*>(sv.W) + (size_t)t0 * 128, (uint32_t)(t1 - t0) * 128u);
      }
    } else {
      for (int c = 0; c < P.nchd; c++)
        tma_store_3d(tm, lb * 4, c * P.CHD, gl, reinterpret_cast<const char*>(sv.W) + (size_t)c * P.CHD * LN * 32);
    }
    bulk_commit();
    bulk_wait_read<0>();   // W is rewritten by whatever comes next
  }
  __syncthreads();
}

// dst = [dst +] a * W through the warps' staging slots and bulk tensor stores / reductions.  Transposing stores transpose
// each 4x4 tile on its way into the slot ([tile][jl][lane]) and leave as ONE 4-D tensor store per sub-chunk: full 128-byte
// lines into the transposed array -- with several GPUs into the slab of the rank that owns those rows (the pencil
// transpose), one tensor map per owner, sub-chunks that straddle two owners stored twice and clipped by the copy engine.
template <int LN>
__device__ __noinline__ void store_warps(const LaneProg& P, const LaneOp& op, const B2TMap* tm, const SmemView& sv, int g, int gl, int lb, Prefetch& pf) {
  constexpr int LSH = Lay<LN>::LSH, HL = LN / 2;
  const int len = op.i0, flags = op.i2, in_tiles = P.in_tiles, CHW = P.CHW, nsc = P.nsc, nw = P.NT >> 5;
  const int w = threadIdx.x >> 5, ln = threadIdx.x & 31;
  const double a = op.a;
  const double* W = sv.W;
  const double2* W2 = reinterpret_cast<const double2*>(sv.W);
  char* slot0 = sv.st + (size_t)w * 2 * P.wslot_bytes;
  const int npc = CHW << LSH;
  int s = pf.ws;
  for (int c = w; c < nsc; c += nw, s ^= 1) {
    double2* st = reinterpret_cast<double2*>(slot0 + (size_t)s * P.wslot_bytes);
    const int J0 = c * CHW;
    if (ln == 0) bulk_wait_read<1>();   // only the store of the OTHER slot may still be reading (slots alternate, across ops too)
    __syncwarp();
    if (flags & ST_TRANS) {
      // piece (tile, jl, lane pair lp) = elements (2lp, jl), (2lp+1, jl); odd tiles read the two in the opposite order so
      // that the 16 threads of a half-warp touch 16 different 8-byte banks
#pragma unroll 3
      for (int pc = ln; pc < npc; pc += 32) {
        const int lp = pc & (HL - 1), jl = (pc / HL) & 3, tt = pc >> LSH;
        const int j = 4 * (J0 + tt) + jl, sw = tt & 1;
        double2 v = make_double2(0.0, 0.0);
        if (j < len) {
          const double* wt = W + ((size_t)(J0 + tt) << (LSH + 1)) + jl;
          const double e0 = wt[4 * (2 * lp + sw)], e1 = wt[4 * (2 * lp + 1 - sw)];
          v.x = a * (sw ? e1 : e0); v.y = a * (sw ? e0 : e1);
        }
        st[pc] = v;
      }
    } else {                  // slot layout [tile][lane][4]: the slab itself
#pragma unroll 3
      for (int pc = ln; pc < npc; pc += 32) {
        const int j0 = 4 * (J0 + (pc >> LSH)) + 2 * (pc & 1);
        double2 v = make_double2(0.0, 0.0);
        if (j0 < len) {
          const double2 wv = W2[((size_t)J0 << LSH) + pc];
          v.x = a * wv.x; v.y = (j0 + 1 < len) ? a * wv.y : 0.0;
        }
        st[pc] = v;
      }
    }
    fence_proxy_async();
    __syncwarp();
    // Several GPUs: a sub-chunk whose box lies completely inside ONE owner's view of the transposed array leaves as one tensor
    // store into that owner's slab.  A box that straddles two owners or overhangs the end of the view is NOT handed to the copy
    // engine (partly out-of-bounds tensor stores on peer memory faulted on hardware): the warp writes those few tiles itself.
    bool peer_irregular = false;
    if ((flags & ST_TRANS) && (flags & ST_PEER)) {
      const int gpr = P.groups_per_rank, o0 = J0 / gpr;
      peer_irregular = (J0 + CHW > (o0 + 1) * gpr) || (J0 + CHW > in_tiles);
      if (peer_irregular) {
        char* const* peers = reinterpret_cast<char* const*>(op.p1);
        const size_t off = static_cast<const char*>(op.p0) - peers[P.rank];
        for (int pc = ln; pc < npc; pc += 32) {
          const int tt = pc >> LSH, J = J0 + tt;
          if (J >= in_tiles) break;
          const int o = J / gpr;
          // destination tile (J - o gpr, g) of owner o: [jl][lane]; slot piece pc & (2^LSH - 1) = (jl, lane pair)
          double* d = reinterpret_cast<double*>(peers[o] + off) + ((size_t)(J - o * gpr) * P.out_tiles + g) * 16
                      + ((pc & ((1 << LSH) - 1)) / HL) * 4 + lb + 2 * (pc & (HL - 1));
          const double2 v = st[pc];
          if (flags & ST_ACC) { atomicAdd(d, v.x); atomicAdd(d + 1, v.y); }
          else *reinterpret_cast<double2*>(d) = v;
        }
      }
    }
    if (ln == 0) {
      // whole lane groups (LN == 4): a destination tile is 128 contiguous bytes, and the view says so ([16][tile column][tile
      // row]: one 128-byte row per tile)
      if (peer_irregular) {
        // (an empty group keeps the slot accounting of bulk_wait_read uniform)
      } else if ((flags & ST_TRANS) && (flags & ST_PEER)) {
        const int gpr = P.groups_per_rank, o = J0 / gpr;
        if (LN == 4) { if (flags & ST_ACC) tma_reduce_add_3d(tm + o, 0, g, J0 - o * gpr, st); else tma_store_3d(tm + o, 0, g, J0 - o * gpr, st); }
        else if (flags & ST_ACC) tma_reduce_add_4d(tm + o, lb, 0, g, J0 - o * gpr, st); else tma_store_4d(tm + o, lb, 0, g, J0 - o * gpr, st);
      } else if (flags & ST_TRANS) {
        if (LN == 4) { if (flags & ST_ACC) tma_reduce_add_3d(tm, 0, g, J0, st); else tma_store_3d(tm, 0, g, J0, st); }
        else if (flags & ST_ACC) tma_reduce_add_4d(tm, lb, 0, g, J0, st); else tma_store_4d(tm, lb, 0, g, J0, st);
      } else if (P.bulk1d) {
        char* dst = static_cast<char*>(const_cast<void*>(op.p0)) + ((size_t)gl * in_tiles + J0) * 128;
        const uint32_t bytes = (uint32_t)(min(J0 + CHW, in_tiles) - J0) * 128u;
        if (flags & ST_ACC) bulk_reduce_add_1d(dst, st, bytes); else bulk_store_1d(dst, st, bytes);
      } else {
        if (flags & ST_ACC) tma_reduce_add_3d(tm, lb * 4, J0, gl, st); else tma_store_3d(tm, lb * 4, J0, gl, st);
      }
      bulk_commit();
    }
  }
  pf.ws = s;
  __syncthreads();   // every warp has read its part of W
}

// Per-thread path: row-major "plain" destinations (GEMM operands), peer GPUs' slabs, TMA switched off.
template <int LN>
__device__ __noinline__ void store_threads(const LaneProg& P, const LaneOp& op, const SmemView& sv, int g, int gl, int lb) {
  constexpr int LSH = Lay<LN>::LSH, HL = LN / 2;
  const int T = P.NT, len = op.i0, flags = op.i2;
  const int npieces = P.in_tiles << LSH;
  const double a = op.a;
  const double* W = sv.W;
  const double2* W2 = reinterpret_cast<const double2*>(sv.W);
  double2* dst = reinterpret_cast<double2*>(const_cast<void*>(op.p0));
  if (flags & ST_TRANS) {
    double* const* peers = reinterpret_cast<double* const*>(op.p1);
    // ST_PSPLITC (GEMM operands of the parity-block Poisson products): the lane index is the column of the plain
    // matrix; lanes (0, 2) of the group are neighbouring even columns, lanes (1, 3) neighbouring odd columns
    const bool csplit = (flags & ST_PSPLITC) && LN == 4 && 4 * g + 3 <= op.i1;
    for (int pc = threadIdx.x; pc < npieces; pc += T) {
      const int lp = pc & (HL - 1), jl = (pc / HL) & 3, J = pc >> LSH, j = 4 * J + jl, sw = J & 1;
      double2 v = make_double2(0.0, 0.0);
      if (j < len) {
        const double* wt = W + ((size_t)J << (LSH + 1)) + jl;
        if (csplit) { v.x = a * wt[4 * lp]; v.y = a * wt[4 * (lp + 2)]; }
        else {
          const double e0 = wt[4 * (2 * lp + sw)], e1 = wt[4 * (2 * lp + 1 - sw)];
          v.x = a * (sw ? e1 : e0); v.y = a * (sw ? e0 : e1);
        }
      }
      double2* d = dst;
      int Jl = J;
      if (flags & ST_PEER) {  // row block J of the transposed array lives on rank J / groups_per_rank
        int owner = J / P.groups_per_rank;
        Jl = J - owner * P.groups_per_rank;
        d = reinterpret_cast<double2*>(reinterpret_cast<char*>(peers[owner]) +
                                       (reinterpret_cast<const char*>(op.p0) - reinterpret_cast<const char*>(peers[P.rank])));
      }
      // tiled: tile (Jl, g) holds [jl][l];  row-major ("plain", for the GEMM): row 4*Jl+jl, columns 4g+l
      const int col = csplit ? (lp ? ((op.i1 + 1) >> 1) : 0) + 2 * g : 4 * g + lb + 2 * lp;
      size_t idx = (flags & ST_PLAIN) ? (((size_t)(4 * Jl + jl) * P.out_tiles * 4 + col) >> 1)
                                      : ((((size_t)Jl * P.out_tiles + g) * 16 + jl * 4 + lb + 2 * lp) >> 1);
      if (flags & ST_ACC) { double2 ov = d[idx]; v.x += ov.x; v.y += ov.y; }
      d[idx] = v;
    }
  } else {
    const size_t slab = (size_t)gl * P.in_tiles * 8;
    for (int pc = threadIdx.x; pc < npieces; pc += T) {
      const int J = pc >> LSH, l = (pc >> 1) & (LN - 1), j0 = 4 * J + (pc & 1) * 2;
      double2 v = make_double2(0.0, 0.0);
      if (j0 < len) {
        const double2 w = W2[pc];
        v.x = a * w.x;
        v.y = (j0 + 1 < len) ? a * w.y : 0.0;
      }
      int row = 4 * gl + lb + l;
      if ((flags & ST_PSPLIT) && row < op.i1) row = (row & 1) ? ((op.i1 + 1) >> 1) + (row >> 1) : (row >> 1);
      if (flags & ST_COLSPLIT) {   // tile J of global group g -> owner J / tpr, tile (g, J mod tpr) of its [all rows][local columns] array
        const int tpr = P.groups_per_rank, o = J / tpr;
        char* const* peers = reinterpret_cast<char* const*>(op.p1);
        double2* d = reinterpret_cast<double2*>(peers[o] + (static_cast<const char*>(op.p0) - peers[P.rank]));
        d[((size_t)g * tpr + (J - o * tpr)) * 8 + (lb + l) * 2 + (pc & 1)] = v;
        continue;
      }
      size_t idx = (flags & ST_PLAIN) ? (((size_t)row * P.in_tiles * 4 + j0) >> 1)
                                      : (slab + (size_t)J * 8 + (lb + l) * 2 + (pc & 1));
      if (flags & ST_ACC) { double2 ov = dst[idx]; v.x += ov.x; v.y += ov.y; }
      dst[idx] = v;
    }
  }
  __syncthreads();
}

// ---- chunked lane ops -------------------------------------------------------------------------
// Thread q of a lane owns CP consecutive PAIRS (2p, 2p+1), p = q*CP + t.  All banded operators of the
// path couple elements at even distance only, so every recurrence is a plain double2 recurrence over
// pairs (no parity bookkeeping).  CP = E+1 is odd and the threads of a warp are lane-fastest, so
// the 8 threads of a quarter-warp hit 8 different 16-byte banks; coefficient vectors are stored
// "pair/scan" ordered, [t][q] as double2 -- one broadcast request serves the LN lanes of a q.
template <int CP, int LN>
__device__ __noinline__ void op_band(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  // y_i = sum_m c_m[i] x_{i+o_m}, o_m even.  Thread q of a lane takes the pairs p = q + t*TPL (coalesced
  // coefficient loads in natural order); results are staged in registers because the operation is in place.
  const int TPL = P.TPL, HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int len_out = op.i0;
  const int h0 = (int)(signed char)(op.i1 & 0xff), h1 = (int)(signed char)((op.i1 >> 8) & 0xff), h2 = (int)(signed char)((op.i1 >> 16) & 0xff);
  const double2* __restrict__ c0 = (const double2*)op.p0;
  const double2* __restrict__ c1 = (const double2*)op.p1;
  const double2* __restrict__ c2 = (const double2*)op.p2;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  const double2 zero = d2(0.0, 0.0);
  double2 y[CP];
#pragma unroll
  for (int t = 0; t < CP; t++) y[t] = zero;
  auto term = [&](int h, const double2* __restrict__ c) {
    const int hp = h >> 1;
#pragma unroll
    for (int t = 0; t < CP; t++) {
      const int p = q + t * TPL, pp = p + hp;
      const bool ok = pp >= 0 && pp < HP && p < HP;
      const double2 x = w2[Lay<LN>::pix(ok ? pp : 0)];
      const double2 cc = c ? ldg(c + (p < HP ? p : 0)) : d2(1.0, 1.0);
      if (ok) y[t] = d2fma(cc, x, y[t]);
    }
  };
  if (h0 != 127) term(h0, c0);
  if (h1 != 127) term(h1, c1);
  if (h2 != 127) term(h2, c2);
  __syncthreads();
#pragma unroll
  for (int t = 0; t < CP; t++) {
    const int p = q + t * TPL;
    double2 v = y[t];
    if (2 * p >= len_out) v.x = 0.0;
    if (2 * p + 1 >= len_out) v.y = 0.0;
    if (p < HP) w2[Lay<LN>::pix(p)] = v;
  }
  __syncthreads();
}

// Chebyshev derivative: b_k = S_{k+1},  S_m = 2 m a_m + S_{m+2};  b_0 *= 1/2;  result * scale.
// In pairs: S[p] = (2(2p) a_2p, 2(2p+1) a_2p+1) + S[p+1];  out[p] = (S[p].y, S[p+1].x).
template <int CP, int LN>
__device__ __noinline__ void op_deriv(const LaneProg& P, const LaneOp& op, double* __restrict__ W, void* scratch) {
  const int TPL = P.TPL, HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  for (int rep = 0; rep < op.i1; rep++) {
    double2 tp[CP];
    double2 tot = d2(0.0, 0.0);
#pragma unroll
    for (int t = 0; t < CP; t++) {
      const int p = q * CP + t;
      double2 a = (p < HP) ? w2[Lay<LN>::pix(p < HP ? p : 0)] : d2(0.0, 0.0);
      tp[t] = d2(2.0 * (2 * p) * a.x, 2.0 * (2 * p + 1) * a.y);
      tot.x += tp[t].x; tot.y += tp[t].y;
    }
    Aff1::V m; m.d[0] = 1; m.d[1] = tot.x; m.d[2] = 1; m.d[3] = tot.y;
    Aff1::S in = lane_scan_state<Aff1, true, LN>(m, TPL, scratch);
    double2 S = d2(in.d[0], in.d[1]);   // S of the first pair of the next chunk
    const double sc = (rep == op.i1 - 1) ? op.a : 1.0;
#pragma unroll
    for (int t = CP - 1; t >= 0; t--) {
      const int p = q * CP + t;
      const double nx = S.x;
      S.x += tp[t].x; S.y += tp[t].y;
      double2 o = d2(S.y * sc, nx * sc);
      if (p == 0) o.x *= 0.5;
      if (p < HP) w2[Lay<LN>::pix(p)] = o;
    }
    __syncthreads();
  }
}

// In-place solve of the LU-factored 4-diagonal (-2,0,+2,+4) system (reference: src/solver/fdma.rs:101-118):
//   forward:  x_i -= fl_i x_{i-2}                     (fl_i = swept low_{i-2})
//   backward: x_i = (x_i - u1_i x_{i+2} - u2_i x_{i+4}) * id_i
// As pair recurrences: y_p = b_p - fl_p * y_{p-1};  x_p = (y_p - u1_p x_{p+1} - u2_p x_{p+2}) id_p.
// Each thread reduces its CP pairs to an affine map; maps are combined by a scan across the lane's threads.
// The four chunk loops stay rolled: the sm_90a build with `#pragma unroll 6` solved wrongly on lanes of 64 points or more
// (O(1) errors in from_ortho / HholtzAdi; the same source is exact in the CPU emulator and with the loops rolled).
template <int CP, int LN>
__device__ __noinline__ void op_fdma(const LaneProg& P, const LaneOp& op, double* __restrict__ W, int gl, int lb, void* scratch) {
  const int TPL = P.TPL, HP = P.LP >> 1;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int n = op.i0;
  double2* w2 = reinterpret_cast<double2*>(W) + 2 * l;
  const double2* __restrict__ cfl = (const double2*)op.p0; const double2* __restrict__ cid = (const double2*)op.p1;
  const double2* __restrict__ cu1 = (const double2*)op.p2; const double2* __restrict__ cu2 = (const double2*)op.p3;
  // shared vectors: [t][q]; per-lane arrays: [group][t][q][lane of 4]  (double2 units, coalesced at every step)
  size_t base; int stride;
  if (op.i2 & FD_PERLANE) { stride = 4 * TPL; base = ((size_t)gl * CP * TPL + q) * 4 + lb + l; }
  else { stride = TPL; base = q; }
  const bool nou2 = op.i2 & FD_NOU2;
  const double2 zero = d2(0.0, 0.0);
  const int p0 = q * CP;
  auto rd = [&](int t) -> double2 {   // right-hand side / intermediate at pair p0+t, zero outside [0, n)
    const int p = p0 + t;
    const bool ok = p < HP;
    double2 v = ok ? w2[Lay<LN>::pix(ok ? p : 0)] : zero;
    if (2 * p >= n) v.x = 0.0;
    if (2 * p + 1 >= n) v.y = 0.0;
    return v;
  };
  // ---- forward elimination: y_p = b_p - fl_p y_{p-1} ----
  {
    double2 A = d2(1.0, 1.0), B = zero;
#pragma unroll 1
    for (int t = 0; t < CP; t++) {
      const double2 f = ldg(cfl + base + (size_t)t * stride), b = rd(t);
      B = d2(fma(-f.x, B.x, b.x), fma(-f.y, B.y, b.y));
      A = d2(-f.x * A.x, -f.y * A.y);
    }
    Aff1::V m; m.d[0] = A.x; m.d[1] = B.x; m.d[2] = A.y; m.d[3] = B.y;
    Aff1::S in = lane_scan_state<Aff1, false, LN>(m, TPL, scratch);
    double2 y = d2(in.d[0], in.d[1]);   // y of the last pair before this chunk (the start state is 0)
#pragma unroll 1
    for (int t = 0; t < CP; t++) {
      const double2 f = ldg(cfl + base + (size_t)t * stride), b = rd(t);
      y = d2(fma(-f.x, y.x, b.x), fma(-f.y, y.y, b.y));
      if (p0 + t < HP) w2[Lay<LN>::pix(p0 + t)] = y;
    }
  }
  // every thread only touched its own chunk of W: no barrier needed before the back substitution.  The scan scratch needs none
  // either: the back substitution's warp totals never overlap the entry states a slower warp may still be reading from the
  // forward scan (lane_scan_state)
  // ---- back substitution: x_p = (y_p - u1_p x_{p+1} - u2_p x_{p+2}) id_p ----
  {
    Aff2::V m = Aff2::identity();
#pragma unroll 1
    for (int t = CP - 1; t >= 0; t--) {
      const size_t k = base + (size_t)t * stride;
      const double2 idv = ldg(cid + k), u1 = ldg(cu1 + k), u2 = nou2 ? zero : ldg(cu2 + k), y = rd(t);
      const double2 m0 = d2(-u1.x * idv.x, -u1.y * idv.y), m1 = d2(-u2.x * idv.x, -u2.y * idv.y), g0 = d2(y.x * idv.x, y.y * idv.y);
      double* M = m.d;   // compose onto the chunk map; state = (x_{p+1}, x_{p+2}) per component
      double r0 = m0.x * M[0] + m1.x * M[2], r1 = m0.x * M[1] + m1.x * M[3], rp = m0.x * M[4] + m1.x * M[5] + g0.x;
      M[2] = M[0]; M[3] = M[1]; M[5] = M[4]; M[0] = r0; M[1] = r1; M[4] = rp;
      M = m.d + 6;
      r0 = m0.y * M[0] + m1.y * M[2]; r1 = m0.y * M[1] + m1.y * M[3]; rp = m0.y * M[4] + m1.y * M[5] + g0.y;
      M[2] = M[0]; M[3] = M[1]; M[5] = M[4]; M[0] = r0; M[1] = r1; M[4] = rp;
    }
    Aff2::S in = lane_scan_state<Aff2, true, LN>(m, TPL, scratch);
    double2 s1 = d2(in.d[0], in.d[2]), s2 = d2(in.d[1], in.d[3]);   // x_{p+1}, x_{p+2} entering the chunk
#pragma unroll 1
    for (int t = CP - 1; t >= 0; t--) {
      const size_t k = base + (size_t)t * stride;
      const double2 idv = ldg(cid + k), u1 = ldg(cu1 + k), u2 = nou2 ? zero : ldg(cu2 + k), y = rd(t);
      double2 x = d2((y.x - u1.x * s1.x - u2.x * s2.x) * idv.x, (y.y - u1.y * s1.y - u2.y * s2.y) * idv.y);
      s2 = s1; s1 = x;
      if (p0 + t < HP) w2[Lay<LN>::pix(p0 + t)] = x;
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// complex FFT of Nc points per lane, in place in shared memory (Stockham autosort, register-staged:
// every thread reads its E points, the CTA syncs, then everything is written back).  Complex point i of a
// lane is pair i of that lane.  tw[t] = exp(-2 pi i t / Nc)
// ---------------------------------------------------------------------------------------------
// One Stockham pass.  FIRST: Ns == 1 (no twiddles).  The Ns == 1 pass scatters each thread's R results to R
// consecutive points (neighbouring q's write points of equal parity = the same bank pair): it writes point i at
// i ^ ((i >> log2 E) & swz) and the following pass reads through the same map (swz = 1), which restores the
// alternation; both sides are then conflict-free.
template <int E, int R, bool FIRST, int LN>
__device__ __forceinline__ void fft_stage(double2* __restrict__ wl, int Nc, int Ns, int q, int TPL, const cplx* __restrict__ tw,
                                          int swz_in, int swz_out) {
  constexpr int NB = E / R, LE = Log2<E>::v;
  cplx v[E];
  cplx w1[NB];
  const int stride = Nc / R;
#pragma unroll
  for (int b = 0; b < NB; b++) {
    const int j = q + b * TPL;
    if (!FIRST) w1[b] = ldg(tw + (j & (Ns - 1)) * (stride / Ns));   // issued ahead of the barrier
#pragma unroll
    for (int r = 0; r < R; r++) {
      int i = j + r * stride;
      i ^= (i >> LE) & swz_in;
      v[b * R + r] = wl[Lay<LN>::pix(i)];
    }
  }
  __syncthreads();
#pragma unroll
  for (int b = 0; b < NB; b++) {
    const int j = q + b * TPL;
    const int k = j & (Ns - 1);
    if (!FIRST) Twid<R>::run(v + b * R, w1[b]);
    Dft<R>::run(v + b * R);
    const int j0 = (j - k) * R + k;
#pragma unroll
    for (int r = 0; r < R; r++) {
      int i = j0 + r * Ns;
      i ^= (i >> LE) & swz_out;
      wl[Lay<LN>::pix(i)] = v[b * R + r];
    }
  }
  __syncthreads();
}

template <int E, int LN>
__device__ __forceinline__ void lane_fft(double* __restrict__ W, int Nc, int TPL, const cplx* __restrict__ tw) {
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  double2* wl = reinterpret_cast<double2*>(W) + 2 * l;
  // radix plan: as many radix-E passes as fit, then one pass with the remainder (1, 2, 4 or 8)
  int swz = (Nc > E) ? 1 : 0;
  fft_stage<E, E, true, LN>(wl, Nc, 1, q, TPL, tw, 0, swz);
  int Ns = E;
  while (Nc / Ns >= E) { fft_stage<E, E, false, LN>(wl, Nc, Ns, q, TPL, tw, swz, 0); swz = 0; Ns *= E; }
  const int rem = Nc / Ns;
  if constexpr (E >= 16) { if (rem == 8) fft_stage<E, 8, false, LN>(wl, Nc, Ns, q, TPL, tw, swz, 0); }
  if constexpr (E >= 8) { if (rem == 4) fft_stage<E, 4, false, LN>(wl, Nc, Ns, q, TPL, tw, swz, 0); }
  if (rem == 2) fft_stage<E, 2, false, LN>(wl, Nc, Ns, q, TPL, tw, swz, 0);
}

// Chebyshev transform (DCT-I of n = N+1 points on Gauss-Lobatto nodes x_j = -cos(pi j/N)) through ONE
// complex FFT of N/2 points (SURVEY A.1):
//   mode 0 (forward):  c_k = (-1)^k X_k / N, c_0 and c_N halved,  X = DCT-I(v)
//   mode 1 (backward): v = DCT-I(y)/2, y_k = (-1)^k c_k, y_0 and y_N doubled
// tw: exp(-2 pi i t/(N/2)), tw2[j] = exp(-2 pi i j/N) (j <= N/2), isin[k] = 1/(4 sin(pi k/N))
template <int E, int LN>
__device__ __noinline__ void op_dct(const LaneProg& P, const LaneOp& op, double* __restrict__ W, double* scratch) {
  const int TPL = P.TPL;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int N = op.i0 - 1, M = N >> 1, mode = op.i1;
  const cplx* tw = (const cplx*)op.p0; const cplx* tw2 = (const cplx*)op.p1; const double* isin = (const double*)op.p2;
  double* w = W + 4 * l;
  cplx* w2 = reinterpret_cast<cplx*>(W) + 2 * l;
  constexpr int NP = E / 2 + 1;
  // ---- pre: x -> g (N/2 complex), pairs (j, M-j); branch-free, 16-byte shared-memory reads ----
  cplx gj[NP], gm[NP];
  double r0 = 0.0;
  const double sg = (mode == 1) ? -1.0 : 1.0, endf = (mode == 1) ? 2.0 : 1.0;   // backward: y_k = (-1)^k c_k, ends doubled
#pragma unroll
  for (int pi = 0; pi < NP; pi++) {
    const int j0 = q + pi * TPL;
    const int j = j0 <= M / 2 ? j0 : M / 2, jm = M - j;
    const cplx pj = w2[Lay<LN>::pix(j)], pjl = w2[Lay<LN>::pix(j > 0 ? j - 1 : 0)], pm = w2[Lay<LN>::pix(jm)], pml = w2[Lay<LN>::pix(jm - 1)];
    const double xo_p = sg * pj.y;                              // x_{2j+1}
    const double xo_m = (j == 0) ? xo_p : sg * pjl.y;           // x_{2j-1}, x_{-1} = x_1
    const double xm_m = sg * pml.y;                             // x_{2jm-1}
    const double xm_p = (jm == M) ? xm_m : sg * pm.y;           // x_{2jm+1}, x_{N+1} = x_{N-1}
    const cplx zj = make_double2(pj.x * (j == 0 ? endf : 1.0), xo_p - xo_m);
    const cplx zmc = make_double2(pm.x * (jm == M ? endf : 1.0), -(xm_p - xm_m));   // conj(z_{M-j})
    const cplx e = cadd(zj, zmc), d = cmul(csub(zj, zmc), ldg(tw2 + j));
    gj[pi] = make_double2(e.x - d.y, e.y + d.x);           // e + i d
    gm[pi] = make_double2(e.x + d.y, -e.y + d.x);          // conj(e) + i conj(d)
    r0 += (j0 < M / 2) ? (xo_p + xm_m) : 0.0;
  }
  r0 = 2.0 * lane_sum<LN>(r0, TPL, scratch);   // R_0 = 2 * sum of odd samples
  __syncthreads();
#pragma unroll
  for (int pi = 0; pi < NP; pi++) {
    const int j = q + pi * TPL;
    if (j <= M / 2) w2[Lay<LN>::pix(j)] = gj[pi];
    if (j > 0 && j < M / 2) w2[Lay<LN>::pix(M - j)] = gm[pi];
  }
  __syncthreads();
  lane_fft<E, LN>(W, M, TPL, tw);
  // ---- post: Z (N reals) -> X (N+1), pairs (k, N-k), 1 <= k <= M-1 in a branch-free unrolled loop ----
  const double fs = (mode == 0) ? 1.0 / N : 0.5;
#pragma unroll
  for (int pi = 0; pi < E + 1; pi++) {
    const int k0 = q + pi * TPL;
    const bool ok = k0 >= 1 && k0 <= M - 1;
    const int k = ok ? k0 : 1;
    const double zk = w[Lay<LN>::eix(k)], zn = w[Lay<LN>::eix(N - k)];
    const double A = 0.5 * (zk + zn), R = (zn - zk) * ldg(isin + k);
    const double sk = (mode == 0 && (k & 1)) ? -fs : fs;      // N is even: k and N-k have the same parity
    if (ok) { w[Lay<LN>::eix(k)] = (A + R) * sk; w[Lay<LN>::eix(N - k)] = (A - R) * sk; }
  }
  if (q == 0) {   // k = 0 (and N), k = M: untouched by the loop above
    const double z0 = w[0], e0 = (mode == 0) ? 0.5 * fs : fs;
    w[0] = (z0 + r0) * e0;
    w[Lay<LN>::eix(N)] = (z0 - r0) * e0;
    w[Lay<LN>::eix(M)] = w[Lay<LN>::eix(M)] * ((mode == 0 && (M & 1)) ? -fs : fs);
  }
  __syncthreads();
}

// Real FFT of n points along the lane (Fourier axis, SURVEY A.4): forward r2c is unnormalised,
// n/2+1 interleaved complex modes; backward c2r carries 1/n and ignores Im of the k=0 and k=n/2 modes.
template <int E, int LN>
__device__ __noinline__ void op_rfft(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  const int TPL = P.TPL, LP = P.LP;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int n = op.i0, M = n >> 1, mode = op.i1;
  const cplx* tw = (const cplx*)op.p0; const cplx* tw2 = (const cplx*)op.p1;
  double* w = W + 4 * l;
  cplx* w2 = reinterpret_cast<cplx*>(W) + 2 * l;
  if (mode == 0) {
    lane_fft<E, LN>(W, M, TPL, tw);
    for (int k = q; k <= M / 2; k += TPL) {
      if (k == 0) {
        cplx z = w2[0];
        w2[0] = make_double2(z.x + z.y, 0.0);
        w2[Lay<LN>::pix(M)] = make_double2(z.x - z.y, 0.0);
      } else {
        cplx zk = w2[Lay<LN>::pix(k)], zm = cconj(w2[Lay<LN>::pix(M - k)]);
        cplx S = cadd(zk, zm), D = cmul(ldg(tw2 + k), csub(zk, zm));   // w_k D
        // X_k = (S - i wD)/2 ; X_{M-k} = conj((S + i wD)/2)
        w2[Lay<LN>::pix(k)] = make_double2(0.5 * (S.x + D.y), 0.5 * (S.y - D.x));
        if (k != M - k) w2[Lay<LN>::pix(M - k)] = make_double2(0.5 * (S.x - D.y), -0.5 * (S.y + D.x));
      }
    }
    __syncthreads();
  } else {
    for (int k = q; k <= M / 2; k += TPL) {
      if (k == 0) {
        double x0 = w[0], xm = w[Lay<LN>::eix(2 * M)];
        // Zc_0 = ((x0+xm) + i(x0-xm))/2 ; FFT input is conj(Zc)
        w2[0] = make_double2(0.5 * (x0 + xm), -0.5 * (x0 - xm));
      } else {
        cplx xk = w2[Lay<LN>::pix(k)], xm = cconj(w2[Lay<LN>::pix(M - k)]);
        cplx S = cadd(xk, xm), D = cmul(cconj(ldg(tw2 + k)), csub(xk, xm));  // conj(w_k) D'
        // Zc_k = (S + i cD)/2 ; Zc_{M-k} = conj((S - i cD)/2); store conjugates
        w2[Lay<LN>::pix(k)] = make_double2(0.5 * (S.x - D.y), -0.5 * (S.y + D.x));
        if (k != M - k) w2[Lay<LN>::pix(M - k)] = make_double2(0.5 * (S.x + D.y), 0.5 * (S.y - D.x));
      }
    }
    __syncthreads();
    lane_fft<E, LN>(W, M, TPL, tw);
    const double s = 1.0 / M;
    for (int e = q; e < LP; e += TPL) {
      double v = w[Lay<LN>::eix(e)];
      w[Lay<LN>::eix(e)] = (e < n) ? ((e & 1) ? -v * s : v * s) : 0.0;
    }
    __syncthreads();
  }
}

// ChebDirichletNeumann stencil (bc = "hc"): the three-term stencil couples neighbouring elements, so the pair structure of
// the other banded operators does not apply; element-strided, register-staged (not on any BASELINE configuration's path).
template <int CP, int LN>
__device__ __noinline__ void op_sten3(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  const int TPL = P.TPL, LP = P.LP;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const double* __restrict__ ca = (const double*)op.p0; const double* __restrict__ cb = (const double*)op.p1;
  const int len_out = op.i0, mode = op.i1;
  double* w = W + 4 * l;
  double y[2 * CP];
#pragma unroll
  for (int i = 0; i < 2 * CP; i++) {
    const int e = q + i * TPL;
    double v = 0.0;
    if (e < LP && e < len_out) {
      v = w[Lay<LN>::eix(e)];
      if (mode == 0) {
        if (e >= 1) v = fma(ldg(ca + e - 1), w[Lay<LN>::eix(e - 1)], v);
        if (e >= 2) v = fma(ldg(cb + e - 2), w[Lay<LN>::eix(e - 2)], v);
      } else {
        if (e + 1 < LP) v = fma(ldg(ca + e), w[Lay<LN>::eix(e + 1)], v);
        if (e + 2 < LP) v = fma(ldg(cb + e), w[Lay<LN>::eix(e + 2)], v);
      }
    }
    y[i] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 2 * CP; i++) {
    const int e = q + i * TPL;
    if (e < LP) w[Lay<LN>::eix(e)] = y[i];
  }
  __syncthreads();
}

// Transform of a lane as a dense mat-vec (DCT-I / r2c / c2r matrices built on the host): the fallback for transform sizes that are
// not 2^k (+1) -- e.g. the reference's criterion sizes 128, 264, 265, 512 (benches/benchmark_navier.rs:6-7).  Thread q of a lane
// accumulates the outputs k = q + i TPL in registers while every thread of the lane walks the same input element.
template <int CP, int LN>
__device__ __noinline__ void op_dense(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  const int TPL = P.TPL, LP = P.LP;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  const int n_out = op.i0, n_in = op.i1;
  const double* __restrict__ M = (const double*)op.p0;
  double* w = W + 4 * l;
  double y[2 * CP];
#pragma unroll
  for (int i = 0; i < 2 * CP; i++) y[i] = 0.0;
  for (int j = 0; j < n_in; j++) {
    const double x = w[Lay<LN>::eix(j)];
#pragma unroll
    for (int i = 0; i < 2 * CP; i++) {
      const int k = q + i * TPL;
      if (k < n_out) y[i] = fma(ldg(M + (size_t)k * n_in + j), x, y[i]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 2 * CP; i++) {
    const int k = q + i * TPL;
    if (k < LP) w[Lay<LN>::eix(k)] = (k < n_out) ? y[i] : 0.0;
  }
  __syncthreads();
}

// PdmaPlus2::solve_lane (src/solver/pdma_plus2.rs:123-157): forward elimination (second order) and back substitution
// (fourth order) over the elements of a lane; one thread per lane ("one thread per system") -- bc = "hc" only.
template <int LN>
__device__ __noinline__ void op_pdma(const LaneProg& P, const LaneOp& op, double* __restrict__ W) {
  const int n = op.i0, L = op.i1;
  if ((int)threadIdx.x < LN) {
    double* w = W + 4 * threadIdx.x;
    const double* __restrict__ l2 = (const double*)op.p0; const double* __restrict__ ka = l2 + L; const double* __restrict__ imu = ka + L;
    const double* __restrict__ al = imu + L; const double* __restrict__ be = al + L; const double* __restrict__ ga = be + L; const double* __restrict__ de = ga + L;
    double z1 = 0.0, z2 = 0.0;
#pragma unroll 4
    for (int i = 0; i < n; i++) {
      double t = fma(-z2, ldg(l2 + i), w[Lay<LN>::eix(i)]);
      t = fma(-z1, ldg(ka + i), t);
      const double z = t * ldg(imu + i);
      w[Lay<LN>::eix(i)] = z;
      z2 = z1; z1 = z;
    }
    double x1 = 0.0, x2 = 0.0, x3 = 0.0, x4 = 0.0;
#pragma unroll 4
    for (int i = n - 1; i >= 0; i--) {
      double t = fma(-x4, ldg(de + i), w[Lay<LN>::eix(i)]);
      t = fma(-x3, ldg(ga + i), t);
      t = fma(-x2, ldg(be + i), t);
      const double x = fma(-x1, ldg(al + i), t);
      w[Lay<LN>::eix(i)] = x;
      x4 = x3; x3 = x2; x2 = x1; x1 = x;
    }
    for (int i = n; i < P.LP; i++) w[Lay<LN>::eix(i)] = 0.0;
  }
  __syncthreads();
}

template <int LN>
__device__ __forceinline__ void op_pointwise(const LaneProg& P, const LaneOp& op, double* __restrict__ W, int g, int lb) {
  const int TPL = P.TPL, LP = P.LP;
  const int l = threadIdx.x & (LN - 1), q = threadIdx.x >> Lay<LN>::LOG;
  double* w = W + 4 * l;
  cplx* w2 = reinterpret_cast<cplx*>(W) + 2 * l;
  switch (op.code) {
    case OP_FDIFF: {   // interleaved complex: (re, im) *= (i k)^d * a
      const int m = op.i0, d = op.i1 & 3, wrap = op.i2;   // wrap = n (FourierC2c): modes in FFT order, index k >= n/2 is wavenumber k - n
      for (int k = q; k < m; k += TPL) {
        cplx c = w2[Lay<LN>::pix(k)];
        double f = op.a;
        const double kk = (double)((wrap && 2 * k >= wrap) ? k - wrap : k);
        for (int t = 0; t < op.i1; t++) f *= kk;
        cplx r;
        if (d == 0) r = make_double2(c.x * f, c.y * f);
        else if (d == 1) r = make_double2(-c.y * f, c.x * f);
        else if (d == 2) r = make_double2(-c.x * f, -c.y * f);
        else r = make_double2(c.y * f, -c.x * f);
        w2[Lay<LN>::pix(k)] = r;
      }
    } break;
    case OP_SCALEVEC: {
      const double* v = (const double*)op.p0;
      for (int e = q; e < op.i0; e += TPL) w[Lay<LN>::eix(e)] *= ldg(v + (e >> op.i1));
    } break;
    case OP_ZEROTAIL:
      for (int e = op.i0 + q; e < LP; e += TPL) w[Lay<LN>::eix(e)] = 0.0;
      break;
    case OP_LANEMASK:
      if (4 * g + lb + l >= op.i0) for (int e = q; e < LP; e += TPL) w[Lay<LN>::eix(e)] = 0.0;
      break;
    case OP_ZEROELEM:
      if (4 * g + lb + l == op.i0 && q == 0) w[Lay<LN>::eix(op.i1)] = 0.0;
      break;
    case OP_SCALE:
      for (int e = q; e < LP; e += TPL) w[Lay<LN>::eix(e)] *= op.a;
      break;
  }
  __syncthreads();
}

#include "lane_fast.cuh"

// E = FFT points per thread (16: radix-16 passes, 128 registers; 8 and 4 for short lanes); LN = lanes per CTA;
// TPLC = threads per lane as a compile-time constant for transform-sized lanes (N = 2*E*TPLC: the hot operators
// then run their compile-time-geometry versions of lane_fast.cuh), 0 = generic geometry read from the program.
template <int E, int LN, int TPLC>
#ifndef B2_LB
#define B2_LB __launch_bounds__(512)
#endif
__global__ void B2_LB lane_kernel(const __grid_constant__ LaneProg Pp) {
  B2_DYN_SMEM(char, smem_raw);
  // The ops run as separate (non-inlined) functions that get the program by reference; a reference into
  // parameter space degrades to generic loads with global-memory latency, so the header and the op list are
  // copied into shared memory once and everything but the tensor maps is read from there.
  static_assert(offsetof(LaneProg, tm) <= B2_PROGCOPY, "program copy area too small");
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&Pp);
    uint32_t* dst = reinterpret_cast<uint32_t*>(smem_raw + B2_BARBYTES);
    for (int i = threadIdx.x; i < (int)(offsetof(LaneProg, tm) / 4); i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const LaneProg& P = *reinterpret_cast<const LaneProg*>(smem_raw + B2_BARBYTES);
  const SmemView sv = smem_view(P, smem_raw);
  double* W = sv.W;
  void* scratch = sv.scratch;
  const int gl = blockIdx.x / (4 / LN);   // local lane group (addresses this GPU's slab)
  const int g = P.group0 + gl;            // global lane group (mode indices, transposed stores)
  const int lb = (blockIdx.x & ((4 / LN) - 1)) * LN;
  Prefetch pf; pf.gl = gl; pf.lb = lb; pf.dphase = 0; pf.wph = 0; pf.ws = 0;
  if (threadIdx.x == 0) {
    mbar_init(sv.dfull, 1);
    for (int i = 0; i < 2 * (P.NT >> 5); i++) mbar_init(&sv.wbar[i], 1);
    mbar_fence_init();
    for (int o = 0; o < P.nops; o++)
      if ((P.ops[o].code == OP_LOAD && (P.ops[o].i2 & (LD_TMA | LD_DIRECT))) || (P.ops[o].code == OP_STORE && (P.ops[o].i2 & (ST_TMA | ST_DIRECT)) && !(P.ops[o].i2 & ST_PEER)))
        tmap_prefetch(&Pp.tm[o]);
  }
  __syncthreads();
  for (int o = 0; o < P.nops; o++) {
    const LaneOp& op = P.ops[o];
    long long t0 = 0;
    if (P.prof) t0 = clock64();
    switch (op.code) {
      case OP_LOAD: {
        PhaseClock pc(P.prof);
        if (op.i2 & LD_DIRECT) load_direct<LN>(P, op, &Pp.tm[o], sv, pf);
        else if (op.i2 & LD_TMA) load_warps<LN>(P, op, &Pp.tm[o], sv, pf);
        else load_threads<LN, (E == 16 ? 8 : 4)>(P, op, sv, gl, lb);
        pc.mark((op.i2 & LD_DIRECT) ? (o == 0 ? 27 : 28) : ((op.i2 & LD_PLAIN) ? 30 : ((op.i2 & LD_STENCIL) ? 31 : 29)));
      }
        break;
      case OP_STORE:
        if (op.i2 & ST_DIRECT) store_direct<LN>(P, op, &Pp.tm[o], sv, g, gl, lb);
        else if (op.i2 & ST_TMA) store_warps<LN>(P, op, (op.i2 & ST_PEER) ? &Pp.tmp[op.i1][0] : &Pp.tm[o], sv, g, gl, lb, pf);
        else store_threads<LN>(P, op, sv, g, gl, lb);
        break;
      case OP_BAND:
        if constexpr (TPLC > 0) band_fast<E, LN, TPLC>(P, op, W); else op_band<E + 1, LN>(P, op, W);
        break;
      case OP_DERIV:
        if constexpr (TPLC > 0) deriv_fast<E, LN, TPLC>(P, op, W, scratch); else op_deriv<E + 1, LN>(P, op, W, scratch);
        break;
      case OP_FDMA:
        if constexpr (TPLC > 0) fdma_fast<E, LN, TPLC>(P, op, W, gl, lb, scratch); else op_fdma<E + 1, LN>(P, op, W, gl, lb, scratch);
        break;
      case OP_DCT:
        if constexpr (TPLC > 0) dct_fast<E, LN, TPLC>(op, W, (double*)scratch, P.prof); else op_dct<E, LN>(P, op, W, (double*)scratch);
        break;
      case OP_RFFT:
        if constexpr (TPLC > 0) rfft_fast<E, LN, TPLC>(P, op, W); else op_rfft<E, LN>(P, op, W);
        break;
      case OP_PREBAND: break;
      case OP_BANDC:
        if constexpr (TPLC > 0) band_chunk<E, LN, TPLC>(P, op, W);
        break;
      case OP_DENSE: op_dense<E + 1, LN>(P, op, W); break;
      case OP_STEN3: op_sten3<E + 1, LN>(P, op, W); break;
      case OP_PDMA: op_pdma<LN>(P, op, W); break;
      default: op_pointwise<LN>(P, op, W, g, lb); break;
    }
    if (P.prof && threadIdx.x == 0) {
      atomicAdd(P.prof + op.code, (unsigned long long)(clock64() - t0));
      atomicAdd(P.prof + 32 + op.code, 1ull);
    }
  }
  if ((threadIdx.x & 31) == 0) bulk_wait<0>();   // shared memory must outlive the bulk stores that read it (every issuing lane waits for its own)
}
