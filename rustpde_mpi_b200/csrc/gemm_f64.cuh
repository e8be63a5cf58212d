// FP64 GEMM of the Poisson eigen-transform (reference: src/solver/poisson.rs:213-219 and :231-235, the two
// `fwd.dot(..)` / `bwd.dot(..)` products) computed directly on the 4x4-tiled arrays of the lane passes.
//
//   C[rowC(b, m)][j] = sum_k A_b[m][k] * B[rowB(b, k)][j]          b = parity block (0 even, 1 odd)
//
// The eigenvectors of the Chebyshev Poisson operator only couple x-indices of equal parity, so each product is two
// half-size GEMMs that read / write the even and the odd rows of the same tiled array.  One CTA computes a 64-row
// slice of BOTH blocks for a block of <= 128 columns, so every tile of B is fetched once for the two blocks:
//   rowX(b, t) = offX[b] + t * strX      interleaved (natural x order: off = {0, 1}, str = 2)  or
//                                        grouped     (eigenmode order: off = {0, ce}, str = 1)
// B and C are tiled arrays (tile (I, J) at ((I * TJ) + J) * 128 bytes, element [i][j] inside): a tile row segment
// is contiguous, so a k-stage of B (32 natural rows = 8 tile rows x <= 32 tiles) is eight 1-D bulk copies
// (cp.async.bulk) -- no tensor map, no layout pass.  Arithmetic: mma.sync.m16n8k8.f64 (SASS DMMA.16x8x8; on sm_90 the
// m16n8k{4,8,16} shapes run at twice the FMA rate of m8n8k4, tools/probe/dmma_probe.cu; tcgen05 / wgmma have no FP64
// path).  Its B operand takes k in slices of 4 per register, so a 4x4 tile IS one B register of 8 columns: thread
// (t = lane % 4, g = lane / 4) reads element [row(t)][g % 4] of tile g / 4 of a k4 slice, conflict-free with a 32-byte
// skew between tile-row slots.  A_b is packed on the host in fragment order ([m slice][k stage][16-row fragment][k4
// slice][lane][2]), so a thread's four A registers of a k8 step are two conflict-free 16-byte loads; one 8 KB bulk copy
// per block and stage.  8 compute warps x (32 x 64) outputs, accumulators in registers (168 registers, no spills: with
// 16 warps of 32 x 32 the 17 warps cap a thread at 96 registers and the fragments spilled), a 4-stage full/empty
// mbarrier pipeline without CTA barriers, fed by a ninth warp that only issues the bulk copies.
#pragma once
#include "async_ops.cuh"

#define G_NSTAGE 4
#define G_THREADS 288                                    // 8 compute warps + one copy warp
#define G_KK 4                                           // k4 slices per stage: a stage holds 16 k per block
#define G_SLOT_PITCH (32 * 16 + 4)                       // doubles per tile-row slot of B: 32 tiles + 32 bytes of skew
#define G_ACHUNK (64 * 4 * G_KK)                         // packed A per block and stage: 64 rows x 16 k
#define G_STAGE_DOUBLES (2 * G_KK * G_SLOT_PITCH + 2 * G_ACHUNK)   // 8 B slots + the two A chunks
#define G_SMEM_BYTES (128 + G_NSTAGE * G_STAGE_DOUBLES * 8)

struct GemmParams {
  const double* A[2];       // packed operands of the two blocks (see pack_gemm_a)
  const double* B;          // tiled source, TJb tiles per row, rowsB tile rows
  double* C;                // tiled destination (this rank's copy; peers at the same heap offset)
  double* const* peers;     // null on one GPU; else device table of the ranks' heap bases
  long long c_off;          // byte offset of C inside the heap (peers)
  int TJb, TJc;             // tiles per row of B and of C
  int rowsB;                // tile rows of B (rows beyond are never read: the stage row is clamped, A is zero there)
  int jc0;                  // tile column of C that column 0 of B maps to (rank * TJb with several GPUs)
  int nmt, ncb;             // 64-row slices per block, column blocks; grid = nmt * ncb
  int nks;                  // k stages of 16 per block
  int Mb[2];                // valid rows per block
  int mstep, bshift;        // global row of (block b, slice mt, local row r) = mt * mstep + b * bshift + r
  int offB[2], strB;        // natural B row of (b, k) = offB[b] + k * strB   (strB = 2: offB = {0, 1})
  int offC[2], strC;        // natural C row of (b, m)
  int rows_per_rank;        // C rows owned by one rank (multiple of 4); >= all rows on one GPU
  int gate;                 // a warp starts stage ks only when every warp has finished stage ks - gate (1 .. G_NSTAGE - 1)
};

// C(16 x 8) += A(16 x 8) B(8 x 8); g = lane / 4, t = lane % 4 (PTX ISA fragment tables for .f64):
//   a[i] = A[g + 8 (i % 2)][t + 4 (i / 2)],  b[i] = B[t + 4 i][g],  c[i] = C[g + 8 (i / 2)][2 t + i % 2]
__device__ __forceinline__ void dmma1688(double* c, const double* a, const double* b) {
#ifdef B2_EMU
  // the emulator's m8n8k4 (a = A[g][t], b = B[t][g], c = C[g][2 t + {0, 1}]): a[h + 2 q] is that fragment of the rows 8 h.. and
  // the k columns 4 q.. of A, b[q] of the k rows 4 q.. of B, c[2 h], c[2 h + 1] of the rows 8 h.. of C; k accumulates in order
  for (int h = 0; h < 2; h++)
    for (int q = 0; q < 2; q++) emu::dmma884(c[2 * h], c[2 * h + 1], a[h + 2 * q], b[q]);
#else
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
#endif
}

// DBG (measurement only, results invalid): 1 = no copies and no waits (arithmetic + shared-memory reads alone), 2 = copies and waits
// without the DMMAs (data movement alone).
template <int DBG>
__global__ void __launch_bounds__(G_THREADS, 1) gemm_pb_kernel(const __grid_constant__ GemmParams P) {
  B2_DYN_SMEM(char, gsm);
  uint64_t* full = reinterpret_cast<uint64_t*>(gsm);       // stage s has landed (bulk copies, transaction count)
  uint64_t* empty = full + G_NSTAGE;                       // all 8 compute warps have finished reading stage s
  double* stage0 = reinterpret_cast<double*>(gsm + 128);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = warp >> 2, wm = (warp >> 1) & 1, wn = warp & 1;
  const int mt = blockIdx.x % P.nmt, cb = blockIdx.x / P.nmt;
  // column blocks of 32 tiles, the remainder last: the (cheap) narrow blocks fill the tail of the last wave
  const int tc0 = cb * 32, ntc = min(32, P.TJb - tc0);
  const int nks = P.nks;
  const bool inter = (P.strB == 2);
  if (tid == 0) {
    for (int s = 0; s < G_NSTAGE; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }
    mbar_fence_init();
  }
  __syncthreads();
  auto issue = [&](int ks) {   // copy warp: stage ks -> buffer ks % G_NSTAGE
    const int s = ks % G_NSTAGE;
    double* st = stage0 + (size_t)s * G_STAGE_DOUBLES;
    const uint32_t rowbytes = (uint32_t)ntc * 128u;
    mbar_arrive_expect_tx(&full[s], 2u * G_KK * rowbytes + 2u * G_ACHUNK * 8u);
    for (int sl = 0; sl < 2 * G_KK; sl++) {
      int trow = inter ? 2 * G_KK * ks + sl : (P.offB[sl & 1] >> 2) + G_KK * ks + (sl >> 1);
      trow = min(trow, P.rowsB - 1);   // beyond the array: any finite data (the packed A is zero there)
      bulk_load_1d(st + sl * G_SLOT_PITCH, P.B + ((size_t)trow * P.TJb + tc0) * 16, rowbytes, &full[s]);
    }
    for (int bb = 0; bb < 2; bb++)
      bulk_load_1d(st + 2 * G_KK * G_SLOT_PITCH + bb * G_ACHUNK, P.A[bb] + ((size_t)mt * nks + ks) * G_ACHUNK, G_ACHUNK * 8u, &full[s]);
  };
  // Warp 8 only moves data: it refills a buffer as soon as all 8 compute warps have released it.  (With the copies issued by
  // a compute thread, that thread's warp fell behind by the issue work of every stage, and -- the skew between the warps being
  // bounded -- all the others waited for it.)
  if (warp == 8) {
    if (lane == 0 && DBG != 1)
      for (int ks = 0; ks < nks; ks++) {
        if (ks >= G_NSTAGE) mbar_wait(&empty[ks % G_NSTAGE], (unsigned)(((ks / G_NSTAGE) - 1) & 1));
        issue(ks);
      }
    return;
  }

  // fragment addresses inside a stage (doubles)
  const int t = lane & 3, g = lane >> 2;
  // k4 slice kk of block b sits in slots 2 kk and 2 kk + 1: both tile rows of its 8 natural rows (interleaved) or slot
  // 2 kk + b (grouped: the copy warp places block b's tile rows there), so every B read is boff + an immediate
  const int slot0 = inter ? (t >> 1) : b, row = inter ? 2 * (t & 1) + b : t;
  const int boff = slot0 * G_SLOT_PITCH + (16 * wn + (g >> 2)) * 16 + row * 4 + (g & 3);
  const int aoff = 2 * G_KK * G_SLOT_PITCH + b * G_ACHUNK + (2 * wm) * 256 + 2 * lane;
  // rows / columns this warp owns; fragments completely outside the valid range are skipped (warp-uniform)
  const int mrow0 = mt * P.mstep + b * P.bshift + 32 * wm;          // global row of fragment 0, row 0
  const int Mv = P.Mb[b];
  const int ncols = 4 * ntc - 64 * wn;                              // valid columns from this warp's first one
  int mf_n = 0, nf_n = 0;
  for (int i = 0; i < 2; i++) if (mrow0 + 16 * i < Mv) mf_n = i + 1;
  for (int j = 0; j < 8; j++) if (8 * j < ncols) nf_n = j + 1;

  double acc[2][8][4];
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < 8; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[i][j][e] = 0.0;

  // No CTA barrier in the main loop, but a bounded skew: a warp starts stage ks only when every warp has finished stage
  // ks - 2.  (The warp scheduler prefers the highest warp id; without the bound the favoured warps run ahead until they
  // starve on data that is only requested once the slowest warp releases a buffer -- every round then pays the copy
  // latency.  With it, the refill of a buffer is always requested two stages before anybody needs it.)
  for (int ks = 0; ks < nks; ks++) {
    const int s = ks % G_NSTAGE;
    if (ks >= P.gate && DBG != 1) mbar_wait(&empty[(ks - P.gate) % G_NSTAGE], (unsigned)(((ks - P.gate) / G_NSTAGE) & 1));
    if (DBG != 1) mbar_wait(&full[s], (unsigned)((ks / G_NSTAGE) & 1));
    const double* st = stage0 + (size_t)s * G_STAGE_DOUBLES;
    if (mf_n > 0 && nf_n > 0 && DBG != 2) {
#pragma unroll
      for (int kh = 0; kh < 2; kh++) {
        double a[2][4];
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
          for (int q = 0; q < 2; q++) {
            const double2 v = *reinterpret_cast<const double2*>(st + aoff + i * 256 + (2 * kh + q) * 64);
            a[i][2 * q] = v.x; a[i][2 * q + 1] = v.y;
          }
#pragma unroll
        for (int j = 0; j < 8; j++) {
          if (j >= nf_n) break;
          double bf[2];
#pragma unroll
          for (int kk = 0; kk < 2; kk++) bf[kk] = st[boff + 2 * (2 * kh + kk) * G_SLOT_PITCH + j * 32];
          dmma1688(acc[0][j], a[0], bf);
          if (mf_n == 2) dmma1688(acc[1][j], a[1], bf);
        }
      }
    }
    __syncwarp();
    if (lane == 0 && DBG != 1) mbar_arrive(&empty[s]);
  }
  // epilogue: thread holds C[16 i + 8 h + g][8 j + 2 t + {0, 1}] of its 32 x 64 block in acc[i][j][2 h + {0, 1}]
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int mg = mrow0 + 16 * i + 8 * h + g;
      if (i >= mf_n || mg >= Mv) continue;
      const int r = P.offC[b] + mg * P.strC;             // natural destination row
      double* base = P.C;
      int rl = r;
      if (P.peers) {
        const int owner = r / P.rows_per_rank;
        rl = r - owner * P.rows_per_rank;
        base = reinterpret_cast<double*>(reinterpret_cast<char*>(P.peers[owner]) + P.c_off);
      }
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int cl = 64 * wn + 8 * j + 2 * t;          // column inside the column block
        if (j >= nf_n || cl >= 4 * ntc) continue;
        const int tc = P.jc0 + tc0 + (cl >> 2);
        double2* dst = reinterpret_cast<double2*>(base + ((size_t)(rl >> 2) * P.TJc + tc) * 16 + (rl & 3) * 4 + (cl & 3));
        *dst = make_double2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
      }
    }
}
