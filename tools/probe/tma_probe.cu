// Memory-pipeline microbenchmark for the lane kernel's slab loads / stores (measurement tool, not product code).
// One "slab" = SLAB bytes contiguous in HBM (a 4-lane group of a 4097-point array = 131 KB).  Each CTA walks slabs
// g = blockIdx.x, blockIdx.x + gridDim.x, ... of a large array and moves every slab HBM -> shared memory (mode L),
// shared memory -> HBM (mode S) or both, overlapped through two buffers (mode C), with a chosen piece size, number of
// issuing threads and CTAs per SM.  Prints GB/s and cycles per slab.
//   build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe/tma_probe tools/probe/tma_probe.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../rustpde_mpi_b200/csrc/async_ops.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

struct Args { const char* src; char* dst; int slab, piece, nslabs, issuers, mode, ldg_u; unsigned long long* cyc; };

// mode 0: bulk loads; 1: bulk stores; 2: load + store overlapped (two buffers); 3: per-thread LDG.128 loads (ldg_u in flight);
// 4: per-thread STG.128 stores
__global__ void __launch_bounds__(512) probe(const __grid_constant__ Args a) {
  extern __shared__ __align__(1024) char sm[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm);   // bar[0], bar[1]
  char* buf0 = sm + 1024;
  char* buf1 = buf0 + a.slab;
  const int tid = threadIdx.x, nt = blockDim.x;
  if (tid == 0) { mbar_init(&bar[0], a.issuers); mbar_init(&bar[1], a.issuers); mbar_fence_init(); }
  __syncthreads();
  const int npieces = a.slab / a.piece;
  // issuer i (thread 32*i) takes pieces i, i + issuers, ...
  const bool issuer = (tid % 32 == 0) && (tid / 32 < a.issuers);
  const int iid = tid / 32;
  unsigned ph0 = 0, ph1 = 0;
  long long t0 = clock64();
  int cnt = 0;
  auto issue_load = [&](char* buf, uint64_t* b, int g) {
    if (!issuer) return;
    int mine = 0;
    for (int p = iid; p < npieces; p += a.issuers) mine++;
    mbar_arrive_expect_tx(b, (uint32_t)mine * a.piece);
    for (int p = iid; p < npieces; p += a.issuers)
      bulk_load_1d(buf + (size_t)p * a.piece, a.src + (size_t)g * a.slab + (size_t)p * a.piece, (uint32_t)a.piece, b);
  };
  auto issue_store = [&](const char* buf, int g) {
    if (!issuer) return;
    for (int p = iid; p < npieces; p += a.issuers)
      bulk_store_1d(a.dst + (size_t)g * a.slab + (size_t)p * a.piece, buf + (size_t)p * a.piece, (uint32_t)a.piece);
    bulk_commit();
  };
  if (a.mode == 0) {
    for (int g = blockIdx.x; g < a.nslabs; g += gridDim.x, cnt++) {
      issue_load(buf0, &bar[0], g);
      mbar_wait(&bar[0], ph0); ph0 ^= 1;
      __syncthreads();
    }
  } else if (a.mode == 1) {
    for (int i = tid; i < a.slab / 16; i += nt) reinterpret_cast<double2*>(buf0)[i] = make_double2(i, tid);
    fence_proxy_async();
    __syncthreads();
    for (int g = blockIdx.x; g < a.nslabs; g += gridDim.x, cnt++) {
      issue_store(buf0, g);
      if (issuer) bulk_wait_read<0>();
      __syncthreads();
    }
    if (issuer) bulk_wait<0>();
  } else if (a.mode == 2) {
    // load slab k+1 into the other buffer while slab k is being stored
    int g = blockIdx.x;
    if (g < a.nslabs) issue_load(buf0, &bar[0], g);
    int cur = 0;
    for (; g < a.nslabs; g += gridDim.x, cnt++, cur ^= 1) {
      char* b = cur ? buf1 : buf0;
      char* nb = cur ? buf0 : buf1;
      if (issuer) bulk_wait_read<0>();   // the store that read `nb` two rounds ago is done with it
      __syncthreads();
      if (g + (int)gridDim.x < a.nslabs) issue_load(nb, &bar[cur ^ 1], g + gridDim.x);
      if (cur) { mbar_wait(&bar[1], ph1); ph1 ^= 1; } else { mbar_wait(&bar[0], ph0); ph0 ^= 1; }
      fence_proxy_async();
      __syncthreads();
      issue_store(b, g);
    }
    if (issuer) bulk_wait<0>();
  } else if (a.mode == 3) {
    const int U = a.ldg_u;
    for (int g = blockIdx.x; g < a.nslabs; g += gridDim.x, cnt++) {
      const double2* s = reinterpret_cast<const double2*>(a.src + (size_t)g * a.slab);
      double2* d = reinterpret_cast<double2*>(buf0);
      const int n = a.slab / 16;
      for (int i0 = tid; i0 < n; i0 += U * nt) {
        double2 v[16];
#pragma unroll
        for (int k = 0; k < 16; k++) if (k < U && i0 + k * nt < n) v[k] = s[i0 + k * nt];
#pragma unroll
        for (int k = 0; k < 16; k++) if (k < U && i0 + k * nt < n) d[i0 + k * nt] = v[k];
      }
      __syncthreads();
    }
  } else if (a.mode == 4) {
    for (int i = tid; i < a.slab / 16; i += nt) reinterpret_cast<double2*>(buf0)[i] = make_double2(i, tid);
    __syncthreads();
    for (int g = blockIdx.x; g < a.nslabs; g += gridDim.x, cnt++) {
      double2* d = reinterpret_cast<double2*>(a.dst + (size_t)g * a.slab);
      const double2* s = reinterpret_cast<const double2*>(buf0);
      const int n = a.slab / 16;
      for (int i = tid; i < n; i += nt) d[i] = s[i];
      __syncthreads();
    }
  }
  if (tid == 0 && cnt) { atomicAdd(a.cyc, (unsigned long long)(clock64() - t0)); atomicAdd(a.cyc + 1, (unsigned long long)cnt); }
}

int main(int argc, char** argv) {
  const int slab = 131072;
  const size_t total = (size_t)4 << 30;   // 4 GiB arrays: every slab comes from HBM
  char *src, *dst; unsigned long long* cyc;
  CK(cudaMalloc(&src, total)); CK(cudaMalloc(&dst, total)); CK(cudaMalloc(&cyc, 16));
  CK(cudaMemset(src, 1, total)); CK(cudaMemset(dst, 0, total));
  CK(cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const char* names[] = {"bulk load", "bulk store", "load+store overlapped", "LDG.128 load", "STG.128 store"};
  auto run = [&](int mode, int piece, int issuers, int ctas_per_sm, int slab_b, int u, int nslabs_total, bool l2) {
    Args a; a.src = src; a.dst = dst; a.slab = slab_b; a.piece = piece; a.issuers = issuers; a.mode = mode; a.ldg_u = u; a.cyc = cyc;
    a.nslabs = l2 ? (int)(((size_t)48 << 20) / slab_b) : nslabs_total;   // l2: a 48 MB working set that stays in L2
    const int reps = l2 ? 12 : 1;
    const size_t smem = 1024 + (size_t)slab_b * (mode == 2 ? 2 : 1);
    const int grid = 132 * ctas_per_sm;
    if (smem * ctas_per_sm > 226 * 1024) return;
    CK(cudaMemset(cyc, 0, 16));
    probe<<<grid, 512, smem>>>(a);   // warm-up
    CK(cudaMemset(cyc, 0, 16));
    CK(cudaEventRecord(e0));
    for (int r = 0; r < reps; r++) probe<<<grid, 512, smem>>>(a);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaGetLastError());
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    unsigned long long h[2]; CK(cudaMemcpy(h, cyc, 16, cudaMemcpyDeviceToHost));
    const double bytes = (double)a.nslabs * slab_b * reps * (mode == 2 ? 2 : 1);
    printf("%-22s slab %6d piece %6d issuers %2d ctas/sm %d %s: %8.1f GB/s  %8.0f cycles/slab/CTA  (%.1f B/clk/SM)\n", names[mode], slab_b, piece, issuers,
           ctas_per_sm, l2 ? "L2 " : "HBM", bytes / ms / 1e6, (double)h[0] / h[1], (double)slab_b * (mode == 2 ? 2 : 1) * ctas_per_sm / ((double)h[0] / h[1]));
  };
  const int N = 16384;   // 2 GiB of 128 KB slabs
  for (int l2 = 0; l2 < 2; l2++) {
    for (int piece : {32768, 8192, 2048}) for (int iss : {1, 4, 16}) run(0, piece, iss, 1, slab, 0, N, l2);
    run(0, 16384, 1, 2, 65536, 0, 2 * N, l2); run(0, 16384, 4, 2, 65536, 0, 2 * N, l2); run(0, 8192, 4, 3, 65536, 0, 2 * N, l2); run(0, 8192, 4, 6, 32768, 0, 4 * N, l2);
    for (int u : {4, 8, 16}) run(3, 0, 1, 1, slab, u, N, l2);
    run(3, 0, 1, 2, 65536, 8, 2 * N, l2);
  }
  for (int piece : {32768, 8192, 2048}) for (int iss : {1, 4, 16}) run(1, piece, iss, 1, slab, 0, N, false);
  run(1, 16384, 4, 2, 65536, 0, 2 * N, false); run(1, 8192, 4, 3, 65536, 0, 2 * N, false);
  run(4, 0, 1, 1, slab, 0, N, false);
  run(2, 32768, 1, 1, 65536, 0, 2 * N, false); run(2, 8192, 4, 1, 65536, 0, 2 * N, false); run(2, 8192, 4, 2, 32768, 0, 4 * N, false); run(2, 8192, 4, 1, 98304, 0, N, false);
  return 0;
}
