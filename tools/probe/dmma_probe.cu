// FP64 tensor-core (mma.sync .f64) throughput probe (measurement tool, not product code).
// For each shape m8n8k4, m16n8k4, m16n8k8, m16n8k16 it first checks the fragment layout the GEMM kernel assumes
// (one MMA on known matrices against a host product), then runs register-resident MMA loops -- NCH independent
// accumulator chains per warp, operands never reloaded -- on one CTA per SM with 1 and 4 warps per scheduler
// (4 and 16 warps per CTA), and prints FMA per clock per SM (clock64 inside each CTA) and TFLOP/s (CUDA events).
//   build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probe/dmma_probe tools/probe/dmma_probe.cu
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

// Fragment layouts of the PTX ISA for .f64 (g = lane / 4, t = lane % 4):
//   m8n8k4     a0 = A[g][t]                        b0 = B[t][g]               c{0,1} = C[g][2t + {0,1}]
//   m16n8kK    a_i = A[g + 8 (i % 2)][t + 4 (i / 2)]   b_i = B[t + 4 i][g]    c{0,1} = C[g][2t + {0,1}], c{2,3} = C[g + 8][..]
template <int M, int K> struct Shape { static constexpr int NA = M * K / 32, NB = K / 4, NC = M / 4; };

template <int M, int K> __device__ __forceinline__ void mma(double* c, const double* a, const double* b);
template <> __device__ __forceinline__ void mma<8, 4>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
}
template <> __device__ __forceinline__ void mma<16, 4>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
template <> __device__ __forceinline__ void mma<16, 8>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
template <> __device__ __forceinline__ void mma<16, 16>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// one MMA on A (M x K, row-major), B (K x 8, row-major) -> C (M x 8) through the layouts above
template <int M, int K> __global__ void layout_check(const double* A, const double* B, double* C) {
  using S = Shape<M, K>;
  const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
  double a[S::NA], b[S::NB], c[S::NC];
  for (int i = 0; i < S::NA; i++) a[i] = A[(g + 8 * (i % 2) * (M == 16)) * K + t + 4 * (M == 16 ? i / 2 : 0)];
  for (int i = 0; i < S::NB; i++) b[i] = B[(t + 4 * i) * 8 + g];
  for (int i = 0; i < S::NC; i++) c[i] = 0.0;
  mma<M, K>(c, a, b);
  for (int i = 0; i < S::NC; i++) C[(g + 8 * (i / 2)) * 8 + 2 * t + (i % 2)] = c[i];
}

#define NCH 8   // independent accumulator chains per warp
template <int M, int K> __global__ void __launch_bounds__(512, 1) rate(const double* src, double* out, int iters, unsigned long long* cyc) {
  using S = Shape<M, K>;
  double a[S::NA], b[S::NB], c[NCH][S::NC];
  for (int i = 0; i < S::NA; i++) a[i] = src[(threadIdx.x + i) & 255];
  for (int i = 0; i < S::NB; i++) b[i] = src[(threadIdx.x + 7 * i + 3) & 255];
  for (int h = 0; h < NCH; h++)
    for (int i = 0; i < S::NC; i++) c[h][i] = 0.0;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++)
#pragma unroll
    for (int h = 0; h < NCH; h++) mma<M, K>(c[h], a, b);
  __syncthreads();
  const long long t1 = clock64();
  if (threadIdx.x == 0) cyc[blockIdx.x] = (unsigned long long)(t1 - t0);
  double s = 0.0;
  for (int h = 0; h < NCH; h++)
    for (int i = 0; i < S::NC; i++) s += c[h][i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int M, int K> void run(const char* name, int nsm, double* src, double* out, unsigned long long* cyc) {
  // layout check
  double hA[16 * 16], hB[16 * 8], hC[16 * 8], ref[16 * 8];
  for (int i = 0; i < M * K; i++) hA[i] = (double)((i * 7) % 13) - 6.0;
  for (int i = 0; i < K * 8; i++) hB[i] = (double)((i * 5) % 11) - 5.0;
  for (int m = 0; m < M; m++)
    for (int n = 0; n < 8; n++) {
      double s = 0.0;
      for (int k = 0; k < K; k++) s += hA[m * K + k] * hB[k * 8 + n];
      ref[m * 8 + n] = s;
    }
  double *dA, *dB, *dC;
  CK(cudaMalloc(&dA, sizeof hA)); CK(cudaMalloc(&dB, sizeof hB)); CK(cudaMalloc(&dC, sizeof hC));
  CK(cudaMemcpy(dA, hA, sizeof hA, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dB, hB, sizeof hB, cudaMemcpyHostToDevice));
  layout_check<M, K><<<1, 32>>>(dA, dB, dC);
  CK(cudaGetLastError());
  CK(cudaMemcpy(hC, dC, sizeof hC, cudaMemcpyDeviceToHost));
  double err = 0.0;
  for (int i = 0; i < M * 8; i++) err = fmax(err, fabs(hC[i] - ref[i]));
  CK(cudaFree(dA)); CK(cudaFree(dB)); CK(cudaFree(dC));
  const double fma_per_mma = (double)M * 8 * K;
  for (int wps = 1; wps <= 4; wps *= 4) {   // warps per scheduler
    const int threads = 4 * 32 * wps, iters = 4096;
    rate<M, K><<<nsm, threads>>>(src, out, 64, cyc);   // warm-up
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    rate<M, K><<<nsm, threads>>>(src, out, iters, cyc);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaGetLastError());
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    unsigned long long* h = (unsigned long long*)malloc(nsm * sizeof(unsigned long long));
    CK(cudaMemcpy(h, cyc, nsm * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    double cmax = 0.0;
    for (int i = 0; i < nsm; i++) cmax = fmax(cmax, (double)h[i]);
    free(h);
    const double fma_cta = fma_per_mma * NCH * iters * (threads / 32);
    printf("%-9s layout_err %.1e  warps/scheduler %d  %7.1f FMA/clk/SM  %6.1f TFLOP/s\n", name, err, wps, fma_cta / cmax,
           2.0 * fma_cta * nsm / (ms * 1e-3) / 1e12);
    CK(cudaEventDestroy(e0)); CK(cudaEventDestroy(e1));
  }
}

int main() {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int nsm = prop.multiProcessorCount;
  printf("%s, %d SMs\n", prop.name, nsm);
  double *src, *out;
  unsigned long long* cyc;
  CK(cudaMalloc(&src, 256 * sizeof(double)));
  double hsrc[256];   // non-zero operands: zeros toggle less and would flatter a power-limited card
  for (int i = 0; i < 256; i++) hsrc[i] = 1e-3 * (1 + (i * 37) % 101);
  CK(cudaMemcpy(src, hsrc, sizeof hsrc, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&out, (size_t)nsm * 512 * sizeof(double)));
  CK(cudaMalloc(&cyc, nsm * sizeof(unsigned long long)));
  run<8, 4>("m8n8k4", nsm, src, out, cyc);
  run<16, 4>("m16n8k4", nsm, src, out, cyc);
  run<16, 8>("m16n8k8", nsm, src, out, cyc);
  run<16, 16>("m16n8k16", nsm, src, out, cyc);
  CK(cudaFree(src)); CK(cudaFree(out)); CK(cudaFree(cyc));
  return 0;
}
