// The banded operators' coefficients as the device forms them (band_coef.cuh), compiled for the GPU exactly as the library is,
// written out for tests/test_band_coef_hardware.py to compare bit for bit with the host's values.  The emulator build of the same
// functions (tests/test_emu_band_coefficients.py) seeds the Newton steps with its own 20-bit reciprocal; only this build runs
// them from the hardware's rcp.approx.ftz.f64.
//
// usage: band_coef_harness OUT.bin   (raw little-endian doubles, in this order)
//   for n = 9, 17, ..., 8193:
//     families: [f = 1 .. 8][i = 0 .. n + 7] band_coef(f, i, n)   (BC_UNIT .. BC_PV4)
//     for CP in 5, 9, 17: BandPairs<BC_PV0, BC_PV2, BC_PV4> walked by chunks of CP pairs starting at p0 = 0, CP, 2 CP, ...
//       while 2 p0 < n + 4: [element i][k0, k1, k2] for i < 2 CP (number of chunks)
//   quotients: [i = 0 .. 2^20 - 1][bc_rcp(4 r (r - 1)), bc_rcp(2 (r^2 - 1)), bc_rcp(4 r (r + 1)), bc_div(i, i + 2)], r = i + 2
//     (row 0 is zero)
#include <cstdio>
#include <vector>

#include "band_coef.cuh"

#define CK(x)                                                                                     \
  do {                                                                                            \
    cudaError_t e_ = (x);                                                                         \
    if (e_ != cudaSuccess) {                                                                      \
      std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));     \
      return 1;                                                                                   \
    }                                                                                             \
  } while (0)

static const int NQ = 1 << 20;

__global__ void families(int n, double* out) {
  const int len = n + 8, t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < 8 * len) out[t] = band_coef(BC_UNIT + t / len, t % len, n);
}

// one thread per chunk, the pair loop unrolled as the lane kernel's chunk loops are
template <int CP>
__global__ void pairs(int n, int nch, double* out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nch) return;
  const int p0 = c * CP;
  BandPairs<BC_PV0, BC_PV2, BC_PV4> pv(n, 2 * p0);
#pragma unroll
  for (int t = 0; t < CP; t++) {
    const int e = 2 * (p0 + t);
    double2 k0, k1, k2;
    pv.at(e, k0, k1, k2);
    double* o = out + 3 * e;
    o[0] = k0.x; o[1] = k1.x; o[2] = k2.x;
    o[3] = k0.y; o[4] = k1.y; o[5] = k2.y;
  }
}

__global__ void quotients(double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NQ) return;
  double* o = out + 4 * (size_t)i;
  if (i == 0) { o[0] = o[1] = o[2] = o[3] = 0.0; return; }
  const double r = i + 2;
  o[0] = bc_rcp(4.0 * r * (r - 1.0));
  o[1] = bc_rcp(2.0 * (r * r - 1.0));
  o[2] = bc_rcp(4.0 * r * (r + 1.0));
  o[3] = bc_div((double)i, i + 2.0);
}

template <int CP>
static int run_pairs(int n, double* d, std::vector<double>& all) {
  int nch = 0;
  for (int p0 = 0; 2 * p0 < n + 4; p0 += CP) nch++;
  const size_t len = (size_t)3 * 2 * CP * nch;
  pairs<CP><<<(nch + 127) / 128, 128>>>(n, nch, d);
  CK(cudaGetLastError());
  std::vector<double> h(len);
  CK(cudaMemcpy(h.data(), d, len * sizeof(double), cudaMemcpyDeviceToHost));
  all.insert(all.end(), h.begin(), h.end());
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 2) { std::fprintf(stderr, "usage: %s OUT.bin\n", argv[0]); return 2; }
  double* d = nullptr;
  CK(cudaMalloc(&d, (size_t)4 * NQ * sizeof(double)));
  std::vector<double> all;
  for (int n = 9; n <= 8193; n = 2 * n - 1) {
    const int len = 8 * (n + 8);
    families<<<(len + 255) / 256, 256>>>(n, d);
    CK(cudaGetLastError());
    std::vector<double> h(len);
    CK(cudaMemcpy(h.data(), d, len * sizeof(double), cudaMemcpyDeviceToHost));
    all.insert(all.end(), h.begin(), h.end());
    if (run_pairs<5>(n, d, all) || run_pairs<9>(n, d, all) || run_pairs<17>(n, d, all)) return 1;
  }
  quotients<<<NQ / 256, 256>>>(d);
  CK(cudaGetLastError());
  std::vector<double> h((size_t)4 * NQ);
  CK(cudaMemcpy(h.data(), d, h.size() * sizeof(double), cudaMemcpyDeviceToHost));
  all.insert(all.end(), h.begin(), h.end());
  CK(cudaFree(d));
  FILE* f = std::fopen(argv[1], "wb");
  if (!f || std::fwrite(all.data(), sizeof(double), all.size(), f) != all.size() || std::fclose(f)) {
    std::fprintf(stderr, "cannot write %s\n", argv[1]);
    return 1;
  }
  std::printf("wrote %zu coefficients\n", all.size());
  return 0;
}
