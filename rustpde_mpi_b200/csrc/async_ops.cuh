// Asynchronous data movement for the lane kernel: TMA tensor copies (global <-> shared), mbarriers,
// bulk async-groups and named barriers, as thin wrappers over sm_90a PTX.
//
// Why: a lane group is a 64-131 KB slab; moving it with per-thread LDG/STG costs registers, issue slots and
// exposes DRAM latency to every warp.  With TMA one elected thread describes a whole chunk (a box of
// 4x4 tiles) and the copy engine streams it into a shared-memory ring while all warps compute; the
// transposing store (the x<->y pencil switch) becomes one 4-D tensor store per chunk.
//
// Under B2_EMU (tests/emu, CPU-only test infrastructure) the same entry points are implemented with
// mutexes/condition variables and memcpy so that the pipeline logic can be unit-tested without a GPU.
#pragma once
#include <stdint.h>

// A tensor map: 128 opaque bytes (CUtensorMap on the GPU; struct EmuTMap under the emulator).
struct alignas(64) B2TMap { unsigned char opaque[128]; };

struct B2TMapDesc {   // host-side description, encoded by b2_encode_tmap()
  void* base;
  int rank;                 // 2..4
  uint64_t dim[4];          // elements (f64), innermost first
  uint64_t stride[4];       // bytes; stride[0] is implied (8)
  uint32_t box[4];          // elements
};

#ifdef B2_EMU
// ------------------------------------------------------------------------------------------------
// emulator implementation
// ------------------------------------------------------------------------------------------------
#include <map>
namespace emu {
struct EmuTMap { void* base; int rank; uint64_t dim[4]; uint64_t stride[4]; uint32_t box[4]; };
static_assert(sizeof(EmuTMap) <= 128, "EmuTMap must fit the opaque map");
struct MBar { int expected = 0, pending = 0; long long tx = 0; unsigned phase = 0; };
inline std::mutex g_mbar_mutex;
inline std::condition_variable g_mbar_cv;
inline std::map<const void*, MBar>& mbars() { static auto* m = new std::map<const void*, MBar>; return *m; }
inline void mbar_complete_locked(MBar& b) {
  if (b.pending == 0 && b.tx == 0) { b.phase ^= 1u; b.pending = b.expected; g_mbar_cv.notify_all(); }
}
inline std::map<int, Barrier*>& named_bars() { static auto* m = new std::map<int, Barrier*>; return *m; }
inline std::mutex g_named_mutex;
// box copy with out-of-bounds handling: loads zero-fill, stores / reductions clip
inline void tma_copy(const EmuTMap& m, const int* c, double* smem, int mode /*0 load, 1 store, 2 reduce-add*/) {
  uint32_t bx[4] = {1, 1, 1, 1}; uint64_t dm[4] = {1, 1, 1, 1}, st[4] = {8, 0, 0, 0}; long long cc[4] = {0, 0, 0, 0};
  for (int i = 0; i < m.rank; i++) { bx[i] = m.box[i]; dm[i] = m.dim[i]; st[i] = i ? m.stride[i] : 8; cc[i] = c[i]; }
  size_t s = 0;
  for (uint32_t i3 = 0; i3 < bx[3]; i3++)
    for (uint32_t i2 = 0; i2 < bx[2]; i2++)
      for (uint32_t i1 = 0; i1 < bx[1]; i1++)
        for (uint32_t i0 = 0; i0 < bx[0]; i0++, s++) {
          const long long g[4] = {cc[0] + i0, cc[1] + i1, cc[2] + i2, cc[3] + i3};
          bool in = true;
          for (int i = 0; i < 4; i++) in = in && g[i] >= 0 && (uint64_t)g[i] < dm[i];
          double* gp = in ? reinterpret_cast<double*>(static_cast<char*>(m.base) + g[0] * st[0] + g[1] * st[1] + g[2] * st[2] + g[3] * st[3]) : nullptr;
          if (mode == 0) smem[s] = in ? *gp : 0.0;
          else if (in) { if (mode == 1) *gp = smem[s]; else { std::lock_guard<std::mutex> lk(g_atomic_mutex); *gp += smem[s]; } }
        }
}
}  // namespace emu

static inline void mbar_init(uint64_t* bar, int count) {
  std::lock_guard<std::mutex> lk(emu::g_mbar_mutex);
  emu::MBar& b = emu::mbars()[bar]; b.expected = count; b.pending = count; b.tx = 0; b.phase = 0;
}
static inline void mbar_fence_init() {}
static inline void mbar_arrive(uint64_t* bar) {
  std::lock_guard<std::mutex> lk(emu::g_mbar_mutex);
  emu::MBar& b = emu::mbars()[bar]; b.pending--; emu::mbar_complete_locked(b);
}
static inline void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  std::lock_guard<std::mutex> lk(emu::g_mbar_mutex);
  emu::MBar& b = emu::mbars()[bar]; b.tx += bytes; b.pending--; emu::mbar_complete_locked(b);
}
static inline void mbar_wait(uint64_t* bar, unsigned parity) {   // returns once the phase with this parity has completed
  std::unique_lock<std::mutex> lk(emu::g_mbar_mutex);
  emu::MBar& b = emu::mbars()[bar];
  emu::g_mbar_cv.wait(lk, [&] { return b.phase != parity; });
}
static inline bool mbar_test(uint64_t* bar, unsigned parity) {   // non-blocking: has the phase with this parity completed?
  std::lock_guard<std::mutex> lk(emu::g_mbar_mutex);
  return emu::mbars()[bar].phase != parity;
}
static inline void emu_tx_done(uint64_t* bar, long long bytes) {
  std::lock_guard<std::mutex> lk(emu::g_mbar_mutex);
  emu::MBar& b = emu::mbars()[bar]; b.tx -= bytes; emu::mbar_complete_locked(b);
}
static inline long long emu_box_bytes(const B2TMap* m) {
  const emu::EmuTMap& e = *reinterpret_cast<const emu::EmuTMap*>(m); long long n = 8;
  for (int i = 0; i < e.rank; i++) n *= e.box[i];
  return n;
}
static inline void tma_load_2d(void* dst, const B2TMap* m, int c0, int c1, uint64_t* bar) {
  const int c[4] = {c0, c1, 0, 0};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, static_cast<double*>(dst), 0);
  emu_tx_done(bar, emu_box_bytes(m));
}
static inline void tma_load_3d(void* dst, const B2TMap* m, int c0, int c1, int c2, uint64_t* bar) {
  const int c[4] = {c0, c1, c2, 0};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, static_cast<double*>(dst), 0);
  emu_tx_done(bar, emu_box_bytes(m));
}
static inline void tma_store_3d(const B2TMap* m, int c0, int c1, int c2, const void* src) {
  const int c[4] = {c0, c1, c2, 0};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, const_cast<double*>(static_cast<const double*>(src)), 1);
}
static inline void tma_reduce_add_3d(const B2TMap* m, int c0, int c1, int c2, const void* src) {
  const int c[4] = {c0, c1, c2, 0};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, const_cast<double*>(static_cast<const double*>(src)), 2);
}
static inline void tma_store_2d(const B2TMap* m, int c0, int c1, const void* src) {
  const int c[4] = {c0, c1, 0, 0};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, const_cast<double*>(static_cast<const double*>(src)), 1);
}
static inline void tma_store_4d(const B2TMap* m, int c0, int c1, int c2, int c3, const void* src) {
  const int c[4] = {c0, c1, c2, c3};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, const_cast<double*>(static_cast<const double*>(src)), 1);
}
static inline void tma_reduce_add_4d(const B2TMap* m, int c0, int c1, int c2, int c3, const void* src) {
  const int c[4] = {c0, c1, c2, c3};
  emu::tma_copy(*reinterpret_cast<const emu::EmuTMap*>(m), c, const_cast<double*>(static_cast<const double*>(src)), 2);
}
static inline void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) { memcpy(dst, src, bytes); emu_tx_done(bar, bytes); }
static inline void bulk_store_1d(void* dst, const void* src, uint32_t bytes) { memcpy(dst, src, bytes); }
static inline void bulk_reduce_add_1d(void* dst, const void* src, uint32_t bytes) {
  std::lock_guard<std::mutex> lk(emu::g_atomic_mutex);
  for (uint32_t i = 0; i < bytes / 8; i++) static_cast<double*>(dst)[i] += static_cast<const double*>(src)[i];
}
static inline void tmap_prefetch(const B2TMap*) {}
static inline void bulk_commit() {}
template <int N> static inline void bulk_wait_read() {}
template <int N> static inline void bulk_wait() {}
static inline void fence_proxy_async() {}
static inline void named_barrier(int id, int count) {
  emu::Barrier* b;
  {
    std::lock_guard<std::mutex> lk(emu::g_named_mutex);
    auto& m = emu::named_bars();
    auto it = m.find(id * 4096 + count);
    if (it == m.end()) { b = new emu::Barrier; b->reset(count); m[id * 4096 + count] = b; } else b = it->second;
  }
  b->wait();
}
static inline int b2_encode_tmap(const B2TMapDesc& d, B2TMap* out) {
  emu::EmuTMap e; memset(&e, 0, sizeof(e));
  e.base = d.base; e.rank = d.rank;
  for (int i = 0; i < d.rank; i++) { e.dim[i] = d.dim[i]; e.stride[i] = d.stride[i]; e.box[i] = d.box[i]; }
  memset(out, 0, sizeof(*out)); memcpy(out->opaque, &e, sizeof(e));
  return 0;
}
#else
// ------------------------------------------------------------------------------------------------
// sm_90a implementation
// ------------------------------------------------------------------------------------------------
#include <cuda.h>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ bool mbar_test(uint64_t* bar, unsigned parity) {   // non-blocking: has the phase with this parity completed?
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const B2TMap* m, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const B2TMap* m, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const B2TMap* m, int c0, int c1, int c2, const void* src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const B2TMap* m, int c0, int c1, int c2, const void* src) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%1, %2, %3}], [%4];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const B2TMap* m, int c0, int c1, const void* src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const B2TMap* m, int c0, int c1, int c2, int c3, const void* src) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%1, %2, %3, %4}], [%5];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(src)) : "memory");
}
__device__ __forceinline__ void tma_reduce_add_4d(const B2TMap* m, int c0, int c1, int c2, int c3, const void* src) {
  asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%1, %2, %3, %4}], [%5];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(src)) : "memory");
}
// contiguous (1-D) bulk copies: addresses and size multiples of 16 bytes
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_store_1d(void* dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(reinterpret_cast<uint64_t>(dst)), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_reduce_add_1d(void* dst, const void* src, uint32_t bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], %2;"
               ::"l"(reinterpret_cast<uint64_t>(dst)), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tmap_prefetch(const B2TMap* m) { asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_barrier(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// host: encode a CUtensorMap through the driver entry point (no link-time dependency on libcuda)
static inline int b2_encode_tmap(const B2TMapDesc& d, B2TMap* out) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return 1;
    fn = reinterpret_cast<EncodeFn>(p);
  }
  static_assert(sizeof(CUtensorMap) == sizeof(B2TMap), "tensor map size");
  cuuint64_t dims[4], strides[3];
  cuuint32_t box[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < d.rank; i++) { dims[i] = d.dim[i]; box[i] = d.box[i]; if (i) strides[i - 1] = d.stride[i]; }
  CUresult r = fn(reinterpret_cast<CUtensorMap*>(out), CU_TENSOR_MAP_DATA_TYPE_FLOAT64, (cuuint32_t)d.rank, d.base, dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r + 1000;
}
#endif
