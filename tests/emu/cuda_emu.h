// SIMT emulator -- TEST INFRASTRUCTURE ONLY (never part of the product, never loaded by
// rustpde_mpi_b200 itself).  It lets the CPU-only test suite compile the *same* kernel and host
// sources (lane_kernel.cuh, b200pde.cu) with g++ and run every CUDA thread of a block as an OS
// thread, so that host logic, lane programs and the per-thread index algebra of the kernels can be
// checked against the oracle without a GPU.  Build: tests/emu/build_emu.py -> tests/emu/libb200pde_emu.so
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __grid_constant__
#define __launch_bounds__(...)
#define __align__(x) alignas(x)
#define __shared__ static

struct alignas(16) double2 { double x, y; };
static inline double2 make_double2(double x, double y) { double2 r; r.x = x; r.y = y; return r; }
using std::fma;
using std::min;
using std::max;

namespace emu {
struct Dim3 { int x = 1, y = 1, z = 1; };

// Sense-reversing barrier on atomics: the waiters spin briefly and then yield (a mutex / condition-variable barrier wakes
// all waiters into one lock: with 32-512 OS threads per block on a few cores that dominated the run time of the suite)
class Barrier {
 public:
  void reset(int n) { n_ = n; count_.store(0); gen_.store(0); }
  void wait() {
    const unsigned g = gen_.load(std::memory_order_acquire);
    if (count_.fetch_add(1, std::memory_order_acq_rel) + 1 == n_) {
      count_.store(0, std::memory_order_relaxed);
      gen_.store(g + 1, std::memory_order_release);
    } else {
      int spins = 0;
      while (gen_.load(std::memory_order_acquire) == g) {
        if (++spins > 2000) std::this_thread::sleep_for(std::chrono::microseconds(50));   // a long wait (another rank's process): get off the cores
        else if (spins > 32) std::this_thread::yield();
      }
    }
  }
 private:
  int n_ = 1;
  std::atomic<int> count_{0};
  std::atomic<unsigned> gen_{0};
};

struct Warp { double buf[32]; double buf2[32]; Barrier bar; };

struct Block {
  Barrier bar;
  std::vector<Warp> warps{32};
  std::vector<char> dyn;
};

inline Block& block() { static Block* b = new Block; return *b; }
inline thread_local Dim3 t_threadIdx, t_blockIdx;
inline Dim3 g_blockDim, g_gridDim;
inline std::mutex g_atomic_mutex;

// persistent worker pool: worker i runs CUDA thread i of the current block
class Pool {
 public:
  static Pool& get() { static Pool* p = new Pool; return *p; }  // leaked on purpose: workers are detached
  void run_block(int T, const std::function<void()>& fn) {
    ensure(T);
    {
      std::lock_guard<std::mutex> lk(m_);
      fn_ = &fn; active_ = T; done_ = 0; gen_++;
    }
    cv_.notify_all();
    std::unique_lock<std::mutex> lk(m_);
    cv_done_.wait(lk, [&] { return done_ == active_; });
  }
 private:
  void ensure(int T) {
    while ((int)workers_.size() < T) {
      int id = (int)workers_.size();
      workers_.emplace_back([this, id] { loop(id); });
      workers_.back().detach();
    }
  }
  void loop(int id) {
    uint64_t seen = 0;
    for (;;) {
      const std::function<void()>* fn;
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (id >= active_) continue;
        fn = fn_;
      }
      t_threadIdx.x = id;
      (*fn)();
      {
        std::lock_guard<std::mutex> lk(m_);
        done_++;
      }
      cv_done_.notify_one();
    }
  }
  std::mutex m_; std::condition_variable cv_, cv_done_;
  std::vector<std::thread> workers_;
  const std::function<void()>* fn_ = nullptr;
  int active_ = 0, done_ = 0; uint64_t gen_ = 0;
};

template <class F> inline void launch(int grid, int blockdim, size_t smem, F&& body) {
  Block& b = block();
  g_blockDim.x = blockdim; g_gridDim.x = grid;
  b.dyn.assign(smem + 256, 0);
  b.bar.reset(blockdim);
  const int nw = (blockdim + 31) / 32;
  for (int w = 0; w < nw; w++) b.warps[w].bar.reset(std::min(32, blockdim - 32 * w));
  for (int bl = 0; bl < grid; bl++) {
    std::function<void()> fn = [&, bl] { t_blockIdx.x = bl; body(); };
    Pool::get().run_block(blockdim, fn);
  }
}

// mma.sync.m8n8k4.f64 for the emulated GEMM: A[row = lane / 4][k = lane % 4], B[k = lane % 4][col = lane / 4],
// C[row = lane / 4][col = 2 (lane % 4) + {0, 1}]; one exchange through the warp's buffers per instruction
inline void dmma884(double& c0, double& c1, double a, double b) {
  Warp& w = block().warps[t_threadIdx.x / 32];
  const int lane = t_threadIdx.x % 32, row = lane >> 2, col = 2 * (lane & 3);
  w.buf[lane] = a; w.buf2[lane] = b;
  w.bar.wait();
  for (int k = 0; k < 4; k++) {
    const double av = w.buf[row * 4 + k];
    c0 = std::fma(av, w.buf2[col * 4 + k], c0);
    c1 = std::fma(av, w.buf2[(col + 1) * 4 + k], c1);
  }
  w.bar.wait();
}

inline double shfl(double v, int src_lane) {
  Warp& w = block().warps[t_threadIdx.x / 32];
  const int lane = t_threadIdx.x % 32;
  w.buf[lane] = v;
  w.bar.wait();
  double r = w.buf[src_lane];
  w.bar.wait();
  return r;
}
}  // namespace emu

#define threadIdx emu::t_threadIdx
#define blockIdx emu::t_blockIdx
#define blockDim emu::g_blockDim
#define gridDim emu::g_gridDim

namespace emu {
// B2_EMU_SKEW_US=<us>[,rev|fwd]: a deterministic race schedule.  After every block barrier warp w sleeps before it resumes:
// rev (default) (nwarps - 1 - w) * us, so low warps resume last; fwd w * us, so high warps resume last.  A read that some
// warp makes after a barrier and that nothing orders against another warp's later write then loses the race every time.
// Unset: no sleep (the normal emulator).  One-warp blocks never sleep.
struct Skew { long us = 0; bool fwd = false; };
inline const Skew& skew() {
  static const Skew s = [] {
    Skew r;
    if (const char* e = getenv("B2_EMU_SKEW_US")) {
      r.us = std::max(0L, atol(e));
      const char* c = strchr(e, ',');
      r.fwd = c && strcmp(c + 1, "fwd") == 0;
    }
    return r;
  }();
  return s;
}
}  // namespace emu
static inline void __syncthreads() {
  emu::block().bar.wait();
  const emu::Skew& s = emu::skew();
  if (s.us > 0) {
    const int nw = (emu::g_blockDim.x + 31) / 32, w = emu::t_threadIdx.x / 32;
    const long d = s.fwd ? w : nw - 1 - w;
    if (d > 0) std::this_thread::sleep_for(std::chrono::microseconds(d * s.us));
  }
}
static inline void __syncwarp() { emu::block().warps[threadIdx.x / 32].bar.wait(); }
static inline double __shfl_up_sync(unsigned, double v, int d, int width = 32) {
  const int lane = threadIdx.x % 32;
  return emu::shfl(v, (lane % width) >= d ? lane - d : lane);
}
static inline double __shfl_down_sync(unsigned, double v, int d, int width = 32) {
  const int lane = threadIdx.x % 32;
  return emu::shfl(v, (lane % width) + d < width ? lane + d : lane);
}
static inline double __shfl_xor_sync(unsigned, double v, int d, int width = 32) {
  const int lane = threadIdx.x % 32;
  const int src = lane ^ d;
  return emu::shfl(v, (src / width == lane / width) ? src : lane);
}
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
  std::lock_guard<std::mutex> lk(emu::g_atomic_mutex);
  unsigned long long o = *p; *p = o + v; return o;
}
static inline long long clock64() { return 0; }
static inline double atomicAdd(double* p, double v) {
  std::lock_guard<std::mutex> lk(emu::g_atomic_mutex);
  double o = *p; *p = o + v; return o;
}

// ---- CUDA runtime subset used by the host code ----
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize };
static inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }
static inline cudaError_t cudaGetLastError() { return 0; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return 0; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { *p = (T*)aligned_alloc(256, (n + 255) / 256 * 256); return *p ? 0 : 1; }
static inline cudaError_t cudaFree(void* p) { free(p); return 0; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return 0; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, int) { *s = nullptr; return 0; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
enum cudaStreamCaptureStatus { cudaStreamCaptureStatusNone = 0 };
static inline cudaError_t cudaStreamIsCapturing(cudaStream_t, cudaStreamCaptureStatus* s) { *s = cudaStreamCaptureStatusNone; return 0; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return 0; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return 0; }
static inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
// CUDA IPC emulated with POSIX shared memory (multi-rank tests: one process per "GPU", gloo for the handles)
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
namespace emu {
struct Shm { void* p; size_t n; char name[48]; };
inline std::vector<Shm>& shms() { static std::vector<Shm>* v = new std::vector<Shm>; return *v; }
inline void unlink_all() { for (auto& s : shms()) shm_unlink(s.name); }
}  // namespace emu
static inline int b2_heap_malloc(void** p, size_t bytes) {
  static int counter = 0;
  emu::Shm s;
  snprintf(s.name, sizeof(s.name), "/b2emu_%d_%d", (int)getpid(), counter++);
  int fd = shm_open(s.name, O_CREAT | O_RDWR, 0600);
  if (fd < 0 || ftruncate(fd, (off_t)bytes) != 0) return 2;
  s.p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (s.p == MAP_FAILED) return 2;
  s.n = bytes;
  if (emu::shms().empty()) atexit(emu::unlink_all);
  emu::shms().push_back(s);
  *p = s.p;
  return 0;
}
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* ptr) {
  for (auto& s : emu::shms())
    if (s.p == ptr) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, s.name, sizeof(s.name)); memcpy(h->reserved + 48, &s.n, sizeof(size_t)); return 0; }
  return 1;
}
static inline cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, int) {
  size_t n; memcpy(&n, h.reserved + 48, sizeof(size_t));
  int fd = shm_open(h.reserved, O_RDWR, 0600);
  if (fd < 0) return 1;
  *p = mmap(nullptr, n, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  return *p == MAP_FAILED ? 1 : 0;
}
typedef void* cudaEvent_t;
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = malloc(8); return 0; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return 0; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return 0; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, int) { *e = malloc(8); return 0; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, int) { return 0; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0; return 0; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return 0; }

#define B2_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>((reinterpret_cast<uintptr_t>(emu::block().dyn.data()) + 127) & ~uintptr_t(127))
#define B2_LAUNCH(kernel, grid, block, smem, stream, ...) emu::launch((grid), (block), (smem), [&] { kernel(__VA_ARGS__); })
