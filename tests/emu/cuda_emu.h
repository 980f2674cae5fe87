// tests/emu/cuda_emu.h -- a tiny CUDA-on-CPU execution model.
//
// TEST INFRASTRUCTURE ONLY.  It lets the *actual kernel sources* under
// setk_b200/csrc/ be compiled with g++ (-DSETK_EMU) into
// tests/emu/libsetk_b200_emu.so so that index bookkeeping, shared-memory
// staging, barrier structure and the C-ABI argument checking can be exercised
// in the CPU test tier (`pytest -m "not gpu"`), where no GPU exists.  The
// product (setk_b200/_lib.py) never loads the emulated library; it loads
// libsetk_b200.so (nvcc, sm_90a) and fails loudly if that is missing.
//
// Model: CTAs run one after another; each CTA is blockDim OS threads;
// __syncthreads / __syncwarp are counting barriers that exited threads drop
// out of (as on sm_70+); warp shuffles go through a per-CTA slot array;
// `__shared__` becomes `static` (valid because CTAs are serialised);
// "device memory" is host memory.
#pragma once
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

// ---------------------------------------------------------------- types ----
struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) double2 { double x, y; };
struct int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline double2 make_double2(double x, double y) { return double2{x, y}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }

// ------------------------------------------------------------ qualifiers ---
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __restrict__ __restrict
#define __launch_bounds__(...)
#define __maxnreg__(...)
#define __shared__ static
#define __constant__ static
#define __align__(n) alignas(n)

// ------------------------------------------------------------- runtime ----
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost,
                      cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
static inline cudaError_t cudaMalloc(void** p, size_t n) {
  *p = aligned_alloc(256, (n + 255) / 256 * 256 + 256);
  return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocAsync(void** p, size_t n, cudaStream_t) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeAsync(void* p, cudaStream_t) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) {
  memcpy(d, s, n); return cudaSuccess;
}
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) {
  memcpy(d, s, n); return cudaSuccess;
}
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) {
  memset(d, v, n); return cudaSuccess;
}
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 4; return cudaSuccess; }
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int) { return cudaSuccess; }

// ------------------------------------------------------------ execution ---
namespace emu {

struct Barrier {
  // Arrival is one compare-and-swap on {generation, arrived} (no mutex: a CTA is 128-512 OS threads
  // and every __syncthreads / __syncwarp / named barrier of every thread used to take the same lock);
  // the mutex + condition variable only serve threads that give up spinning.
  std::mutex m;
  std::condition_variable cv;
  std::atomic<int> expected{0};
  std::atomic<uint64_t> state{0};           // (generation << 32) | arrived
  std::atomic<int> sleepers{0};
  void init(int n) { expected.store(n); state.store(0); sleepers.store(0); }
  void wake() {
    if (sleepers.load(std::memory_order_acquire) > 0) {
      { std::lock_guard<std::mutex> lk(m); }
      cv.notify_all();
    }
  }
  unsigned generation() const { return (unsigned)(state.load(std::memory_order_acquire) >> 32); }
  void wait() {
    uint64_t s = state.load(std::memory_order_acquire);
    unsigned g;
    for (;;) {
      g = (unsigned)(s >> 32);
      const int arrived = (int)(s & 0xffffffffu) + 1;
      const bool last = arrived >= expected.load(std::memory_order_acquire);
      const uint64_t ns = last ? ((uint64_t)(g + 1) << 32) : (((uint64_t)g << 32) | (unsigned)arrived);
      if (state.compare_exchange_weak(s, ns, std::memory_order_acq_rel, std::memory_order_acquire)) {
        if (last) { wake(); return; }
        // a thread may have dropped out between our read of `expected` and this arrival (it saw us
        // not yet arrived and left the release to us): look again
        if (arrived >= expected.load(std::memory_order_acquire)) {
          uint64_t cur = ns;
          if (state.compare_exchange_strong(cur, (uint64_t)(g + 1) << 32, std::memory_order_acq_rel)) {
            wake();
            return;
          }
        }
        break;
      }
    }
    // spin first (kernels with many short barrier episodes), then block
    for (int i = 0; i < 4000; ++i) {
      if (generation() != g) return;
      if ((i & 15) == 15) std::this_thread::yield();
    }
    std::unique_lock<std::mutex> lk(m);
    sleepers.fetch_add(1, std::memory_order_acq_rel);
    cv.wait(lk, [&] { return generation() != g; });
    sleepers.fetch_sub(1, std::memory_order_acq_rel);
  }
  void drop() {  // a thread that exited no longer participates
    const int e = expected.fetch_sub(1, std::memory_order_acq_rel) - 1;
    uint64_t s = state.load(std::memory_order_acquire);
    for (;;) {
      const int arrived = (int)(s & 0xffffffffu);
      if (e <= 0 || arrived == 0 || arrived < e) return;
      const uint64_t ns = (uint64_t)((unsigned)(s >> 32) + 1) << 32;
      if (state.compare_exchange_weak(s, ns, std::memory_order_acq_rel, std::memory_order_acquire)) {
        wake();
        return;
      }
    }
  }
};

struct Ctx {
  int nthreads = 0;
  Barrier cta;
  std::vector<Barrier> warps;
  Barrier named[16];              // bar.sync id, n (id 1..15)
  std::mutex named_m;
  std::vector<uint64_t> slots;
  std::vector<float> gather;      // [nthreads][8]: warp all-gather scratch (emulated mma.sync)
  unsigned char* dyn = nullptr;
  bool serial = false;
};

extern thread_local Ctx* g_ctx;
extern thread_local int g_tid;
static constexpr size_t kDynBytes = 256 * 1024;

inline void die(const char* msg) { fprintf(stderr, "cuda_emu: %s\n", msg); abort(); }

template <class F>
void launch(dim3 grid, dim3 block, size_t smem, bool serial, F&& body);

}  // namespace emu

extern thread_local uint3 threadIdx, blockIdx;
extern thread_local dim3 blockDim, gridDim;

namespace emu {
template <class F>
void launch(dim3 grid, dim3 block, size_t smem, bool serial, F&& body) {
  if (smem > kDynBytes) die("dynamic shared memory request too large");
  const int nthr = (int)(block.x * block.y * block.z);
  static unsigned char* dyn = (unsigned char*)aligned_alloc(1024, kDynBytes);
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        Ctx ctx;
        ctx.nthreads = nthr;
        ctx.serial = serial;
        ctx.dyn = dyn;
        ctx.cta.init(nthr);
        ctx.warps = std::vector<Barrier>((nthr + 31) / 32);
        for (int w = 0; w < (int)ctx.warps.size(); ++w) {
          int n = nthr - 32 * w; ctx.warps[w].init(n > 32 ? 32 : n);
        }
        ctx.slots.assign(nthr, 0);
        ctx.gather.assign((size_t)nthr * 8, 0.f);
        memset(dyn, 0xCD, smem);   // shared memory starts as garbage, like on the device
        auto run = [&](int tid) {
          g_ctx = &ctx; g_tid = tid;
          threadIdx = uint3{tid % block.x, (tid / block.x) % block.y, tid / (block.x * block.y)};
          blockIdx = uint3{bx, by, bz};
          blockDim = block; gridDim = grid;
          body();
          if (!serial) { ctx.cta.drop(); ctx.warps[tid / 32].drop(); }
        };
        if (serial) {
          for (int t = 0; t < nthr; ++t) run(t);
        } else {
          std::vector<std::thread> th;
          th.reserve(nthr);
          for (int t = 0; t < nthr; ++t) th.emplace_back(run, t);
          for (auto& t : th) t.join();
        }
      }
}
inline void sync_cta() {
  if (g_ctx->serial) die("__syncthreads in a kernel launched as barrier-free");
  g_ctx->cta.wait();
}
// bar.sync id, nthreads: the first arrival fixes the participant count
inline void named_sync(int id, int nthreads) {
  if (g_ctx->serial) die("named barrier in a kernel launched as barrier-free");
  if (id < 1 || id > 15) die("named barrier id");
  Barrier& b = g_ctx->named[id];
  {
    std::unique_lock<std::mutex> lk(g_ctx->named_m);
    if (b.expected.load() == 0) b.init(nthreads);
    else if (b.expected.load() != nthreads) die("named barrier used with two different thread counts");
  }
  b.wait();
}
inline void sync_warp() {
  if (g_ctx->serial) die("__syncwarp in a kernel launched as barrier-free");
  g_ctx->warps[g_tid / 32].wait();
}
// every lane of the warp contributes n <= 8 floats; all[i * 32 + l] = value i of lane l
inline void warp_allgather(const float* mine, int n, float* all) {
  float* buf = g_ctx->gather.data();
  for (int i = 0; i < n; ++i) buf[(size_t)g_tid * 8 + i] = mine[i];
  sync_warp();
  const int w0 = g_tid & ~31;
  for (int l = 0; l < 32; ++l) {
    const int src = w0 + l < g_ctx->nthreads ? w0 + l : g_tid;
    for (int i = 0; i < n; ++i) all[i * 32 + l] = buf[(size_t)src * 8 + i];
  }
  sync_warp();
}
template <class T>
inline T shfl_idx(T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle payload");
  uint64_t bits = 0; memcpy(&bits, &v, sizeof(T));
  g_ctx->slots[g_tid] = bits;
  sync_warp();
  int src = (g_tid & ~31) + (src_lane & 31);
  if (src >= g_ctx->nthreads) src = g_tid;
  uint64_t r = g_ctx->slots[src];
  sync_warp();
  T out; memcpy(&out, &r, sizeof(T));
  return out;
}
}  // namespace emu

static inline void __syncthreads() { emu::sync_cta(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::sync_warp(); }
template <class T> static inline T __shfl_sync(unsigned, T v, int lane, int = 32) { return emu::shfl_idx(v, lane); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) { return emu::shfl_idx(v, (emu::g_tid & 31) ^ m); }
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d, int = 32) {
  int l = (emu::g_tid & 31) + (int)d; return emu::shfl_idx(v, l > 31 ? (emu::g_tid & 31) : l);
}
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32) {
  int l = (emu::g_tid & 31) - (int)d; return emu::shfl_idx(v, l < 0 ? (emu::g_tid & 31) : l);
}

// -------------------------------------------------------------- atomics ---
static inline unsigned atomicMax(unsigned* a, unsigned v) {
  unsigned old = __atomic_load_n(a, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(a, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
static inline int atomicMax(int* a, int v) {
  int old = __atomic_load_n(a, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(a, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
static inline unsigned atomicOr(unsigned* a, unsigned v) { return __atomic_fetch_or(a, v, __ATOMIC_RELAXED); }
static inline unsigned long long atomicMax(unsigned long long* a, unsigned long long v) {
  unsigned long long old = __atomic_load_n(a, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(a, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
static inline long long __double_as_longlong(double f) { long long u; memcpy(&u, &f, 8); return u; }
static inline double __longlong_as_double(long long u) { double f; memcpy(&f, &u, 8); return f; }
static inline unsigned atomicAdd(unsigned* a, unsigned v) { return __atomic_fetch_add(a, v, __ATOMIC_RELAXED); }
static inline int atomicAdd(int* a, int v) { return __atomic_fetch_add(a, v, __ATOMIC_RELAXED); }
static inline unsigned long long atomicAdd(unsigned long long* a, unsigned long long v) {
  return __atomic_fetch_add(a, v, __ATOMIC_RELAXED);
}
static inline float atomicAdd(float* a, float v) {
  uint32_t* p = (uint32_t*)a; uint32_t old = __atomic_load_n(p, __ATOMIC_RELAXED);
  for (;;) {
    float f; memcpy(&f, &old, 4); f += v; uint32_t nw; memcpy(&nw, &f, 4);
    if (__atomic_compare_exchange_n(p, &old, nw, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) { memcpy(&f, &old, 4); return f; }
  }
}
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

// ----------------------------------------------------------------- math ---
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline void sincospi(double x, double* s, double* c) { *s = sin(M_PI * x); *c = cos(M_PI * x); }
static inline void sincospif(float x, float* s, float* c) {
  *s = (float)sin(M_PI * (double)x); *c = (float)cos(M_PI * (double)x);
}
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline double rsqrt(double x) { return 1.0 / sqrt(x); }
static inline float __fdividef(float a, float b) { return a / b; }
// round-to-nearest single operations that the compiler must not contract into an FMA
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline unsigned __brev(unsigned v) {
  unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((v >> i) & 1u) << (31 - i); return r;
}
#ifndef min
template <class T> static inline T min(T a, T b) { return a < b ? a : b; }
template <class T> static inline T max(T a, T b) { return a > b ? a : b; }
#endif
