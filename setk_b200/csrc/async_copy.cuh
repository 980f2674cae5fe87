// async_copy.cuh -- TMA 1-D bulk copies (cp.async.bulk, SASS UBLKCP) global ->
// shared completing on an mbarrier, used by the fused kernels to stream audio
// tiles one tile ahead of the math with zero issue-slot cost on the SM.
//
//   producer (one thread):  mbar_expect_tx(bar, total_bytes);
//                           bulk_g2s(dst, src, bytes, bar);   (any number, sum == total)
//   consumers (all threads): mbar_wait(bar, parity);          parity = phase & 1
//
// Sizes and both addresses must be multiples of 16 bytes.
// Under SETK_EMU the same protocol is modelled with atomics + memcpy.
#pragma once
#include "compat.cuh"

namespace setk {

struct alignas(8) MBar {
  unsigned long long v;
};

#ifdef SETK_EMU

// layout of the emulated barrier word: [63:56] magic, [55:48] arrival count of a phase,
// [47:40] arrivals still pending, [39:32] phase, [31:0] transaction bytes still pending
#define SETK_EMU_MBAR_MAGIC 0xB5ull
__device__ inline unsigned long long mbar_load(const MBar* b) {
  const unsigned long long v = __atomic_load_n(&b->v, __ATOMIC_SEQ_CST);
  if ((v >> 56) != SETK_EMU_MBAR_MAGIC)
    emu::die("mbarrier used before mbar_init (missing __syncthreads after init?)");
  return v;
}
__device__ inline void mbar_init(MBar* b, int count) {
  if (count < 1 || count > 255) emu::die("mbar_init: count");
  __atomic_store_n(&b->v, (SETK_EMU_MBAR_MAGIC << 56) | ((unsigned long long)count << 48) |
                              ((unsigned long long)count << 40), __ATOMIC_SEQ_CST);
}
// apply (arrivals, bytes) to the barrier; completes the phase when both reach zero
__device__ inline void mbar_update(MBar* b, int arrivals, long long bytes) {
  for (;;) {
    unsigned long long v = mbar_load(b);
    long long pend = (long long)((v >> 40) & 0xff) - arrivals;
    long long tx = (long long)(int)(v & 0xffffffffull) + bytes;
    if (pend < 0) emu::die("mbarrier: more arrivals than its count");
    unsigned long long phase = (v >> 32) & 0xff;
    const unsigned long long count = (v >> 48) & 0xff;
    if (pend == 0 && tx == 0) { phase = (phase + 1) & 0xff; pend = (long long)count; }
    const unsigned long long nv = (SETK_EMU_MBAR_MAGIC << 56) | (count << 48) |
                                  ((unsigned long long)pend << 40) | (phase << 32) |
                                  ((unsigned long long)(unsigned)(int)tx);
    if (__atomic_compare_exchange_n(&b->v, &v, nv, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) return;
  }
}
__device__ inline void fence_proxy_async() {}
__device__ inline void mbar_expect_tx(MBar* b, unsigned bytes) { mbar_update(b, 1, (long long)bytes); }
__device__ inline void mbar_add_tx(MBar* b, unsigned bytes) { mbar_update(b, 0, (long long)bytes); }
__device__ inline void mbar_arrive(MBar* b) { mbar_update(b, 1, 0); }
__device__ inline void bulk_g2s(void* dst, const void* src, unsigned bytes, MBar* b) {
  mbar_load(b);
  if ((bytes & 15u) || (reinterpret_cast<uintptr_t>(dst) & 15u) || (reinterpret_cast<uintptr_t>(src) & 15u))
    emu::die("cp.async.bulk needs 16-byte aligned addresses and size");
  memcpy(dst, src, bytes);
  mbar_update(b, 0, -(long long)bytes);
}
// returns once the phase with the given parity has completed (a fresh barrier has
// "completed" the phase of parity 1, as on the device)
__device__ inline void mbar_wait(MBar* b, unsigned parity) {
  long long spins = 0;
  while (((mbar_load(b) >> 32) & 1ull) == (unsigned long long)(parity & 1u)) {
    std::this_thread::yield();
    if (++spins > 400000000LL) emu::die("mbar_wait: no progress (deadlock in the kernel's protocol?)");
  }
}
// named barriers (bar.sync id, n) and the register re-budgeting of warp-specialised kernels
__device__ inline void named_bar_sync(int id, int nthreads) { emu::named_sync(id, nthreads); }
template <int R> __device__ inline void setmaxnreg_inc() {}
template <int R> __device__ inline void setmaxnreg_dec() {}
// 4-byte cp.async (LDGSTS): global -> shared without a register round trip
__device__ inline void cp_async_f32(float* dst, const float* src) { *dst = *src; }
__device__ inline void cp_async_8(void* dst, const void* src) { memcpy(dst, src, 8); }
__device__ inline void cp_async_wait_all() {}
__device__ inline void cp_async_commit() {}
__device__ inline void cp_async_wait_group1() {}

#else

__device__ __forceinline__ unsigned smem_u32(const void* p) {
  return static_cast<unsigned>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(MBar* b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// order prior generic-proxy accesses to shared memory before later async-proxy ones
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(MBar* b, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(MBar* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
// more transaction bytes for the current phase WITHOUT arriving (the caller arrives later itself)
__device__ __forceinline__ void mbar_add_tx(MBar* b, unsigned bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes)
               : "memory");
}
// named barrier among nthreads threads (a multiple of 32) of the CTA; id 1..15
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// warp-group register re-budgeting (SASS USETMAXREG); all warps of the warpgroup execute it
template <int R> __device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R> __device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, MBar* b) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(b))
      : "memory");
}
// One try: true when the phase with the given parity has completed.  The thread may be
// suspended by the hardware for up to `hint_ns` while it waits (it wakes when the phase
// completes), which keeps a long wait from burning issue slots in a polling loop.
__device__ __forceinline__ bool mbar_try_wait(MBar* b, unsigned parity, unsigned hint_ns) {
  unsigned ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity), "r"(hint_ns)
      : "memory");
  return ok != 0;
}
#ifndef SETK_MBAR_HINT_NS
#define SETK_MBAR_HINT_NS 20000
#endif
__device__ __forceinline__ bool mbar_try_wait_nohint(MBar* b, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(MBar* b, unsigned parity) {
#if SETK_MBAR_HINT_NS > 0
  while (!mbar_try_wait(b, parity, SETK_MBAR_HINT_NS)) {}
#else
  while (!mbar_try_wait_nohint(b, parity)) {}
#endif
}

// 4-byte cp.async (LDGSTS): global -> shared without a register round trip
__device__ __forceinline__ void cp_async_f32(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// 8-byte cp.async (one complex64 or one double)
__device__ __forceinline__ void cp_async_8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// all but the most recently committed group have landed
__device__ __forceinline__ void cp_async_wait_group1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

#endif

}  // namespace setk
