// sm90.cuh — thin inline-PTX wrappers for the sm_90a features the renderer uses:
// mbarrier, bulk-async copy (TMA), warpgroup MMA (wgmma) with shared-memory operand descriptors.
// No CUTLASS/CuTe dependency: the descriptor bit layout follows the PTX ISA "matrix descriptor" table of
// wgmma (asynchronous warpgroup level matrix shared memory layout).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include "wgmma_ss.cuh"

namespace pnr {

#ifndef PNR_WATCHDOG_CYCLES
#define PNR_WATCHDOG_CYCLES (8000000000LL)  // ~4 s @ 2 GHz: a stuck barrier traps instead of hanging the box
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// One lane of a fully converged warp (PTX elect.sync): the compiler knows the guarded code is single-thread.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// The MMA-issuing warps wait here while earlier wgmmas are in flight: no call (printf) in the loop, or ptxas
// serializes every wgmma of the kernel.  The watchdog traps without a message.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > PNR_WATCHDOG_CYCLES) __trap();
}
// One arrival on `bar` if `pred` (a predicated instruction, not a branch: safe next to in-flight wgmmas).
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %1, 0;\n\t"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(bar),
      "r"((uint32_t)pred)
      : "memory");
}
// mbar_wait for warps whose waits are long (the weight-stream warp): back off between polls so the spinning warp
// does not take issue slots from the MMA-issuing warpgroup that shares its scheduler.  No printf either: ptxas
// serializes the wgmmas of a kernel that contains a call, on whichever warp it runs.
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(40);
    if ((++spins & 0x3FFu) == 0 && (clock64() - t0) > PNR_WATCHDOG_CYCLES) __trap();
  }
}

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// ---------------------------------------------------------------- proxies / bulk copy
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 1-D bulk async copy global -> shared, completion counted in bytes on an mbarrier (TMA engine).
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          dst_smem),
      "l"(src_gmem), "r"(bytes), "r"(bar)
      : "memory");
}

// ---------------------------------------------------------------- named barriers
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor, K-major, no swizzle ("interleaved" 8 x 16-byte core matrices, each stored as 128
// contiguous bytes).  lbo_bytes: distance between the core matrices adjacent in K (one K16 step reads two of them);
// sbo_bytes: distance between 8-row groups along M / N.
__device__ __forceinline__ uint64_t make_smem_desc_noswz(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;   // base offset 0, layout type 0 = no swizzle
}
// Operand element formats (template argument of the kernels and of Wgmma<N, FMT>).
constexpr int kFmtF16 = 0, kFmtBF16 = 1;

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// ksteps K16 steps of D (+)= A * B^T, each PASSES products (x3: A_hi B_hi + A_lo B_hi + A_hi B_lo); the descriptors'
// address fields advance by a_inc16 / b_inc16 (16-byte units) per step.  acc = 0: the first product overwrites D.
template <int N, int PASSES, int FMT>
__device__ __forceinline__ void mma_run(float* d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, int ksteps,
                                        uint32_t a_inc16, uint32_t b_inc16, uint32_t acc) {
#pragma unroll 1
  for (int ks = 0; ks < ksteps; ++ks) {
    const uint64_t ao = (uint64_t)(ks * a_inc16), bo = (uint64_t)(ks * b_inc16);   // address field, 16-byte units
    Wgmma<N, FMT>::run(d, a_hi + ao, b_hi + bo, ks == 0 ? acc : 1u);
    if (PASSES == 3) {
      Wgmma<N, FMT>::run(d, a_lo + ao, b_hi + bo, 1u);
      Wgmma<N, FMT>::run(d, a_hi + ao, b_lo + bo, 1u);
    }
  }
}

// mma_run (x3) over NP = 16 .. 256 columns (N rounded up to 16) as two wgmma halves of <= 128 columns: the first into
// d0, the rest - from row 128 of the B images on - into d1.  Fences; the caller commits and waits.
template <int FMT>
__device__ __forceinline__ void mma_run_halves(float (&d0)[64], float (&d1)[64], int NP, uint64_t a_hi, uint64_t a_lo,
                                               uint64_t b_hi, uint64_t b_lo, int ksteps, uint32_t a_inc16,
                                               uint32_t b_inc16, uint32_t acc) {
  const int n0 = NP < 128 ? NP : 128;
  const uint64_t h1 = (128u * 16u) >> 4;   // row 128 of the B images, 16-byte units
  wgmma_fence();
#define PNR_HALF_N(NN, D, BH, BL) \
  case NN / 8: mma_run<NN, 3, FMT>(D, a_hi, a_lo, BH, BL, ksteps, a_inc16, b_inc16, acc); break;
#define PNR_HALF_ALL(D, BH, BL)                                                                                   \
  PNR_HALF_N(16, D, BH, BL) PNR_HALF_N(32, D, BH, BL) PNR_HALF_N(48, D, BH, BL) PNR_HALF_N(64, D, BH, BL)            \
  PNR_HALF_N(80, D, BH, BL) PNR_HALF_N(96, D, BH, BL) PNR_HALF_N(112, D, BH, BL) PNR_HALF_N(128, D, BH, BL)
  switch (n0 >> 3) { PNR_HALF_ALL(d0, b_hi, b_lo) default: __trap(); }   // not a multiple of 16
  if (NP > 128) {
    switch ((NP - 128) >> 3) { PNR_HALF_ALL(d1, b_hi + h1, b_lo + h1) default: __trap(); }
  }
#undef PNR_HALF_ALL
#undef PNR_HALF_N
}

// ---------------------------------------------------------------- 16-bit hi/lo split
// x = hi + lo + residual, both parts rounded to nearest even in the operand format:
//   bf16 (8-bit significand):  residual <= 2^-18 |x|, fp32 exponent range (never overflows)
//   fp16 (11-bit significand): residual <= 2^-22 |x|, requires |x| < 65504
// Two values are packed per 32-bit word with the lower K index in the low half (K-major A operand).
template <int FMT>
__device__ __forceinline__ void split_x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  if (FMT == kFmtBF16) {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));  // d.hi = a, d.lo = b
    const float h0 = __uint_as_float(hi << 16);
    const float h1 = __uint_as_float(hi & 0xFFFF0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(x1 - h1), "f"(x0 - h0));
  } else {
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
  }
}

}  // namespace pnr
