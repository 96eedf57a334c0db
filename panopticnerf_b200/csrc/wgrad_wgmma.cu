// wgrad_wgmma.cu — weight-gradient GEMM of the MLP backward (SURVEY.md 8(f) rank 2) on sm_90a tensor cores.
//
//   dW[o, i] = sum_s dZ[s, o] * X[s, i]        db[o] = sum_s dZ[s, o]        (s over S samples, S ~ 10^5 .. 10^7)
//
// dZ [S, No] and X [S, Ni] are the fp32 operands the fused backward kernel stashes (mlp_wgmma.cu, BWD programs) or
// the inputs / output gradients of the layers after the trunk; No, Ni <= 256.  The reduction runs over the SAMPLES,
// so this is a split-K GEMM with a tiny output.  A CTA owns 128 output rows (blockIdx.y: which 128) and every
// gridDim.x-th slab of 64 samples; its two warpgroups accumulate 64 rows x NP columns each in registers (two wgmma
// halves of <= 128 columns) over runs of kWgFlush slabs and add each run to the CTA's partial product in global
// memory; a second kernel adds the partials in CTA order (deterministic).  Per slab:
//   * the 256 consumer threads read the slab: a work item is 4 consecutive features of 8 consecutive samples (8
//     16-byte loads), split into 16-bit hi / lo parts and written as four 16-byte rows of the no-swizzle K-major
//     images (K = samples): a thread's 8 samples of one feature ARE one core-matrix row, so the transposition
//     dZ -> dZ^T costs nothing.  Two slots: a slab is written while the previous one's MMAs run;
//   * wgmma m64nNk16, both operands from shared memory: A = dZ^T (64 output features per warpgroup x K = 16 samples),
//     B = X^T (N = Ni padded to 16), three products per K step: hi.hi + lo.hi + hi.lo.  bf16 parts: ~2^-17 per product,
//     fp32 exponent range, gradients need no scaling.  fp16 parts: ~2^-21 per product; dZ is multiplied by a
//     caller-supplied power of two on load (a device scalar, exact) so that the parts of ~1e-6 gradients stay normal,
//     and the sums are divided by it at the end.
// The kernel is HBM-bound: 4 (No + Ni) bytes per sample against 6 No Ni tensor flops; X is read once per block of
// 128 output rows.
#include <cstddef>
#include "common.cuh"
#include "sm90.cuh"

namespace pnr {

constexpr int kWgConsumers = 256;
constexpr int kWgThreads = kWgConsumers;
constexpr int kWgSlab = 64;                         // samples per stage
constexpr int kWgRows = 256;                        // features of an operand, at most
constexpr int kWgALbo = 128 * 16;                   // A images: [8 K-cores][128 rows][16 B]
constexpr int kWgAPart = (kWgSlab / 8) * kWgALbo;   // 16 KB
constexpr int kWgBLbo = kWgRows * 16;               // B images: [8 K-cores][256 rows][16 B]
constexpr int kWgBPart = (kWgSlab / 8) * kWgBLbo;   // 32 KB
constexpr int kWgStage = 2 * kWgAPart + 2 * kWgBPart;   // A hi, A lo, B hi, B lo: 96 KB
constexpr int kWgRing = 2;
// Slabs per run of the register accumulators.  The tensor cores' fp32 accumulation truncates: on all-positive operands
// (activations are >= 0, gradient columns have a mean) a run of n accumulating wgmmas loses ~0.75 n 2^-24 of the sum
// (measured on an H100), so one run over a CTA's whole share of the samples lost 5e-5 of the sum at S = 393 216
// (256 x 256) and 8e-4 at S = 2^23.  Every kWgFlush slabs the run is added to the CTA's partial product in global
// memory (round to nearest) and restarted, which bounds the drift at ~8e-6 of the sum whatever S is.  Each flush
// costs a pipeline drain and a read-modify-write of the partial: pnr_wgrad takes ~20 % longer at 393 216 x 256 x 256.
constexpr int kWgFlush = 16;
constexpr int kWgSmemDb = kWgRing * kWgStage;       // [8 sample groups][128] partial bias sums
constexpr int kWgSmemTotal = kWgSmemDb + 8 * 128 * 4;

struct WgradParams {
  const float* dz; int64_t ld_dz; int No;
  const float* x; int64_t ld_x; int Ni;
  int64_t S;
  int vec_a, vec_b;   // 16-byte loads possible (base and row stride 16-byte aligned)
  int mh;        // blocks of 128 output features (gridDim.y)
  int NP;        // Ni padded to a multiple of 16
  float* part;   // [gridDim.x][mh * 128][NP]
  float* dbp;    // [gridDim.x][256] or NULL
  const float* a_scale;   // device scalar (power of two) applied to dZ on load; NULL: 1
};

template <int FMT>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  float* dbs = reinterpret_cast<float*>(smem + kWgSmemDb);
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, lane = threadIdx.x & 31;
  const int ob = blockIdx.y;                                  // output rows [128 ob, 128 ob + 128)
  const int64_t n_slabs = (p.S + kWgSlab - 1) / kWgSlab;
  const int n_mine = (int)((n_slabs - (int64_t)blockIdx.x + (int64_t)gridDim.x - 1) / (int64_t)gridDim.x);   // >= 1: grid <= n_slabs
  const float sc = p.a_scale != nullptr ? __ldg(p.a_scale) : 1.0f;
  const int n_bq = p.NP / 4;                                  // B items per sample group: feature quads of X
  const int n_items = 32 * 8 + n_bq * 8;                      // A: 32 quads x 8 sample groups; B: n_bq quads x 8
  float db[4] = {0.f, 0.f, 0.f, 0.f};                         // item 0 of every thread is an A item: its bias sums
  float acc0[64], acc1[64];
  const uint32_t b_lbo = kWgBLbo;
  // accumulators -> this CTA's partial product (fragment rows 16 w + lane/4 (+8), columns 8 j + 2 (lane % 4)): stored by
  // the first flush, added to by the later ones (fp32, round to nearest; each element has one reader and writer, this
  // thread: no atomics, deterministic)
  const int o0 = ob * 128 + wg * 64 + ((t >> 5) * 16) + (lane >> 2);
  auto out = [&](const float (&d)[64], int cbase, int nh, bool add) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (8 * j < nh) {
        const int col = cbase + 8 * j + 2 * (lane & 3);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float2* dst = reinterpret_cast<float2*>(p.part + ((int64_t)blockIdx.x * (p.mh * 128) + o0 + 8 * hr) * p.NP + col);
          float2 v = make_float2(d[4 * j + 2 * hr], d[4 * j + 2 * hr + 1]);
          if (add) {
            const float2 o = *dst;
            v = make_float2(o.x + v.x, o.y + v.y);
          }
          *dst = v;
        }
      }
    }
  };
#pragma unroll 1
  for (int i = 0; i < n_mine; ++i) {
    const int slot = i & 1;
    uint8_t* stage = smem + slot * kWgStage;
    const int64_t s0 = ((int64_t)blockIdx.x + (int64_t)i * gridDim.x) * kWgSlab;
    // ---- convert the slab (slot i & 1 was last read by slab i - 2, whose MMAs have retired)
#pragma unroll 1
    for (int item = threadIdx.x; item < n_items; item += kWgThreads) {
      const bool isA = item < 256;
      const int j = isA ? item : item - 256;
      const int quad = isA ? (j & 31) : (j % n_bq), sg = isA ? (j >> 5) : (j / n_bq);
      const int f0 = isA ? ob * 128 + 4 * quad : 4 * quad;    // first feature of the operand
      const int F = isA ? p.No : p.Ni;
      const bool vec = (isA ? p.vec_a : p.vec_b) != 0;
      const int64_t ld = isA ? p.ld_dz : p.ld_x;
      const float* src = (isA ? p.dz : p.x) + (f0 < F ? f0 : 0);
      const int64_t s = s0 + sg * 8;
      const int64_t left = p.S - s;
      const int nv = f0 >= F ? 0 : (left >= 8 ? 8 : (left > 0 ? (int)left : 0));
      const int nc = F - f0;
      float4 v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < nv) {
          const float* q = src + (s + k) * ld;
          if (vec && nc >= 4) {
            v[k] = __ldg(reinterpret_cast<const float4*>(q));
          } else {
            v[k].x = __ldg(q);
            if (nc > 1) v[k].y = __ldg(q + 1);
            if (nc > 2) v[k].z = __ldg(q + 2);
            if (nc > 3) v[k].w = __ldg(q + 3);
          }
        }
      }
      const float m = isA ? sc : 1.0f;
      uint8_t* img = stage + (isA ? 0 : 2 * kWgAPart) + sg * (isA ? kWgALbo : kWgBLbo) + 4 * quad * 16;
      const int part = isA ? kWgAPart : kWgBPart;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = (c == 0 ? v[k].x : c == 1 ? v[k].y : c == 2 ? v[k].z : v[k].w);
        uint32_t h[4], l[4];
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) split_x2<FMT>(x[2 * qq] * m, x[2 * qq + 1] * m, h[qq], l[qq]);
        *reinterpret_cast<uint4*>(img + c * 16) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(img + c * 16 + part) = make_uint4(l[0], l[1], l[2], l[3]);
        if (isA) db[c] += ((x[0] + x[1]) + (x[2] + x[3])) + ((x[4] + x[5]) + (x[6] + x[7]));
      }
    }
    fence_proxy_async_smem();            // generic-proxy stores -> visible to the MMAs' async proxy
    __syncthreads();                     // (each warpgroup reads rows the other one wrote)
    // ---- this warpgroup's MMAs of the slab: A rows [64 wg, 64 wg + 64) of the block
    const uint32_t sa = smem_u32(stage) + (uint32_t)(wg * 64 * 16), sb = smem_u32(stage) + 2u * kWgAPart;
    const uint64_t a_hi = make_smem_desc_noswz(sa, kWgALbo, 128), a_lo = make_smem_desc_noswz(sa + kWgAPart, kWgALbo, 128);
    const uint64_t b_hi = make_smem_desc_noswz(sb, b_lbo, 128), b_lo = make_smem_desc_noswz(sb + kWgBPart, b_lbo, 128);
    const int n0 = p.NP < 128 ? p.NP : 128;
    const uint32_t acc = i % kWgFlush == 0 ? 0u : 1u;   // a run restarts after each flush
    mma_run_halves<FMT>(acc0, acc1, p.NP, a_hi, a_lo, b_hi, b_lo, kWgSlab / 16, (2u * kWgALbo) >> 4, (2u * kWgBLbo) >> 4, acc);
    wgmma_commit();
    wgmma_wait<1>();   // slab i - 1's MMAs have retired: its slot may be rewritten by slab i + 1
    __syncthreads();   // (by either warpgroup)
    if ((i + 1) % kWgFlush == 0 || i + 1 == n_mine) {
      wgmma_wait<0>();
      out(acc0, 0, n0, i >= kWgFlush);
      if (p.NP > 128) out(acc1, 128, p.NP - 128, i >= kWgFlush);
    }
  }
  // ---- bias partial sums: 8 sample groups per feature, added in a fixed order
  if (threadIdx.x < 256) {
    const int quad = threadIdx.x & 31, sg = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < 4; ++c) dbs[sg * 128 + 4 * quad + c] = db[c];
  }
  __syncthreads();
  if (p.dbp != nullptr && (int)threadIdx.x < 128 && ob * 128 + (int)threadIdx.x < p.No) {
    const int f = threadIdx.x;
    float sum = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) sum += dbs[g * 128 + f];
    p.dbp[(int64_t)blockIdx.x * kWgRows + ob * 128 + f] = sum;
  }
}

// dW[o, i] (+)= sum over the CTAs' partial products, in CTA order; db likewise.
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, const float* __restrict__ dbp, int G, int rows, int NP,
                                    int No, int Ni, float* __restrict__ dW, int64_t ld_w, float* __restrict__ db,
                                    int accumulate, const float* __restrict__ a_scale) {
  const float inv = a_scale != nullptr ? 1.0f / __ldg(a_scale) : 1.0f;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < No * NP) {
    const int o = idx / NP, i = idx - o * NP;
    if (i < Ni) {
      const float* src = part + (int64_t)o * NP + i;
      const int64_t stride = (int64_t)rows * NP;
      float s = 0.f;
      int c = 0;
      for (; c + 4 <= G; c += 4) {
        const float v0 = src[(c + 0) * stride], v1 = src[(c + 1) * stride], v2 = src[(c + 2) * stride], v3 = src[(c + 3) * stride];
        s = (((s + v0) + v1) + v2) + v3;
      }
      for (; c < G; ++c) s += src[c * stride];
      float* d = dW + (int64_t)o * ld_w + i;
      s *= inv;
      *d = accumulate ? *d + s : s;
    }
  }
  if (db != nullptr && idx < No) {   // (G == 0: S = 0, no partials and possibly no workspace; the sum is 0)
    float s = 0.f;
    for (int c = 0; c < G; ++c) s += dbp[(int64_t)c * kWgRows + idx];
    db[idx] = accumulate ? db[idx] + s : s;
  }
}

// CTAs along the samples: one per SM over all output blocks, at most one per slab (<= num_sms: the workspace size)
static int wgrad_grid(int64_t S, int mh, int dev) {
  const int64_t n_slabs = (S + kWgSlab - 1) / kWgSlab;
  const int per = num_sms(dev) / mh > 0 ? num_sms(dev) / mh : 1;
  return (int)(n_slabs < per ? n_slabs : per);
}

}  // namespace pnr

using namespace pnr;

extern "C" size_t pnr_wgrad_workspace_bytes(int32_t No, int32_t Ni) {
  if (No <= 0 || Ni <= 0 || No > 256 || Ni > 256) return 0;
  const int mh = No > 128 ? 2 : 1, NP = (Ni + 15) / 16 * 16;
  return (size_t)num_sms() * ((size_t)mh * 128 * NP + kWgRows) * sizeof(float);
}

template <int FMT>
static int wgrad_launch(const WgradParams& p, int grid, int dev, cudaStream_t st) {
  const int rc = opt_in_smem((const void*)wgrad_kernel<FMT>, kWgSmemTotal, dev);
  if (rc != PNR_OK) return rc;
  wgrad_kernel<FMT><<<dim3(grid, p.mh), kWgThreads, kWgSmemTotal, st>>>(p);
  PNR_LAUNCH_CHECK("wgrad_kernel");
  return PNR_OK;
}

extern "C" int pnr_wgrad(const float* dz, int64_t ld_dz, int32_t No, const float* x, int64_t ld_x, int32_t Ni, int64_t S,
                         int32_t precision, const float* dz_scale, float* dW, int64_t ld_w, float* db, int32_t accumulate,
                         void* workspace, size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(precision == PNR_PREC_BF16X3 || precision == PNR_PREC_FP16X3, "pnr_wgrad: x3 precisions only (got %d)", precision);
  PNR_CHECK_ARG(dz != nullptr && x != nullptr && dW != nullptr, "pnr_wgrad: dz, x and dW are required");
  PNR_CHECK_ARG(No >= 1 && No <= 256 && Ni >= 1 && Ni <= 256, "pnr_wgrad: No = %d, Ni = %d must be in [1, 256] (split wider layers by columns)", No, Ni);
  PNR_CHECK_ARG(ld_dz >= No, "pnr_wgrad: leading dimensions: ld_dz = %lld < No = %d", (long long)ld_dz, No);
  PNR_CHECK_ARG(ld_x >= Ni, "pnr_wgrad: leading dimensions: ld_x = %lld < Ni = %d", (long long)ld_x, Ni);
  PNR_CHECK_ARG(ld_w >= Ni, "pnr_wgrad: leading dimensions: ld_w = %lld < Ni = %d", (long long)ld_w, Ni);
  PNR_CHECK_ARG(S >= 0, "pnr_wgrad: S = %lld", (long long)S);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int dev = 0;
  int rc = current_device("pnr_wgrad", &dev);
  if (rc != PNR_OK) return rc;
  const int mh = No > 128 ? 2 : 1, NP = (Ni + 15) / 16 * 16;
  const int grid = S > 0 ? wgrad_grid(S, mh, dev) : 0;
  const size_t need = (size_t)grid * ((size_t)mh * 128 * NP + kWgRows) * sizeof(float);
  PNR_CHECK_ARG(grid == 0 || (workspace != nullptr && workspace_bytes >= need),
                "pnr_wgrad: workspace of %zu bytes, %zu needed (pnr_wgrad_workspace_bytes)", workspace_bytes, need);
  PNR_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "pnr_wgrad: workspace must be 16-byte aligned");
  WgradParams p;
  p.dz = dz; p.ld_dz = ld_dz; p.No = No;
  p.x = x; p.ld_x = ld_x; p.Ni = Ni;
  p.S = S; p.mh = mh; p.NP = NP;
  p.part = static_cast<float*>(workspace);
  p.dbp = db != nullptr ? p.part + (size_t)grid * mh * 128 * NP : nullptr;
  p.a_scale = dz_scale;
  p.vec_a = (reinterpret_cast<uintptr_t>(dz) & 15) == 0 && (ld_dz & 3) == 0;
  p.vec_b = (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (ld_x & 3) == 0;
  if (grid > 0) {
    rc = precision == PNR_PREC_FP16X3 ? wgrad_launch<kFmtF16>(p, grid, dev, st) : wgrad_launch<kFmtBF16>(p, grid, dev, st);
    if (rc != PNR_OK) return rc;
  }
  const int n = No * NP;
  wgrad_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(p.part, p.dbp, grid, mh * 128, NP, No, Ni, dW, ld_w, db, accumulate, dz_scale);
  PNR_LAUNCH_CHECK("wgrad_reduce_kernel");
  return PNR_OK;
}
