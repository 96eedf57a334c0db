// linear_wgmma.cu — y = act(x W^T + b) for the layers AFTER the trunk on the training path (SURVEY.md 8(f) rank 2):
// alpha / feature / view / rgb / the two heads, forward and input gradient (dL/dx = g W, i.e. the same product
// with the transposed matrix), on sm_90a tensor cores with the same 3-product operand split as the fused MLP
// kernel.  (The render path never comes here: there these layers are steps of the fused kernel's program.  On the
// training path they are differentiated one by one by autograd, so each is a GEMM of its own.)
//
//   y[s, n] = act( sum_k x[s, k] W[n, k] + b[n] ),   s < S (10^5 .. 10^7 samples),  K <= 512,  N <= 256
//
// Persistent, one CTA per SM, tiles of 128 samples; per 64-feature K chunk:
//   * each of the two consumer warpgroups reads its 64 rows of the chunk (16 lanes per 256-byte row segment), scales
//     them (a power of two for gradients, exact), splits them into 16-bit hi / lo parts and writes them as half
//     core-matrix rows of the no-swizzle K-major A operand (2 slots, so a chunk is written while the previous one's
//     MMAs run);
//   * one warp streams the matching K chunk of the weights - packed once per call by linear_pack_kernel into hi / lo
//     images of [8 K-cores][NP rows][16 B] - with cp.async.bulk into a 2-stage ring (L2-resident source);
//   * the warpgroup issues wgmma m64nNk16 (N = NP in halves of <= 128), hi.hi + lo.hi + hi.lo, accumulators in
//     registers; after the tile's last chunk: * 1/scale, + bias, optional ReLU, stores to the samples' rows of y.
// HBM-bound by construction for the shapes of this network (4 (K + N) bytes per sample against 6 K N tensor flops).
#include <cstddef>
#include "common.cuh"
#include "sm90.cuh"

namespace pnr {

constexpr int kLnConsumers = 256;                        // two warpgroups, 64 rows each
constexpr int kLnThreads = kLnConsumers + 32;            // + weight stream warp
constexpr int kLnTile = 128;
constexpr int kLnChunk = 64;                             // K per stage
constexpr int kLnALbo = kLnTile * 16;                    // distance of K-adjacent core matrices in the A images
constexpr int kLnAPart = 8 * kLnALbo;                    // one 16-bit image of the A chunk (16 KB)
constexpr int kLnAStage = 2 * kLnAPart;                  // hi + lo
constexpr int kLnBStageMax = 2 * 8 * 256 * 16;           // hi + lo images of a [64 K][256 rows] weight chunk: 64 KB
constexpr int kLnRing = 2;
constexpr int kLnSmemA = 0;
constexpr int kLnSmemB = kLnRing * kLnAStage;            // 64 KB
constexpr int kLnSmemBars = kLnSmemB + kLnRing * kLnBStageMax;   // 192 KB
constexpr int kLnSmemTotal = kLnSmemBars + 256;

struct LinearParams {
  const float* x; int64_t ld_x; int K;
  const uint8_t* wpk;     // packed weights: per 64-wide K chunk, hi image then lo image of [8][NP][16 B]
  const float* bias;      // [N] or NULL
  float* y; int64_t ld_y; int N;
  int64_t S;
  int NP, n_chunks, relu, vec_in;
  const float* in_scale;  // device scalar (power of two) applied to x; the result is divided by it.  NULL: 1
};

// W [N, K] (row stride ld_w; `trans`: the matrix is given as [K, N] and read transposed) -> packed 16-bit images.
// One thread per (chunk, K-core, row): 8 consecutive K values of one row = one 16-byte core-matrix row.
template <int FMT>
__global__ void linear_pack_kernel(const float* __restrict__ W, int64_t ld_w, int N, int K, int NP, int n_chunks, int trans,
                                   uint8_t* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_chunks * 8 * NP) return;
  const int row = idx % NP, kc = (idx / NP) % 8, c = idx / (8 * NP);
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = c * kLnChunk + kc * 8 + j;
    v[j] = (row < N && k < K) ? (trans ? W[(int64_t)k * ld_w + row] : W[(int64_t)row * ld_w + k]) : 0.f;
  }
  uint32_t h[4], l[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) split_x2<FMT>(v[2 * q], v[2 * q + 1], h[q], l[q]);
  uint8_t* img = out + (size_t)c * (2 * 8 * NP * 16) + (size_t)(kc * NP + row) * 16;
  *reinterpret_cast<uint4*>(img) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(img + 8 * NP * 16) = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int FMT>
__global__ void __launch_bounds__(kLnThreads, 1) linear_kernel(const LinearParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kLnSmemBars);
  const uint32_t bar_b_full = smem_u32(&bars[0]);      // [2] weight chunk landed (complete_tx)
  const uint32_t bar_b_empty = smem_u32(&bars[2]);     // [2] its MMAs retired (one arrival per consumer warp)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n_tiles = (p.S + kLnTile - 1) / kLnTile;
  const int n_iter = (int)((n_tiles - (int64_t)blockIdx.x + (int64_t)gridDim.x - 1) / (int64_t)gridDim.x);   // >= 1
  const int n_chunks = p.n_chunks;
  const uint32_t b_stage_bytes = (uint32_t)(2 * 8 * p.NP * 16);
  if (threadIdx.x == 0) {
    for (int s = 0; s < kLnRing; ++s) {
      mbar_init(bar_b_full + 8 * s, 1);
      mbar_init(bar_b_empty + 8 * s, kLnConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kLnConsumers / 32) {
    // =============================================================== weight stream (one elected thread)
    if (elect_one()) {
      uint32_t gb = 0;
      for (int it = 0; it < n_iter; ++it) {
        for (int c = 0; c < n_chunks; ++c, ++gb) {
          const uint32_t slot = gb & 1u, ph = (gb >> 1) & 1u;
          mbar_wait_backoff(bar_b_empty + 8 * slot, ph ^ 1u);
          mbar_arrive_expect_tx(bar_b_full + 8 * slot, b_stage_bytes);
          bulk_g2s(smem_u32(smem + kLnSmemB + slot * kLnBStageMax), p.wpk + (size_t)c * b_stage_bytes, b_stage_bytes,
                   bar_b_full + 8 * slot);
        }
      }
    }
  } else {
    // =============================================================== consumer warpgroups
    const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
    const int seg = t & 15, kc = seg >> 1, half = seg & 1;   // 16-byte segment of a row's 256-byte chunk
    const float sc = p.in_scale != nullptr ? __ldg(p.in_scale) : 1.0f;
    const float inv = 1.0f / sc;
    const uint32_t b_lbo = (uint32_t)p.NP * 16u, b_part = 8u * (uint32_t)p.NP * 16u;
    float acc0[64], acc1[64];
    uint32_t g = 0;   // chunk counter (ring position)
    for (int it = 0; it < n_iter; ++it) {
      const int64_t tile0 = ((int64_t)blockIdx.x + (int64_t)it * gridDim.x) * kLnTile + wg * 64;   // first row of this warpgroup
#pragma unroll 1
      for (int c = 0; c < n_chunks; ++c, ++g) {
        const uint32_t slot = g & 1u, ph = (g >> 1) & 1u;
        // ---- this thread's 16-byte segment of 8 rows (8 apart) -> hi / lo half core-matrix rows
        const int k = c * kLnChunk + seg * 4;
        float4 v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int64_t s = tile0 + (t >> 4) + 8 * i;
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (s < p.S) {
            const float* q = p.x + s * p.ld_x + k;
            if (p.vec_in && k + 4 <= p.K) {
              v[i] = __ldg(reinterpret_cast<const float4*>(q));
            } else {
              if (k < p.K) v[i].x = __ldg(q);
              if (k + 1 < p.K) v[i].y = __ldg(q + 1);
              if (k + 2 < p.K) v[i].z = __ldg(q + 2);
              if (k + 3 < p.K) v[i].w = __ldg(q + 3);
            }
          }
        }
        uint8_t* img = smem + kLnSmemA + slot * kLnAStage + kc * kLnALbo + (wg * 64 + (t >> 4)) * 16 + half * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          uint32_t h0, l0, h1, l1;
          split_x2<FMT>(v[i].x * sc, v[i].y * sc, h0, l0);
          split_x2<FMT>(v[i].z * sc, v[i].w * sc, h1, l1);
          *reinterpret_cast<uint2*>(img + i * 128) = make_uint2(h0, h1);
          *reinterpret_cast<uint2*>(img + i * 128 + kLnAPart) = make_uint2(l0, l1);
        }
        fence_proxy_async_smem();
        named_bar_sync(1 + wg, 128);   // this warpgroup's rows of the chunk are written
        mbar_wait(bar_b_full + 8 * slot, ph);
        const uint32_t sa = smem_u32(smem + kLnSmemA + slot * kLnAStage) + (uint32_t)(wg * 64 * 16);
        const uint32_t sb = smem_u32(smem + kLnSmemB + slot * kLnBStageMax);
        const int kleft = p.K - c * kLnChunk;
        const int ksteps = kleft >= kLnChunk ? kLnChunk / 16 : (kleft + 15) / 16;
        mma_run_halves<FMT>(acc0, acc1, p.NP, make_smem_desc_noswz(sa, kLnALbo, 128),
                            make_smem_desc_noswz(sa + kLnAPart, kLnALbo, 128), make_smem_desc_noswz(sb, b_lbo, 128),
                            make_smem_desc_noswz(sb + b_part, b_lbo, 128), ksteps, (2u * kLnALbo) >> 4, (2u * b_lbo) >> 4,
                            c == 0 ? 0u : 1u);
        wgmma_commit();
        wgmma_wait<1>();   // the previous chunk's MMAs have retired: its weight slot is free (its A slot is rewritten next)
        if (g > 0 && lane == 0) mbar_arrive(bar_b_empty + 8 * ((g - 1) & 1u));
      }
      wgmma_wait<0>();
      // ---- epilogue: fragment rows 16 w + lane/4 (+8), columns 8 j + 2 (lane % 4) (+1)
      const int wl = (threadIdx.x >> 5) & 3;
      const int64_t r0 = tile0 + wl * 16 + (lane >> 2);
      auto out = [&](const float (&d)[64], int cbase, int nh) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = cbase + 8 * j + 2 * (lane & 3);
          if (8 * j < nh) {
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const int64_t s = r0 + 8 * hr;
              if (s < p.S) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  if (col + e < p.N) {
                    const float tv = d[4 * j + 2 * hr + e] * inv + (p.bias != nullptr ? __ldg(p.bias + col + e) : 0.f);
                    p.y[s * p.ld_y + col + e] = p.relu && !(tv != tv) ? fmaxf(tv, 0.f) : tv;   // NaN stays NaN (as torch.relu)
                  }
                }
              }
            }
          }
        }
      };
      out(acc0, 0, p.NP < 128 ? p.NP : 128);
      if (p.NP > 128) out(acc1, 128, p.NP - 128);
    }
    if (g > 0 && lane == 0) mbar_arrive(bar_b_empty + 8 * ((g - 1) & 1u));
  }
}

template <int FMT>
static int linear_launch(const LinearParams& p, const float* W, int64_t ld_w, int trans, uint8_t* wpk, int dev, cudaStream_t st) {
  const int rc = opt_in_smem((const void*)linear_kernel<FMT>, kLnSmemTotal, dev);
  if (rc != PNR_OK) return rc;
  const int n_pack = p.n_chunks * 8 * p.NP;
  linear_pack_kernel<FMT><<<(n_pack + 127) / 128, 128, 0, st>>>(W, ld_w, p.N, p.K, p.NP, p.n_chunks, trans, wpk);
  PNR_LAUNCH_CHECK("linear_pack_kernel");
  const int64_t n_tiles = (p.S + kLnTile - 1) / kLnTile;
  const int sms = num_sms(dev);
  const int grid = (int)(n_tiles < sms ? n_tiles : sms);
  if (grid > 0) {
    linear_kernel<FMT><<<grid, kLnThreads, kLnSmemTotal, st>>>(p);
    PNR_LAUNCH_CHECK("linear_kernel");
  }
  return PNR_OK;
}

}  // namespace pnr

using namespace pnr;

extern "C" size_t pnr_linear_workspace_bytes(int32_t N, int32_t K) {
  if (N <= 0 || K <= 0 || N > 256 || K > 512) return 0;
  const int NP = (N + 15) / 16 * 16, n_chunks = (K + kLnChunk - 1) / kLnChunk;
  return (size_t)n_chunks * 2 * 8 * NP * 16;
}

extern "C" int pnr_linear(const float* x, int64_t ld_x, int32_t K, const float* W, int64_t ld_w, int32_t transposed,
                          const float* bias, int32_t N, int64_t S, int32_t relu, int32_t precision, const float* in_scale,
                          float* y, int64_t ld_y, void* workspace, size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(x != nullptr && W != nullptr && y != nullptr, "pnr_linear: x, W and y are required");
  PNR_CHECK_ARG(N >= 1 && N <= 256 && K >= 1 && K <= 512, "pnr_linear: N = %d must be in [1, 256], K = %d in [1, 512]", N, K);
  PNR_CHECK_ARG(ld_x >= K, "pnr_linear: leading dimensions: ld_x = %lld < K = %d", (long long)ld_x, K);
  PNR_CHECK_ARG(ld_y >= N, "pnr_linear: leading dimensions: ld_y = %lld < N = %d", (long long)ld_y, N);
  PNR_CHECK_ARG(ld_w >= (transposed ? N : K), "pnr_linear: leading dimensions: ld_w = %lld < %s = %d", (long long)ld_w,
                transposed ? "N" : "K", transposed ? N : K);
  PNR_CHECK_ARG(S >= 0, "pnr_linear: S = %lld", (long long)S);
  PNR_CHECK_ARG(precision == PNR_PREC_BF16X3 || precision == PNR_PREC_FP16X3, "pnr_linear: x3 precisions only (got %d)", precision);
  const size_t need = pnr_linear_workspace_bytes(N, K);
  PNR_CHECK_ARG(workspace != nullptr && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0,
                "pnr_linear: workspace of %zu bytes (16-byte aligned), %zu needed (pnr_linear_workspace_bytes)", workspace_bytes, need);
  if (S == 0) return PNR_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int dev = 0;
  const int rc = current_device("pnr_linear", &dev);
  if (rc != PNR_OK) return rc;
  LinearParams p;
  p.x = x; p.ld_x = ld_x; p.K = K;
  p.wpk = static_cast<const uint8_t*>(workspace);
  p.bias = bias;
  p.y = y; p.ld_y = ld_y; p.N = N;
  p.S = S;
  p.NP = (N + 15) / 16 * 16;
  p.n_chunks = (K + kLnChunk - 1) / kLnChunk;
  p.relu = relu != 0;
  p.vec_in = (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (ld_x & 3) == 0 && ld_x >= (K + 3) / 4 * 4;
  p.in_scale = in_scale;
  uint8_t* wpk = static_cast<uint8_t*>(workspace);
  return precision == PNR_PREC_FP16X3 ? linear_launch<kFmtF16>(p, W, ld_w, transposed != 0, wpk, dev, st)
                                      : linear_launch<kFmtBF16>(p, W, ld_w, transposed != 0, wpk, dev, st);
}
