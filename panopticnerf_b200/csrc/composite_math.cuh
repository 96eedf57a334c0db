// composite_math.cuh — the per-sample arithmetic of alpha compositing (SURVEY.md 8(a) a9), shared by the standalone
// compositing kernel and its backward (stream_kernels.cu) and the compositing epilogue of the fused MLP kernel
// (mlp_wgmma.cu), so that all three produce the same per-sample weights bit for bit (the fine sampler consumes them,
// the backward differentiates them).
//
// A ray's samples are handled in aligned groups of 32 (one warp, lane = sample index mod 32):
//   alpha_i = 1 - exp(-relu(sigma_i) * dist_i),   t_i = 1 - alpha_i + 1e-10,
//   T_i = carry * prod_{j<i in group} t_j   (shuffle ladder, exclusive),   w_i = alpha_i * T_i,
//   carry <- carry * prod_{group} t   (groups of one ray in order: the product order is fixed by the sample index).
#pragma once
#include <cuda_runtime.h>

namespace pnr {

__device__ __forceinline__ float comp_dnorm(float dx, float dy, float dz) {
  return sqrtf(dx * dx + dy * dy + dz * dz);
}

// dist_i * |d| for sample i of N (the last sample's distance is 1e10)
__device__ __forceinline__ float comp_dist(float zi, float z_next, bool has_next, float dnorm) {
  return (has_next ? (z_next - zi) : 1e10f) * dnorm;
}

__device__ __forceinline__ float comp_alpha(float sigma_raw, float dist, bool masked) {
  float sig = fmaxf(sigma_raw, 0.f);
  if (masked) sig = 0.f;
  return 1.0f - expf(-sig * dist);
}

__device__ __forceinline__ float comp_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// Exclusive product scan of t over the 32 lanes of a warp.  Returns the exclusive prefix of this lane; `total`
// receives the product over all 32 lanes (the same value in every lane).
__device__ __forceinline__ float comp_scan32(float t, int lane, float* total) {
  float incl = t;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float o = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl *= o;
  }
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) excl = 1.0f;
  *total = __shfl_sync(0xffffffffu, incl, 31);
  return excl;
}

__device__ __forceinline__ float comp_disp(float depth, float acc) {
  const float q = depth / acc;  // NaN when acc == 0, as in the oracle
  return 1.0f / ((q != q) ? q : fmaxf(1e-10f, q));
}

}  // namespace pnr
