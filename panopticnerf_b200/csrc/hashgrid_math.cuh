// hashgrid_math.cuh — the per-point arithmetic of the multi-resolution hash encoding (Mueller et al. 2022), shared by
// the standalone encoder (panoptic_kernels.cu: hashgrid_kernel / hashgrid_backward_kernel) and the hash-grid prologue
// of the fused MLP kernel (mlp_wgmma.cu), so that the features the MLP sees on chip are bit-identical to those of
// pnr_hashgrid_encode by construction.
//
// Level l has resolution res_l = floor(base * scale^l) (double, on the host).  A point in [0,1]^3 is scaled by res_l,
// its cell's 8 corners are looked up in the level's table of T = 2^T_log2 entries x F features - by the dense index
// x + y*(res+1) + z*(res+1)^2 when (res+1)^3 <= T, else by the spatial hash (x * 1) ^ (y * 2654435761) ^ (z * 805459861)
// mod T - and blended trilinearly, corners in the order x fastest.  Every operation is a separately rounded fp32 op.
#pragma once
#include <math.h>
#include <stdint.h>

namespace pnr {

constexpr int kHashMaxLevels = 32;

// Byte alignment the table needs: a corner's F = 2 / 4 features are read as one float2 / float4
inline bool hash_table_aligned(const float* table, int F) {
  const uintptr_t a = F == 4 ? 16 : F == 2 ? 8 : 4;
  return (reinterpret_cast<uintptr_t>(table) & (a - 1)) == 0;
}

// res_l = floor(base * scale^l), evaluated in double
inline void hash_level_resolutions(int L, float base, float scale, uint32_t* res) {
  for (int l = 0; l < L; ++l) res[l] = (uint32_t)floor((double)base * pow((double)scale, (double)l));
}

__device__ __forceinline__ uint32_t hash_index(uint32_t x, uint32_t y, uint32_t z, uint32_t res1, bool dense, uint32_t mask) {
  if (dense) return x + y * res1 + z * res1 * res1;
  return (x ^ (y * 2654435761u) ^ (z * 805459861u)) & mask;
}

// x -> [0,1]^3 through aabb {lo.xyz, hi.xyz} (null: x is already normalised), clamped: outside points take the border cell
__device__ __forceinline__ void hash_normalize(const float (&x)[3], const float* aabb, float (&v)[3]) {
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    float t = x[d];
    if (aabb) t = __fdiv_rn(__fsub_rn(t, aabb[d]), __fsub_rn(aabb[3 + d], aabb[d]));
    v[d] = fminf(fmaxf(t, 0.0f), 1.0f);
  }
}

// The cell of v at resolution res: lower corner c and the fractional position w inside it.
__device__ __forceinline__ void hash_cell(const float (&v)[3], uint32_t res, uint32_t (&c)[3], float (&w)[3]) {
  const float res_f = (float)res;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float p = __fmul_rn(v[d], res_f);
    float fl = floorf(p);
    if (fl >= res_f) fl = res_f - 1.0f;                // v == 1 belongs to the last cell (weight 1 on its far corner)
    c[d] = (uint32_t)fl;
    w[d] = __fsub_rn(p, fl);
  }
}

// Trilinear weight of corner k (dx = k & 1, dy = k >> 1 & 1, dz = k >> 2) and its table row.
__device__ __forceinline__ float hash_corner(const uint32_t (&c)[3], const float (&w)[3], int k, uint32_t res1, bool dense,
                                             uint32_t mask, uint32_t& idx) {
  const uint32_t dx = k & 1, dy = (k >> 1) & 1, dz = k >> 2;
  const float wx = dx ? w[0] : __fsub_rn(1.0f, w[0]);
  const float wy = dy ? w[1] : __fsub_rn(1.0f, w[1]);
  const float wz = dz ? w[2] : __fsub_rn(1.0f, w[2]);
  idx = hash_index(c[0] + dx, c[1] + dy, c[2] + dz, res1, dense, mask);
  return __fmul_rn(__fmul_rn(wx, wy), wz);
}

// The F features of one level at v, ADDED to acc[0..F) (the caller starts from zeros): tab = the level's table
// [T, F], sum over the corners in order.
template <int F>
__device__ __forceinline__ void hash_level_blend(const float* __restrict__ tab, const float (&v)[3], uint32_t res,
                                                 uint32_t T_log2, float* acc) {
  const uint32_t T = 1u << T_log2, mask = T - 1u, res1 = res + 1u;
  const bool dense = (uint64_t)res1 * res1 * res1 <= (uint64_t)T;
  float w[3];
  uint32_t c[3];
  hash_cell(v, res, c, w);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    uint32_t idx;
    const float wk = hash_corner(c, w, k, res1, dense, mask, idx);
    if (F == 2) {
      const float2 t = __ldg(reinterpret_cast<const float2*>(tab) + idx);
      acc[0] = __fadd_rn(acc[0], __fmul_rn(wk, t.x));
      acc[1] = __fadd_rn(acc[1], __fmul_rn(wk, t.y));
    } else if (F == 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(tab) + idx);
      acc[0] = __fadd_rn(acc[0], __fmul_rn(wk, t.x));
      acc[1] = __fadd_rn(acc[1], __fmul_rn(wk, t.y));
      acc[2] = __fadd_rn(acc[2], __fmul_rn(wk, t.z));
      acc[3] = __fadd_rn(acc[3], __fmul_rn(wk, t.w));
    } else {
#pragma unroll
      for (int f = 0; f < F; ++f) acc[f] = __fadd_rn(acc[f], __fmul_rn(wk, __ldg(tab + (size_t)idx * F + f)));
    }
  }
}

}  // namespace pnr
