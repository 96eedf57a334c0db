// panoptic_kernels.cu — SURVEY 8(f) rank 4: what follows / feeds the render path in the 360 model.
//   * panoptic label fusion + colour mapping of the composited maps (per ray; one warp per ray),
//   * the multi-resolution hash-grid feature encoder (per point and level; gather-bound, L2 / HBM).
// The reference's versions are not in the mount: both rules are stated here and in oracle/reference_panoptic.py
// ("chosen, unverified"), and the kernels are held to that oracle.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <algorithm>
#include "../../include/pnr.h"
#include "common.cuh"
#include "hashgrid_math.cuh"

namespace pnr {
namespace {

// argmax over the channels c < n with keep(c); lanes stride the channels; NaN counts as -inf; ties -> lowest index;
// -1 when no channel is kept
template <class Keep>
__device__ __forceinline__ int warp_argmax_if(const float* __restrict__ v, int n, int lane, Keep keep) {
  float best = -INFINITY;
  int arg = 0x7fffffff;
  for (int c = lane; c < n; c += 32) {
    if (!keep(c)) continue;
    float x = v[c];
    if (x != x) x = -INFINITY;
    if (x > best || arg == 0x7fffffff) { best = x; arg = c; }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, d);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, d);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  return arg == 0x7fffffff ? -1 : arg;
}

struct FuseArgs {
  const float* sem; const float* inst; int64_t R; int C, K;
  const uint8_t* is_thing;      // [C] 1 = the class has instances
  const int32_t* inst_class;    // [K] class channel of instance slot k
  const int32_t* inst_id;       // [K] global instance id of slot k (KITTI-360: semanticId*1000 + n), or null
  const int32_t* class_id;      // [C] dataset id of class channel c (stuff id = class_id*1000), or null: the channel
  const uint8_t* palette;       // [C,3] u8 colours, or null
  int32_t* panoptic; int16_t* sem_label; int16_t* inst_slot; uint8_t* color;
};

// Fusion rule: s = argmax of the semantic map.  A stuff class gives id(s)*1000.  A thing class takes the best
// instance slot AMONG THE SLOTS OF THAT CLASS (the instance head cannot contradict the semantic head); without such
// a slot the pixel falls back to id(s)*1000.  Colour: the class colour, for instances averaged with a colour hashed
// from the instance id (Knuth multiplicative hash, one byte per channel).
__global__ void __launch_bounds__(256) panoptic_fuse_kernel(FuseArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= a.R) return;
  const int s = warp_argmax_if(a.sem + r * a.C, a.C, lane, [](int) { return true; });
  int k = -1;
  if (s >= 0 && a.K > 0 && a.inst != nullptr && a.is_thing != nullptr && a.is_thing[s])
    k = warp_argmax_if(a.inst + r * a.K, a.K, lane, [&](int c) { return a.inst_class[c] == s; });
  if (lane != 0) return;
  const int cid = s < 0 ? -1 : (a.class_id ? a.class_id[s] : s);
  const int pan = s < 0 ? -1 : (k >= 0 ? (a.inst_id ? a.inst_id[k] : cid * 1000 + k + 1) : cid * 1000);
  if (a.panoptic) a.panoptic[r] = pan;
  if (a.sem_label) a.sem_label[r] = (int16_t)s;
  if (a.inst_slot) a.inst_slot[r] = (int16_t)k;
  if (a.color) {
    uint32_t c0 = 0, c1 = 0, c2 = 0;
    if (s >= 0 && a.palette) { c0 = a.palette[s * 3]; c1 = a.palette[s * 3 + 1]; c2 = a.palette[s * 3 + 2]; }
    if (k >= 0) {
      const uint32_t h = (uint32_t)pan * 2654435761u;
      c0 = (c0 + ((h >> 8) & 0xFFu) + 1u) >> 1;
      c1 = (c1 + ((h >> 16) & 0xFFu) + 1u) >> 1;
      c2 = (c2 + ((h >> 24) & 0xFFu) + 1u) >> 1;
    }
    a.color[r * 3] = (uint8_t)c0; a.color[r * 3 + 1] = (uint8_t)c1; a.color[r * 3 + 2] = (uint8_t)c2;
  }
}

// ------------------------------------------------------------------------------------------------ hash grid
// Multi-resolution hash encoding (Mueller et al. 2022, the published algorithm): level l has resolution
// res_l = floor(base * scale^l); a point x in [0,1]^3 is scaled by res_l, its cell's 8 corners are looked up in a
// table of T entries x F features - by the dense index x + y*(res+1) + z*(res+1)^2 when (res+1)^3 <= T, else by
// the spatial hash (x * 1) ^ (y * 2654435761) ^ (z * 805459861) mod T - and blended trilinearly.
// out[n, L*F], level-major.  blockIdx.y = a group of consecutive levels, so a block's gathers stay inside a few
// levels' tables (the coarse levels live in L1/L2, the fine ones stream from HBM at one 32-byte sector per corner).
struct HashArgs {
  const float* x; int64_t n; const float* table; float* out;
  const float* aabb;   // device {lo.xyz, hi.xyz} or null (x already in [0,1]^3)
  int L, F, T_log2;
  uint32_t res[kHashMaxLevels];   // resolution of every level (hash_level_resolutions)
};

// One thread = one point x LPT consecutive levels with LPT * F = 8 features: its output is one whole 32-byte sector
// (a thread per (point, level) writes 8 bytes into every 128-byte row - four partial writes per sector from four
// different blocks, which the memory system turns into read-modify-writes: measured 4x the algorithmic write traffic
// plus as much again in sector fills, profiles/r02_hashgrid_fuse_ncu.txt, first capture).
template <int F>
__global__ void __launch_bounds__(256) hashgrid_kernel(HashArgs a) {
  constexpr int LPT = 8 / F;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int l0 = blockIdx.y * LPT;
  if (i >= a.n) return;
  const uint32_t T = 1u << a.T_log2;
  float v[3];
  const float x[3] = {a.x[i * 3], a.x[i * 3 + 1], a.x[i * 3 + 2]};
  hash_normalize(x, a.aabb, v);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
  for (int ll = 0; ll < LPT; ++ll) {
    const int l = l0 + ll;
    if (l >= a.L) break;
    hash_level_blend<F>(a.table + (size_t)l * T * F, v, a.res[l], (uint32_t)a.T_log2, acc + ll * F);
  }
  const int width = a.L * F;
  float* o = a.out + i * (int64_t)width + l0 * F;
  const int n_out = min(8, width - l0 * F);
  if (n_out == 8 && (width & 7) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 31) == 0) {
    reinterpret_cast<float4*>(o)[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    reinterpret_cast<float4*>(o)[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < n_out) o[j] = acc[j];
  }
}

// Gradient of the encoder w.r.t. its table: dL/dtable[l, idx, f] += w_corner * dL/dout[i, l*F + f] over the 8 corners
// of every point's cell - the same thread layout and index arithmetic as the forward kernel, scatter instead of gather
// (fp32 atomic adds at L2; colliding points are what a hash table is for, so the summation order - and the last bits -
// vary from run to run, as in every hash-grid trainer).  grad_table is ACCUMULATED into (zero it first).
template <int F>
__global__ void __launch_bounds__(256) hashgrid_backward_kernel(HashArgs a, const float* __restrict__ gout, float* gtab) {
  constexpr int LPT = 8 / F;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int l0 = blockIdx.y * LPT;
  if (i >= a.n) return;
  const uint32_t T = 1u << a.T_log2, mask = T - 1u;
  float v[3];
  const float x[3] = {a.x[i * 3], a.x[i * 3 + 1], a.x[i * 3 + 2]};
  hash_normalize(x, a.aabb, v);
  const float* go = gout + i * (int64_t)(a.L * F);
#pragma unroll
  for (int ll = 0; ll < LPT; ++ll) {
    const int l = l0 + ll;
    if (l >= a.L) break;
    const uint32_t res = a.res[l], res1 = res + 1u;
    const bool dense = (uint64_t)res1 * res1 * res1 <= (uint64_t)T;
    float w[3], g[F];
    uint32_t c[3];
#pragma unroll
    for (int f = 0; f < F; ++f) g[f] = go[l * F + f];
    hash_cell(v, res, c, w);
    float* tab = gtab + (size_t)l * T * F;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      uint32_t idx;
      const float wk = hash_corner(c, w, k, res1, dense, mask, idx);
      if (F == 2) {
        atomicAdd(reinterpret_cast<float2*>(tab) + idx, make_float2(wk * g[0], wk * g[1]));
      } else if (F == 4) {
        atomicAdd(reinterpret_cast<float4*>(tab) + idx, make_float4(wk * g[0], wk * g[1], wk * g[2], wk * g[3]));
      } else {
#pragma unroll
        for (int f = 0; f < F; ++f) atomicAdd(tab + (size_t)idx * F + f, wk * g[f]);
      }
    }
  }
}

// ---------------------------------------------------------------------------- hash grid, fixed-point table gradient
// pnr_hashgrid_backward_fixed (rule: include/pnr.h).  Every contribution w_k * g is rounded once to an int64 at the
// level's power-of-two scale 2^s_l and summed with integer atomics, which are associative: the result does not depend
// on the order of the points, the launch or the GPU.  Three kernels: the level maxima (and s_l), the scatter, and the
// finalize that turns the integer sums into fp32 and adds them to grad_table.
//
// Warp combining in the scatter: the lanes of a warp whose corner falls in the same row sum their integers first
// (one atomic per distinct row and feature).  Integer sums, so the result is the same bit for bit either way;
// PNR_HASH_FIXED_COMBINE=0 builds the plain scatter (tools/time_hashgrid_backward.py times both).
#ifndef PNR_HASH_FIXED_COMBINE
#define PNR_HASH_FIXED_COMBINE 1
#endif

constexpr int32_t kNoScale = INT32_MIN;   // scale of a level whose finite gradients are all zero: it adds nothing
constexpr int kFixedMaxBlocks = 2048;

// The workspace, in this order: int64 acc [L, T, F]; u32 poison bits, one per (l, e, f) entry, in 16-byte units;
// u32 max_bits [L] (|g| of the largest finite gradient of the level, as fp32 bits); i32 scale [L]; u32 flags [2]
// (any non-finite gradient, blocks done); the whole rounded up to 16 bytes.
struct FixedLayout {
  size_t acc, poison, max_bits, scale, flags, total;
  FixedLayout(int L, int F, int T_log2) {
    const size_t entries = (size_t)L * F << T_log2;
    acc = 0;
    poison = entries * sizeof(int64_t);
    max_bits = poison + ((entries + 31) / 32 * 4 + 15) / 16 * 16;
    scale = max_bits + (size_t)L * 4;
    flags = scale + (size_t)L * 4;
    total = (flags + 8 + 15) / 16 * 16;
  }
};

struct FixedWs {
  int64_t* acc; uint32_t* poison; uint32_t* max_bits; int32_t* scale; uint32_t* flags;
};

__device__ __forceinline__ double pow2d(int e) {            // 2^e, exact, for |e| <= 1022
  return __longlong_as_double((long long)(e + 1023) << 52);
}

// e of frexp(m) = frac * 2^e, frac in [0.5, 1), for a positive finite fp32 m given by its bits (subnormals included)
__device__ __forceinline__ int frexp_exponent(uint32_t bits) {
  const uint32_t E = bits >> 23;
  return E ? (int)E - 126 : 32 - __clz(bits) - 149;
}

// m_l = max |grad_out[p, l*F + f]| over the finite values, as fp32 bits (for non-negative floats the bit patterns order
// like the values, so atomicMax on them is the max in any order); flags[0] = 1 when any value is non-finite.  The
// grid stride is a multiple of the row width W = L*F, so each thread stays on one column.  The last block to finish
// derives s_l = 61 - ceil(log2 n) - e_l from the maxima.
__global__ void __launch_bounds__(256) hashgrid_fixed_maxima_kernel(const float* __restrict__ g, int64_t total, int W,
                                                                    int F, int L, int clog2n, FixedWs w) {
  __shared__ uint32_t smax[kHashMaxLevels];
  __shared__ int sbad;
  __shared__ bool last;
  if (threadIdx.x < kHashMaxLevels) smax[threadIdx.x] = 0;
  if (threadIdx.x == 0) sbad = 0;
  __syncthreads();
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x / W * W;
  if (tid < stride) {
    uint32_t m = 0;
    bool bad = false;
#pragma unroll 4
    for (int64_t i = tid; i < total; i += stride) {
      const uint32_t b = __float_as_uint(g[i]) & 0x7fffffffu;
      if (b >= 0x7f800000u) bad = true;
      else m = max(m, b);
    }
    if (m) atomicMax(&smax[(int)(tid % W) / F], m);
    if (bad) sbad = 1;
  }
  __syncthreads();
  if (threadIdx.x < L && smax[threadIdx.x]) atomicMax(&w.max_bits[threadIdx.x], smax[threadIdx.x]);
  if (threadIdx.x == 0 && sbad) atomicOr(&w.flags[0], 1u);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&w.flags[1], 1u) == gridDim.x - 1;
  __syncthreads();
  if (last && threadIdx.x < L) {
    __threadfence();
    const uint32_t mb = atomicOr(&w.max_bits[threadIdx.x], 0u);
    w.scale[threadIdx.x] = mb ? 61 - clog2n - frexp_exponent(mb) : kNoScale;
  }
}

// Sends one corner's F integers (and the F poison bits of its non-finite gradients) to row idx of the level.
template <int F>
__device__ __forceinline__ void fixed_emit(int64_t* __restrict__ acc, uint32_t* __restrict__ poison, size_t row,
                                           const long long (&q)[F], uint32_t bad, bool live) {
  const size_t b0 = row * F;                                  // first poison bit of the row: its F bits share a word
#if PNR_HASH_FIXED_COMBINE
  const unsigned lane = threadIdx.x & 31u;
  const unsigned grp = __match_any_sync(0xffffffffu, live ? (unsigned)row : 0xffffffffu);
  if (grp == (1u << lane)) {
    if (!live) return;
#pragma unroll
    for (int f = 0; f < F; ++f)
      if (q[f]) atomicAdd(reinterpret_cast<unsigned long long*>(acc) + b0 + f, (unsigned long long)q[f]);
    if (bad) atomicOr(poison + (b0 >> 5), bad << (b0 & 31));
    return;
  }
  // the group's sum mod 2^64 from three 22-bit limbs (each limb's sum over <= 32 lanes stays below 2^27)
  const bool leader = (unsigned)(__ffs(grp) - 1) == lane;
#pragma unroll
  for (int f = 0; f < F; ++f) {
    const unsigned long long u = (unsigned long long)q[f];
    const unsigned s0 = __reduce_add_sync(grp, (unsigned)(u & 0x3fffffu));
    const unsigned s1 = __reduce_add_sync(grp, (unsigned)((u >> 22) & 0x3fffffu));
    const unsigned s2 = __reduce_add_sync(grp, (unsigned)(u >> 44));
    const unsigned long long t = (unsigned long long)s0 + ((unsigned long long)s1 << 22) + ((unsigned long long)s2 << 44);
    if (leader && live && t) atomicAdd(reinterpret_cast<unsigned long long*>(acc) + b0 + f, t);
  }
  const uint32_t bm = __reduce_or_sync(grp, bad);
  if (leader && live && bm) atomicOr(poison + (b0 >> 5), bm << (b0 & 31));
#else
  if (!live) return;
#pragma unroll
  for (int f = 0; f < F; ++f)
    if (q[f]) atomicAdd(reinterpret_cast<unsigned long long*>(acc) + b0 + f, (unsigned long long)q[f]);
  if (bad) atomicOr(poison + (b0 >> 5), bad << (b0 & 31));
#endif
}

// The scatter: hashgrid_backward_kernel's thread layout (one point x 8/F levels) and corner arithmetic; contribution
// c = fp32(w_k * g), q = round-to-nearest-even(c * 2^s_l) as an int64, acc[l, idx, f] += q.  A non-finite g sets the
// poison bits of its (l, idx_k, f) at all 8 corners instead.  Lanes past n stay in the loop (as dead lanes) so that a
// warp's combining sees all 32 lanes.
template <int F>
__global__ void __launch_bounds__(256) hashgrid_fixed_scatter_kernel(HashArgs a, const float* __restrict__ gout, FixedWs w) {
  constexpr int LPT = 8 / F;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int l0 = blockIdx.y * LPT;
  const bool live = i < a.n;
#if !PNR_HASH_FIXED_COMBINE
  if (!live) return;
#endif
  const uint32_t T = 1u << a.T_log2, mask = T - 1u;
  float v[3] = {0.f, 0.f, 0.f};
  if (live) {
    const float x[3] = {a.x[i * 3], a.x[i * 3 + 1], a.x[i * 3 + 2]};
    hash_normalize(x, a.aabb, v);
  }
  const float* go = gout + (live ? i : 0) * (int64_t)(a.L * F);
#pragma unroll
  for (int ll = 0; ll < LPT; ++ll) {
    const int l = l0 + ll;
    if (l >= a.L) break;
    const int32_t s = w.scale[l];
    const double up = s == kNoScale ? 0.0 : pow2d(s);      // kNoScale: every finite g of the level is 0
    const uint32_t res = a.res[l], res1 = res + 1u;
    const bool dense = (uint64_t)res1 * res1 * res1 <= (uint64_t)T;
    float wv[3], g[F];
    uint32_t c[3], bad = 0;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      g[f] = live ? go[l * F + f] : 0.f;
      if (!isfinite(g[f])) { bad |= 1u << f; g[f] = 0.f; }
    }
    hash_cell(v, res, c, wv);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      uint32_t idx;
      const float wk = hash_corner(c, wv, k, res1, dense, mask, idx);
      long long q[F];
#pragma unroll
      for (int f = 0; f < F; ++f) q[f] = __double2ll_rn(__dmul_rn((double)__fmul_rn(wk, g[f]), up));
      fixed_emit<F>(w.acc, w.poison, (size_t)l * T + idx, q, bad, live);
    }
  }
}

// grad_table[i] += fp32((double)acc[i] * 2^-s_l): int64 -> double (RN), the exact power-of-two product, double -> float
// (RN), one fp32 add.  NaN where a poison bit is set; a level without a scale is left as it is.
__global__ void __launch_bounds__(256) hashgrid_fixed_finalize_kernel(FixedWs w, int64_t total, int TF_log2, float* gtab) {
  const bool any_bad = w.flags[0] != 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (any_bad && ((w.poison[i >> 5] >> (i & 31)) & 1u)) {
      gtab[i] = __int_as_float(0x7fffffff);
      continue;
    }
    const int32_t s = w.scale[i >> TF_log2];
    if (s == kNoScale) continue;
    gtab[i] = __fadd_rn(gtab[i], __double2float_rn(__dmul_rn(__ll2double_rn(w.acc[i]), pow2d(-s))));
  }
}

}  // namespace
}  // namespace pnr

using namespace pnr;

extern "C" int pnr_panoptic_fuse(const float* semantic_map, const float* instance_map, int64_t R, int32_t C, int32_t K,
                                 const uint8_t* is_thing, const int32_t* inst_class, const int32_t* inst_id,
                                 const int32_t* class_id, const uint8_t* palette, int32_t* panoptic, int16_t* sem_label,
                                 int16_t* inst_slot, uint8_t* color, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(R > 0 && semantic_map && C > 0 && C < 32768 && K >= 0 && K < 32768, "pnr_panoptic_fuse: bad sizes / null semantic_map");
  PNR_CHECK_ARG(!(instance_map && K > 0) || (is_thing && inst_class),
                "pnr_panoptic_fuse: instance_map needs is_thing [C] and inst_class [K]");
  FuseArgs a{semantic_map, K > 0 ? instance_map : nullptr, R, C, K, is_thing, inst_class, inst_id, class_id, palette,
             panoptic, sem_label, inst_slot, color};
  panoptic_fuse_kernel<<<(unsigned)((R + 7) / 8), 256, 0, (cudaStream_t)stream>>>(a);
  PNR_LAUNCH_CHECK("panoptic_fuse_kernel");
  return PNR_OK;
}

extern "C" int pnr_hashgrid_encode(const float* x, int64_t n, const float* aabb, const float* table, int32_t L, int32_t F,
                                   int32_t T_log2, float base_resolution, float per_level_scale, float* out, void* stream) {
  if (n == 0) return PNR_OK;
  PNR_CHECK_ARG(x && table && out && n > 0, "pnr_hashgrid_encode: null pointer");
  PNR_CHECK_ARG(L >= 1 && L <= 32 && (F == 1 || F == 2 || F == 4 || F == 8), "pnr_hashgrid_encode: L=%d F=%d (L in [1,32], F in {1,2,4,8})", L, F);
  PNR_CHECK_ARG(hash_table_aligned(table, F), "pnr_hashgrid_encode: table not aligned to its %d features (a float%d per corner)", F, F);
  PNR_CHECK_ARG(T_log2 >= 4 && T_log2 <= 28, "pnr_hashgrid_encode: T_log2=%d outside [4,28]", T_log2);
  PNR_CHECK_ARG(base_resolution >= 1.0f && per_level_scale >= 1.0f, "pnr_hashgrid_encode: base_resolution / per_level_scale < 1");
  const double finest = (double)base_resolution * pow((double)per_level_scale, (double)(L - 1));
  PNR_CHECK_ARG(finest < 1048576.0, "pnr_hashgrid_encode: finest resolution %.0f >= 2^20", finest);
  HashArgs a{x, n, table, out, aabb, L, F, T_log2, {}};
  hash_level_resolutions(L, base_resolution, per_level_scale, a.res);
  const int lpt = 8 / F;   // levels per thread: 8 output features = one 32-byte sector
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)((L + lpt - 1) / lpt));
  switch (F) {
    case 1: hashgrid_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(a); break;
    case 2: hashgrid_kernel<2><<<grid, 256, 0, (cudaStream_t)stream>>>(a); break;
    case 4: hashgrid_kernel<4><<<grid, 256, 0, (cudaStream_t)stream>>>(a); break;
    default: hashgrid_kernel<8><<<grid, 256, 0, (cudaStream_t)stream>>>(a); break;
  }
  PNR_LAUNCH_CHECK("hashgrid_kernel");
  return PNR_OK;
}

extern "C" int pnr_hashgrid_backward(const float* x, int64_t n, const float* aabb, const float* grad_out, int32_t L, int32_t F,
                                     int32_t T_log2, float base_resolution, float per_level_scale, float* grad_table,
                                     void* stream) {
  if (n == 0) return PNR_OK;
  PNR_CHECK_ARG(x && grad_out && grad_table && n > 0, "pnr_hashgrid_backward: null pointer");
  PNR_CHECK_ARG(L >= 1 && L <= 32 && (F == 1 || F == 2 || F == 4 || F == 8), "pnr_hashgrid_backward: L=%d F=%d (L in [1,32], F in {1,2,4,8})", L, F);
  PNR_CHECK_ARG(T_log2 >= 4 && T_log2 <= 28, "pnr_hashgrid_backward: T_log2=%d outside [4,28]", T_log2);
  PNR_CHECK_ARG(base_resolution >= 1.0f && per_level_scale >= 1.0f, "pnr_hashgrid_backward: base_resolution / per_level_scale < 1");
  const double finest = (double)base_resolution * pow((double)per_level_scale, (double)(L - 1));
  PNR_CHECK_ARG(finest < 1048576.0, "pnr_hashgrid_backward: finest resolution %.0f >= 2^20", finest);
  HashArgs a{x, n, nullptr, nullptr, aabb, L, F, T_log2, {}};
  hash_level_resolutions(L, base_resolution, per_level_scale, a.res);
  const int lpt = 8 / F;
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)((L + lpt - 1) / lpt));
  switch (F) {
    case 1: hashgrid_backward_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(a, grad_out, grad_table); break;
    case 2: hashgrid_backward_kernel<2><<<grid, 256, 0, (cudaStream_t)stream>>>(a, grad_out, grad_table); break;
    case 4: hashgrid_backward_kernel<4><<<grid, 256, 0, (cudaStream_t)stream>>>(a, grad_out, grad_table); break;
    default: hashgrid_backward_kernel<8><<<grid, 256, 0, (cudaStream_t)stream>>>(a, grad_out, grad_table); break;
  }
  PNR_LAUNCH_CHECK("hashgrid_backward_kernel");
  return PNR_OK;
}

static bool hash_fixed_shape_ok(int32_t L, int32_t F, int32_t T_log2) {
  return L >= 1 && L <= 32 && (F == 1 || F == 2 || F == 4 || F == 8) && T_log2 >= 4 && T_log2 <= 28;
}

extern "C" size_t pnr_hashgrid_fixed_workspace_bytes(int32_t L, int32_t F, int32_t T_log2) {
  return hash_fixed_shape_ok(L, F, T_log2) ? FixedLayout(L, F, T_log2).total : 0;
}

extern "C" int pnr_hashgrid_backward_fixed(const float* x, int64_t n, const float* aabb, const float* grad_out, int32_t L,
                                           int32_t F, int32_t T_log2, float base_resolution, float per_level_scale,
                                           float* grad_table, void* workspace, size_t workspace_bytes, void* stream) {
  static const char* fn = "pnr_hashgrid_backward_fixed";
  if (n == 0) return PNR_OK;
  PNR_CHECK_ARG(n > 0, "%s: n=%lld", fn, (long long)n);
  PNR_CHECK_ARG(x, "%s: x is null", fn);
  PNR_CHECK_ARG(grad_out, "%s: grad_out is null", fn);
  PNR_CHECK_ARG(grad_table, "%s: grad_table is null", fn);
  PNR_CHECK_ARG(L >= 1 && L <= 32 && (F == 1 || F == 2 || F == 4 || F == 8), "%s: L=%d F=%d (L in [1,32], F in {1,2,4,8})", fn, L, F);
  PNR_CHECK_ARG(T_log2 >= 4 && T_log2 <= 28, "%s: T_log2=%d outside [4,28]", fn, T_log2);
  PNR_CHECK_ARG(base_resolution >= 1.0f && per_level_scale >= 1.0f, "%s: base_resolution / per_level_scale < 1", fn);
  const double finest = (double)base_resolution * pow((double)per_level_scale, (double)(L - 1));
  PNR_CHECK_ARG(finest < 1048576.0, "%s: finest resolution %.0f >= 2^20", fn, finest);
  const FixedLayout lay(L, F, T_log2);
  PNR_CHECK_ARG(workspace != nullptr && workspace_bytes >= lay.total,
                "%s: workspace of %zu bytes, %zu needed (pnr_hashgrid_fixed_workspace_bytes)", fn, workspace_bytes, lay.total);
  PNR_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "%s: workspace must be 16-byte aligned", fn);
  char* ws = static_cast<char*>(workspace);
  const FixedWs w{reinterpret_cast<int64_t*>(ws + lay.acc), reinterpret_cast<uint32_t*>(ws + lay.poison),
                  reinterpret_cast<uint32_t*>(ws + lay.max_bits), reinterpret_cast<int32_t*>(ws + lay.scale),
                  reinterpret_cast<uint32_t*>(ws + lay.flags)};
  cudaStream_t st = (cudaStream_t)stream;
  PNR_CUDA(cudaMemsetAsync(workspace, 0, lay.total, st));
  int clog2n = 0;
  while (clog2n < 63 && ((int64_t)1 << clog2n) < n) ++clog2n;
  const int W = L * F;
  const int64_t total_g = n * W;
  const unsigned mblocks = (unsigned)std::min<int64_t>((total_g + 1023) / 1024, kFixedMaxBlocks);
  hashgrid_fixed_maxima_kernel<<<mblocks, 256, 0, st>>>(grad_out, total_g, W, F, L, clog2n, w);
  PNR_LAUNCH_CHECK("hashgrid_fixed_maxima_kernel");
  HashArgs a{x, n, nullptr, nullptr, aabb, L, F, T_log2, {}};
  hash_level_resolutions(L, base_resolution, per_level_scale, a.res);
  const int lpt = 8 / F;
  const dim3 grid((unsigned)((n + 255) / 256), (unsigned)((L + lpt - 1) / lpt));
  switch (F) {
    case 1: hashgrid_fixed_scatter_kernel<1><<<grid, 256, 0, st>>>(a, grad_out, w); break;
    case 2: hashgrid_fixed_scatter_kernel<2><<<grid, 256, 0, st>>>(a, grad_out, w); break;
    case 4: hashgrid_fixed_scatter_kernel<4><<<grid, 256, 0, st>>>(a, grad_out, w); break;
    default: hashgrid_fixed_scatter_kernel<8><<<grid, 256, 0, st>>>(a, grad_out, w); break;
  }
  PNR_LAUNCH_CHECK("hashgrid_fixed_scatter_kernel");
  const int64_t entries = (int64_t)W << T_log2;
  const unsigned fblocks = (unsigned)std::min<int64_t>((entries + 255) / 256, 8 * kFixedMaxBlocks);
  hashgrid_fixed_finalize_kernel<<<fblocks, 256, 0, st>>>(w, entries, T_log2 + __builtin_ctz((unsigned)F), grad_table);
  PNR_LAUNCH_CHECK("hashgrid_fixed_finalize_kernel");
  return PNR_OK;
}


// ------------------------------------------------------------------------------------------------ losses
// SURVEY 8(f) rank 2, the loss side (the reference's NetworkWrapper computes these with torch ops on the rendered
// maps; its exact terms are not in the mount - the four below are the paper's: photometric, depth, 2D pseudo-label
// cross-entropy on the rendered semantics, and the cross-entropy of the fixed (bounding-primitive) semantics), plus the
// instance term (softmax cross-entropy of the rendered instance logits against the dominant primitive's slot; rule
// chosen here, DESIGN 3.4).
// One pass per ray: the per-ray value of every term and the gradient w.r.t. every map it reads, already scaled by
// the term's weight and normaliser, so that `pnr_composite_backward` can consume them directly.
namespace pnr {
namespace {

struct LossArgs {
  pnr_loss_args a;
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, d));
  return v;
}
__device__ __forceinline__ float warp_add(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// Softmax cross-entropy of the logits s[0, n) against `label` (0 <= label < n), one warp, lanes stride the logits.
// Returns lse(s) - s[label] on every lane; when d != null writes d[c] = scale(softmax(s)[c] - [c == label]).
template <class Scale>
__device__ __forceinline__ float softmax_xent(const float* __restrict__ s, int n, int label, int lane,
                                              float* __restrict__ d, Scale scale) {
  float m = -INFINITY;
  for (int c = lane; c < n; c += 32) m = fmaxf(m, s[c]);
  m = warp_max(m);
  float z = 0.f;
  for (int c = lane; c < n; c += 32) z += expf(s[c] - m);
  z = warp_add(z);
  // lse - s[label] and softmax = exp(s - lse) are not formed through lse = m + log(z): with logits of ~1e4, lse
  // rounds at ~1e-3 and that error would go straight into the loss and every probability.  m - s[c] is exact
  // or rounded relative to itself, so both stay within a few ulps of their own value.
  if (d != nullptr)
    for (int c = lane; c < n; c += 32) d[c] = scale(expf(s[c] - m) / z - (c == label ? 1.f : 0.f));
  return (m - s[label]) + logf(z);
}

// Instance targets, before the loss pass: inst_label[r] = the lowest slot holding the maximum of fixed_instance_map[r]
// when that maximum is >= inst_min_weight, else -1 (a NaN anywhere in the row makes the maximum NaN: not counted).
// *n_inst (zeroed before the launch) += the block's count: one integer atomic per block, so the count is exact.
__global__ void __launch_bounds__(256) instance_labels_kernel(LossArgs L) {
  const pnr_loss_args& a = L.a;
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  bool counted = false;
  if (r < a.R) {
    const float* v = a.fixed_instance_map + r * a.K;
    float best = -INFINITY;
    int arg = 0x7fffffff;
    bool nan = false;
    for (int c = lane; c < a.K; c += 32) {
      const float x = v[c];
      if (x != x) nan = true;
      else if (x > best || arg == 0x7fffffff) { best = x; arg = c; }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, d);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, d);
      if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
    }
    nan = __any_sync(0xffffffffu, nan);
    counted = !nan && best >= a.inst_min_weight;
    if (lane == 0) a.inst_label[r] = counted ? arg : -1;
  }
  const int n = __syncthreads_count(lane == 0 && counted);
  if (threadIdx.x == 0 && n > 0) atomicAdd(a.n_inst, n);
}

__global__ void __launch_bounds__(256) losses_kernel(LossArgs L) {
  const pnr_loss_args& a = L.a;
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= a.R) return;
  float l_rgb = 0.f, l_depth = 0.f, l_sem = 0.f, l_fix = 0.f;
  // photometric: sum over the 3 channels of (rgb - gt)^2, fine and (optionally) coarse
  if (a.rgb_gt != nullptr && lane < 3) {
    const float gt = a.rgb_gt[r * 3 + lane];
    if (a.rgb_map != nullptr) {
      const float d = a.rgb_map[r * 3 + lane] - gt;
      l_rgb += d * d;
      if (a.d_rgb_map) a.d_rgb_map[r * 3 + lane] = 2.0f * d * a.w_rgb * a.inv_n_rgb;
    }
    if (a.rgb_map0 != nullptr) {
      const float d = a.rgb_map0[r * 3 + lane] - gt;
      l_rgb += d * d;
      if (a.d_rgb_map0) a.d_rgb_map0[r * 3 + lane] = 2.0f * d * a.w_rgb * a.inv_n_rgb;
    }
  }
  l_rgb = warp_add(l_rgb);
  // depth: |depth - gt| where gt > 0
  if (a.depth_map != nullptr && a.depth_gt != nullptr) {
    const float gt = a.depth_gt[r];
    const bool ok = gt > 0.f;
    const float d = a.depth_map[r] - gt;
    l_depth = ok ? fabsf(d) : 0.f;
    if (a.d_depth_map && lane == 0) a.d_depth_map[r] = ok ? (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * a.w_depth * a.inv_n_depth : 0.f;
  }
  const int label = a.label ? a.label[r] : -1;
  const bool has = label >= 0 && label < a.C;
  const float conf = (has && a.label_weight) ? a.label_weight[r] : 1.0f;
  // 2D pseudo-label cross-entropy on the rendered semantics
  if (a.semantic_map != nullptr && a.C > 0) {
    const float* s = a.semantic_map + r * a.C;
    // the map is a rendered probability: -log(max(p_label, eps)); the gradient passes at p == eps, as torch.clamp_min's
    if (a.sem_is_prob) {
      const float p = has ? s[label] : 1.0f;
      const float pc = fmaxf(p, a.eps);
      l_sem = has ? -logf(pc) * conf : 0.f;
      if (a.d_semantic_map)
        for (int c = lane; c < a.C; c += 32)
          a.d_semantic_map[r * a.C + c] = (has && c == label && p >= a.eps) ? -conf * a.w_sem * a.inv_n_sem / pc : 0.f;
    } else if (has) {        // the map is rendered logits: softmax cross-entropy
      l_sem = softmax_xent(s, a.C, label, lane, a.d_semantic_map ? a.d_semantic_map + r * a.C : nullptr,
                           [&](float g) { return g * conf * a.w_sem * a.inv_n_sem; }) * conf;
    } else if (a.d_semantic_map) {
      for (int c = lane; c < a.C; c += 32) a.d_semantic_map[r * a.C + c] = 0.f;
    }
  }
  // instance: softmax cross-entropy of the rendered instance logits against the label pass's target
  if (a.instance_map != nullptr) {
    const int k = a.inst_label[r];
    float* d = a.d_instance_map ? a.d_instance_map + r * a.K : nullptr;
    float l_inst = 0.f;
    if (k >= 0) {
      const float n = (float)*a.n_inst;     // >= 1: this ray is counted
      l_inst = softmax_xent(a.instance_map + r * a.K, a.K, k, lane, d, [&](float g) { return g * a.w_inst / n; });
    } else if (d != nullptr) {
      for (int c = lane; c < a.K; c += 32) d[c] = 0.f;
    }
    if (a.per_ray_inst != nullptr && lane == 0) a.per_ray_inst[r] = l_inst;
  }
  // fixed (bounding-primitive) semantics: a rendered probability by construction
  if (a.fixed_semantic_map != nullptr && a.C > 0) {
    const float p = has ? a.fixed_semantic_map[r * a.C + label] : 1.0f;
    const float pc = fmaxf(p, a.eps);
    l_fix = has ? -logf(pc) * conf : 0.f;
    if (a.d_fixed_semantic_map)
      for (int c = lane; c < a.C; c += 32)
        a.d_fixed_semantic_map[r * a.C + c] = (has && c == label && p >= a.eps) ? -conf * a.w_fix * a.inv_n_sem / pc : 0.f;
  }
  if (a.per_ray != nullptr && lane == 0)
    *reinterpret_cast<float4*>(a.per_ray + r * 4) = make_float4(l_rgb, l_depth, l_sem, l_fix);
}

}  // namespace
}  // namespace pnr

extern "C" int pnr_losses(const pnr_loss_args* args, void* stream) {
  PNR_CHECK_ARG(args, "pnr_losses: null pointer");
  if (args->R == 0) return PNR_OK;
  PNR_CHECK_ARG(args->R > 0 && args->C >= 0 && args->C < 32768, "pnr_losses: bad sizes");
  PNR_CHECK_ARG(!(args->rgb_map || args->rgb_map0) || args->rgb_gt, "pnr_losses: rgb maps without rgb_gt");
  PNR_CHECK_ARG(!(args->semantic_map || args->fixed_semantic_map) || (args->label && args->C > 0),
                "pnr_losses: semantic maps need label [R] and C > 0");
  PNR_CHECK_ARG(args->eps > 0.f, "pnr_losses: eps must be > 0");
  const bool inst = args->instance_map != nullptr;
  if (inst) {
    PNR_CHECK_ARG(args->K >= 1 && args->K <= 32767, "pnr_losses: K=%d outside [1,32767] with instance_map", args->K);
    PNR_CHECK_ARG(args->fixed_instance_map, "pnr_losses: instance_map without fixed_instance_map");
    PNR_CHECK_ARG(args->inst_label, "pnr_losses: instance_map needs inst_label [R]");
    PNR_CHECK_ARG(args->n_inst, "pnr_losses: instance_map needs n_inst");
    PNR_CHECK_ARG(args->inst_min_weight > 0.f && args->inst_min_weight <= 1.f,
                  "pnr_losses: inst_min_weight=%g outside (0,1]", (double)args->inst_min_weight);
  }
  LossArgs L{*args};
  const unsigned blocks = (unsigned)((args->R + 7) / 8);
  if (inst) {
    PNR_CUDA(cudaMemsetAsync(args->n_inst, 0, sizeof(int32_t), (cudaStream_t)stream));
    instance_labels_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(L);
    PNR_LAUNCH_CHECK("instance_labels_kernel");
  }
  losses_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(L);
  PNR_LAUNCH_CHECK("losses_kernel");
  return PNR_OK;
}
