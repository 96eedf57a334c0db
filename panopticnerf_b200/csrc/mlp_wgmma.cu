// mlp_wgmma.cu — fused Network.forward (SURVEY.md 8(a) a7 + a8) on sm_90a tensor cores (wgmma).
//
// One persistent CTA per SM walks tiles of kRows = 64 samples (the M of one warpgroup MMA).  Per tile the whole MLP
// runs on-chip:
//   * the consumer warpgroup (128 threads) forms pts = o + d*z and the positional encodings gamma(x) (threads 0-63,
//     one row each) and gamma(d) (threads 64-127), splits them into 16-bit hi/lo parts and writes them into shared
//     memory in the no-swizzle K-major operand layout (a hash-grid network: h(x) gathered from its table in place of
//     gamma(x), hashgrid_math.cuh);
//   * one weight-stream warp copies the pre-packed weight stages (<= 32 KB: hi image then lo image of an N-row x 64-K
//     tile) from L2 into a 4-slot shared-memory ring, one K-half of a stage per 16 KB slot, with cp.async.bulk +
//     mbarrier complete_tx;
//   * the consumer warpgroup issues wgmma m64nNk16 (N <= 128 per half of a step), both operands in shared memory:
//     A = an embedding or the previous layer's activations, B = the weight stage; fp32 accumulators in registers;
//   * once a step's MMAs have retired, its epilogue adds the bias, applies the ReLU, splits into hi/lo and stores the
//     next layer's A operand over the one the step has just consumed.  A trunk step does this straight from the
//     accumulator registers (epi_regs_act); every other step passes its accumulators through a 64 x 128 fp32 staging
//     tile in shared memory (one 128-column window at a time) to a row epilogue with two threads per row (column
//     shares).  The sigma head (N=1) and rgb head (N=3) are CUDA-core dot products inside the row epilogue; semantic /
//     instance logits are written straight to `raw`.
//
// The per-tile program (mlp_program.h) is built on the host once per weight load.  This kernel runs its steps in
// order, each one's epilogue after all of its MMAs, and takes from the program the stage list (weight bytes, N,
// operand columns, K steps) and the epilogue table.
//
// Precision: operands are 16-bit (fp16 or bf16), accumulation fp32.  The "x3" modes compute every product
// as A_hi*B_hi + A_lo*B_hi + A_hi*B_lo with x = hi + lo split in the operand format: ~2^-21 relative
// per product for fp16x3 (default; what the 1e-4 parity tolerance needs with margin), ~2^-17 for
// bf16x3 (fp32 exponent range).  The 1-pass modes keep the first term only (fast, out of tolerance).
// Range check: a value written into an operand (the embeddings included) whose hi part rounds to inf (fp16 modes:
// |x| >= 65520) or that is NaN sets bit 0 of the context's sticky status word (pnr_status): overflow is reported, never
// silent.  The ReLU keeps a NaN, as torch.relu does, so a NaN input or parameter reaches the outputs as well.
#include <cstddef>
#include "common.cuh"
#include "composite_math.cuh"
#include "hashgrid_math.cuh"
#include "mlp_program.h"
#include "sm90.cuh"

namespace pnr {

// Write 8 consecutive K elements (one 16-byte core-matrix row) of this thread's row, split hi/lo; returns the hi part.
template <int PASSES, int FMT>
__device__ __forceinline__ uint4 store_core_row(uint8_t* hi_base, uint8_t* lo_base, int kcore, int row,
                                                const float (&v)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split_x2<FMT>(v[2 * j], v[2 * j + 1], h[j], l[j]);
  const int off = (kcore * kRows + row) * 16;
  *reinterpret_cast<uint4*>(hi_base + off) = make_uint4(h[0], h[1], h[2], h[3]);
  if (PASSES == 3) *reinterpret_cast<uint4*>(lo_base + off) = make_uint4(l[0], l[1], l[2], l[3]);
  return make_uint4(h[0], h[1], h[2], h[3]);
}

// gamma(p) = [p, sin(2^0 p), cos(2^0 p), ...] padded with zeros to KPAD, streamed out 8 at a time.
// The values carry a sign: `vmax` collects the magnitudes of the hi parts (range check), as in hash_rows.
template <int PASSES, int FMT, int LMAX, int KPAD>
__device__ __forceinline__ void encode_row(const float (&p)[3], int L, uint8_t* hi_base,
                                           uint8_t* lo_base, int row, uint32_t& vmax) {
  float v[KPAD];
#pragma unroll
  for (int i = 0; i < KPAD; ++i) v[i] = 0.f;
  v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
  float f = 1.0f;
#pragma unroll
  for (int k = 0; k < LMAX; ++k) {
    if (k < L) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float sn, cs;
        sincosf(p[c] * f, &sn, &cs);
        if (3 + 6 * k + c < KPAD) v[3 + 6 * k + c] = sn;
        if (3 + 6 * k + 3 + c < KPAD) v[3 + 6 * k + 3 + c] = cs;
      }
    }
    f *= 2.0f;
  }
#pragma unroll
  for (int g = 0; g < KPAD / 8; ++g) {
    float w8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) w8[j] = v[g * 8 + j];
    const uint4 h = store_core_row<PASSES, FMT>(hi_base, lo_base, g, row, w8);
    vmax = __vimax3_u16x2(vmax, h.x & 0x7FFF7FFFu, h.y & 0x7FFF7FFFu);
    vmax = __vimax3_u16x2(vmax, h.z & 0x7FFF7FFFu, h.w & 0x7FFF7FFFu);
  }
}

// h(x) of one row (hash-grid trunk input): core rows [g0, g1) of the embedding operand, each = 8 features = 8 / F whole
// levels (hash_level_blend, the arithmetic of pnr_hashgrid_encode), features past L*F = the zero padding; split hi/lo
// like gamma(x).  The features carry a sign: `vmax` collects the magnitudes of the hi parts (range check).
template <int PASSES, int FMT, int F>
__device__ __forceinline__ void hash_rows(const MlpParams& p, const float (&v)[3], int g0, int g1, uint8_t* hi_base,
                                          uint8_t* lo_base, int row, uint32_t& vmax) {
  constexpr int kLevelsPerCore = 8 / F;
  const size_t level_floats = (size_t)F << p.hash_T_log2;
#pragma unroll 1
  for (int g = g0; g < g1; ++g) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // one level at a time (a rolled loop keeps this rarely taken branch small next to the MMA code)
#pragma unroll 1
    for (int ll = 0; ll < kLevelsPerCore; ++ll) {
      const int l = g * kLevelsPerCore + ll;
      if (l >= p.hash_L) break;
      float f[F];
#pragma unroll
      for (int j = 0; j < F; ++j) f[j] = 0.f;
      hash_level_blend<F>(p.hash_table + (size_t)l * level_floats, v, p.hash_res[l], (uint32_t)p.hash_T_log2, f);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j / F == ll) acc[j] = f[j % F];
    }
    const uint4 h = store_core_row<PASSES, FMT>(hi_base, lo_base, g, row, acc);
    vmax = __vimax3_u16x2(vmax, h.x & 0x7FFF7FFFu, h.y & 0x7FFF7FFFu);
    vmax = __vimax3_u16x2(vmax, h.z & 0x7FFF7FFFu, h.w & 0x7FFF7FFFu);
  }
}

template <int PASSES, int FMT>
__device__ __forceinline__ void hash_rows_f(const MlpParams& p, const float (&v)[3], int g0, int g1, uint8_t* hi_base,
                                            uint8_t* lo_base, int row, uint32_t& vmax) {
  switch (p.hash_F) {
    case 1: hash_rows<PASSES, FMT, 1>(p, v, g0, g1, hi_base, lo_base, row, vmax); break;
    case 2: hash_rows<PASSES, FMT, 2>(p, v, g0, g1, hi_base, lo_base, row, vmax); break;
    case 4: hash_rows<PASSES, FMT, 4>(p, v, g0, g1, hi_base, lo_base, row, vmax); break;
    default: hash_rows<PASSES, FMT, 8>(p, v, g0, g1, hi_base, lo_base, row, vmax); break;
  }
}

// ------------------------------------------------------------------------------------------------
// Epilogue building blocks.  One thread owns one accumulator row; groups are 16 columns.
// ------------------------------------------------------------------------------------------------

// relu(x) that keeps a NaN, as torch.relu does (fmaxf(NaN, 0) = 0 would hide a NaN input or parameter from the range
// check and from the outputs): one FMNMX.NAN, the instruction count of fmaxf.
__device__ __forceinline__ float relu_nan(float x) {
  float y;
  asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(y) : "f"(x));
  return y;
}

// relu(acc + bias) of columns 4q .. 4q + 3 of a 16-column group, b = their bias
__device__ __forceinline__ float4 relu_bias4(const uint32_t (&r)[16], int q, float4 b) {
  return make_float4(relu_nan(__uint_as_float(r[4 * q + 0]) + b.x), relu_nan(__uint_as_float(r[4 * q + 1]) + b.y),
                     relu_nan(__uint_as_float(r[4 * q + 2]) + b.z), relu_nan(__uint_as_float(r[4 * q + 3]) + b.w));
}

// activation -> next layer's A operand: v = act(acc + bias); [sigma += v . wsig]; split into hi / lo parts.
// `vmax` collects the largest hi-part bit patterns seen (two 16-bit lanes; range check of the operand format).
template <int PASSES, int FMT>
__device__ __forceinline__ void epi_group_act(const uint32_t (&r)[16], int g, const EpiDesc& ed,
                                              const float* bias, const float* wsig, float& sig, uint32_t& vmax,
                                              uint32_t (&hi)[8], uint32_t (&lo)[8]) {
  const float4* b4 = reinterpret_cast<const float4*>(bias + g * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = relu_bias4(r, q, b4[q]);
    if (ed.sigma) {
      const float4 w = reinterpret_cast<const float4*>(wsig + g * 16)[q];
      sig += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
    }
    split_x2<FMT>(v.x, v.y, hi[2 * q], lo[2 * q]);
    split_x2<FMT>(v.z, v.w, hi[2 * q + 1], lo[2 * q + 1]);
    // Range check on the packed hi parts (one 3-input 16x2 max per four values): v >= +0 or the canonical (positive)
    // NaN after the ReLU, so the 16-bit patterns order like the values, with +inf (what an overflowing conversion
    // yields, fp16: v >= 65520) and NaN on top.  The ReLU keeps a NaN accumulator (a NaN input, bias or weight), so it
    // is seen here and reaches the outputs.
#ifndef PNR_ABL_NOVMAX
    vmax = __vimax3_u16x2(vmax, hi[2 * q], hi[2 * q + 1]);
#endif
  }
}

// the 16 activations of group g -> this row of the next layer's A operand (two 16-byte core-matrix rows per part)
template <int PASSES>
__device__ __forceinline__ void epi_group_store(int g, const EpiDesc& ed, uint8_t* op, int row, const uint32_t (&hi)[8],
                                                const uint32_t (&lo)[8]) {
  uint8_t* h = op + (((ed.dst_col - kColOpBase) / 4 + 2 * g) * kRows + row) * 16;
  *reinterpret_cast<uint4*>(h) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(h + kOpKCoreBytes) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
  if (PASSES == 3) {
    uint8_t* l = op + (((ed.dst_lo_col - kColOpBase) / 4 + 2 * g) * kRows + row) * 16;
    *reinterpret_cast<uint4*>(l) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    *reinterpret_cast<uint4*>(l + kOpKCoreBytes) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
  }
}

__device__ __forceinline__ void epi_group_rgb(const uint32_t (&r)[16], int g, const EpiDesc& ed, const float* bias,
                                              const float* wr, float& c0, float& c1, float& c2) {
  // bias and the three weight rows come as 16-byte shared-memory loads (every offset is a multiple of 4 floats)
  const float4* b4 = reinterpret_cast<const float4*>(bias + g * 16);
  const float4* w0 = reinterpret_cast<const float4*>(wr + g * 16);
  const float4* w1 = reinterpret_cast<const float4*>(wr + ed.n + g * 16);
  const float4* w2 = reinterpret_cast<const float4*>(wr + 2 * ed.n + g * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 b = b4[q], a0 = w0[q], a1 = w1[q], a2 = w2[q];
    const float4 v = relu_bias4(r, q, b);
    c0 += v.x * a0.x; c1 += v.x * a1.x; c2 += v.x * a2.x;
    c0 += v.y * a0.y; c1 += v.y * a1.y; c2 += v.y * a2.y;
    c0 += v.z * a0.z; c1 += v.z * a1.z; c2 += v.z * a2.z;
    c0 += v.w * a0.w; c1 += v.w * a1.w; c2 += v.w * a2.w;
  }
}

// logits straight to the raw row.  `dst` / `n_valid` / `c0` describe the half the group lies in: channel of column c
// = (c - c0) relative to dst, real while < n_valid.
__device__ __forceinline__ void epi_group_logits(const uint32_t (&r)[16], int g, int c0, int n_valid,
                                                 const float* bias, float* dst) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int ch = g * 16 + j - c0;
    if (ch < n_valid) dst[ch] = __uint_as_float(r[j]) + bias[g * 16 + j];
  }
}

// ------------------------------------------------------------------------------------------------
// Backward programs (BWD kernels): the three hand-overs that write an A operand, and the gradient output.
//   EPI_RELU_TO_A   forward layer: v = relu(acc + bias); its sign pattern is saved (slot n_valid-1) for the way back
//   EPI_LOADG_TO_A  last forward layer: v = incoming gradient where acc + bias > 0 (relu' = 0 at 0, like autograd)
//   EPI_MASK_TO_A   backward layer: v = acc where the saved pattern of the layer below is set
// `mask_row` = this thread's row in slot 0 / group 0 of the pattern array; `gin` = this row of the incoming gradient.
// ------------------------------------------------------------------------------------------------
template <int PASSES, int FMT>
__device__ __forceinline__ void epi_group_bwd(const uint32_t (&r)[16], int g, const EpiDesc& ed, const float* bias,
                                              uint16_t* mask_row, const float* gin, float* stash_row, float gscale,
                                              float gunscale, uint32_t& vmax, uint32_t (&hi)[8], uint32_t (&lo)[8]) {
  float v[16];
  float sscale = gunscale;     // what the stash receives: gradients unscaled, forward activations as they are
  if (ed.kind == EPI_MASK_TO_A) {
    const uint32_t m = ed.n_valid ? mask_row[((ed.n_valid - 1) * 16 + g) * kRows] : 0xFFFFu;
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = ((m >> j) & 1u) ? __uint_as_float(r[j]) : 0.f;
  } else {
    const float4* b4 = reinterpret_cast<const float4*>(bias + g * 16);
    uint32_t m = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 x = relu_bias4(r, q, b4[q]);
      v[4 * q + 0] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) m |= (v[j] > 0.f ? 1u : 0u) << j;
    if (ed.kind == EPI_LOADG_TO_A) {
      const float4* g4 = reinterpret_cast<const float4*>(gin + g * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 x = g4[q];
        v[4 * q + 0] = ((m >> (4 * q + 0)) & 1u) ? x.x * gscale : 0.f;
        v[4 * q + 1] = ((m >> (4 * q + 1)) & 1u) ? x.y * gscale : 0.f;
        v[4 * q + 2] = ((m >> (4 * q + 2)) & 1u) ? x.z * gscale : 0.f;
        v[4 * q + 3] = ((m >> (4 * q + 3)) & 1u) ? x.w * gscale : 0.f;
      }
    } else {
      sscale = 1.0f;
      if (ed.n_valid) mask_row[((ed.n_valid - 1) * 16 + g) * kRows] = (uint16_t)m;
    }
  }
  if (stash_row != nullptr) {   // fp32 copy of the operand for the weight-gradient GEMMs
    float4* s4 = reinterpret_cast<float4*>(stash_row + g * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      s4[q] = make_float4(v[4 * q] * sscale, v[4 * q + 1] * sscale, v[4 * q + 2] * sscale, v[4 * q + 3] * sscale);
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    split_x2<FMT>(v[4 * q + 0], v[4 * q + 1], hi[2 * q], lo[2 * q]);
    split_x2<FMT>(v[4 * q + 2], v[4 * q + 3], hi[2 * q + 1], lo[2 * q + 1]);
    // gradients carry a sign: the range check compares magnitudes
    vmax = __vimax3_u16x2(vmax, hi[2 * q] & 0x7FFF7FFFu, hi[2 * q + 1] & 0x7FFF7FFFu);
  }
}

// the trunk's output activations: relu(acc + bias) of this group -> the sample's output row (16-byte stores)
__device__ __forceinline__ void epi_group_actout(const uint32_t (&r)[16], int g, const float* bias, float* dst) {
  const float4* b4 = reinterpret_cast<const float4*>(bias + g * 16);
  float4* d4 = reinterpret_cast<float4*>(dst + g * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q) d4[q] = relu_bias4(r, q, b4[q]);
}

// gradient w.r.t. the embedded input: accumulator columns [0, n_valid) of this group -> the sample's output row
// (accumulating: all loads first - one memory latency per group, not one per column).  `vec`: the output rows are
// 16-byte aligned and padded to whole groups (row stride a multiple of 4 floats >= the step's width; the padding
// columns receive the zero-padded weights' zeros): four 16-byte accesses per group instead of sixteen 4-byte ones
// whose 32 lanes each touch a different sector.
__device__ __forceinline__ void epi_group_gradout(const uint32_t (&r)[16], int g, int n_valid, bool accumulate, bool vec,
                                                  float us, float* dst) {
  if (vec) {
    float4* d4 = reinterpret_cast<float4*>(dst + g * 16);
    float4 prev[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) prev[q] = accumulate ? d4[q] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      d4[q] = make_float4(prev[q].x + __uint_as_float(r[4 * q + 0]) * us, prev[q].y + __uint_as_float(r[4 * q + 1]) * us,
                          prev[q].z + __uint_as_float(r[4 * q + 2]) * us, prev[q].w + __uint_as_float(r[4 * q + 3]) * us);
    return;
  }
  float prev[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) prev[j] = (accumulate && g * 16 + j < n_valid) ? dst[g * 16 + j] : 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j)
    if (g * 16 + j < n_valid) dst[g * 16 + j] = prev[j] + __uint_as_float(r[j]) * us;
}

// ------------------------------------------------------------------------------------------------
// Compositing epilogue building blocks (COMP kernels).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum32(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}
// x[j] = this lane's (= this sample's) value of column j.  Returns the sum over the 32 lanes of column
// comp_col_of_lane(lane), by a fixed exchange tree (16 shuffles): lanes swap the half of the columns they give up.
__device__ __forceinline__ float comp_reduce16(const float (&x)[16], int lane) {
  float y[8], z[4], u[2];
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
#pragma unroll
  for (int j = 0; j < 8; ++j) y[j] = (b4 ? x[j + 8] : x[j]) + __shfl_xor_sync(0xffffffffu, b4 ? x[j] : x[j + 8], 16);
#pragma unroll
  for (int j = 0; j < 4; ++j) z[j] = (b3 ? y[j + 4] : y[j]) + __shfl_xor_sync(0xffffffffu, b3 ? y[j] : y[j + 4], 8);
#pragma unroll
  for (int j = 0; j < 2; ++j) u[j] = (b2 ? z[j + 2] : z[j]) + __shfl_xor_sync(0xffffffffu, b2 ? z[j] : z[j + 2], 4);
  float v = (b1 ? u[1] : u[0]) + __shfl_xor_sync(0xffffffffu, b1 ? u[0] : u[1], 2);
  return v + __shfl_xor_sync(0xffffffffu, v, 1);
}
__device__ __forceinline__ int comp_col_of_lane(int lane) { return (lane >> 1) & 15; }   // 8*b4 + 4*b3 + 2*b2 + b1

// logits of one 16-column group, weighted by this sample's compositing weight and summed over the warp's 32 samples
// (one aligned group of a ray); the even lanes write the per-quarter partial sums.
__device__ __forceinline__ void epi_group_logits_comp(const uint32_t (&r)[16], int g, int c0, int n_valid, int ch_base,
                                                      const float* bias, float w, int lane, float* qsum_q) {
  float x[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) x[j] = w * (__uint_as_float(r[j]) + bias[g * 16 + j]);
  const float tot = comp_reduce16(x, lane);
  const int ch = g * 16 + comp_col_of_lane(lane) - c0;
  if ((lane & 1) == 0 && ch < n_valid) qsum_q[ch_base + ch] = tot;
}

// Bit pattern of +inf in the operand format: a hi part >= this is an overflowed (or NaN) activation.
template <int FMT>
__device__ __forceinline__ constexpr uint32_t inf_bits16() {
  return FMT == kFmtF16 ? 0x7C00u : 0x7F80u;
}

// ------------------------------------------------------------------------------------------------
// Weight ring.  The ring region (kRing program stages of kStageBytes) is run as kSlots slots of half a stage: a stage
// arrives as one slot per K-half, slot j holding the K16 steps [k0, k0 + kn) of the stage's hi image and then (x3) the
// same steps of its lo image.  The images keep K-cores outermost, so each part is one contiguous range of the packed
// stream.  Four slots keep two stages in flight while one is consumed.
// ------------------------------------------------------------------------------------------------
constexpr int kSlots = 4;
constexpr int kSlotBytes = kRing * kStageBytes / kSlots;
static_assert(2 * kSlotBytes == kStageBytes, "a program stage is two ring slots");
// ring slot and barrier phase of the gs-th slot taken (the weight stream and the consumers count alike)
__device__ __forceinline__ uint32_t ring_slot(uint32_t gs) { return gs % kSlots; }
__device__ __forceinline__ uint32_t ring_phase(uint32_t gs) { return (gs / kSlots) & 1; }

__device__ __forceinline__ int stage_slots(const StageDesc& sd) { return sd.ksteps > 1 ? 2 : 1; }
// the K16 steps [k0, k0 + kn) of slot j of the stage (the first K-half is the larger one)
__device__ __forceinline__ void slot_ksteps(const StageDesc& sd, int j, int& k0, int& kn) {
  const int h = (sd.ksteps + 1) >> 1;
  k0 = j ? h : 0;
  kn = j ? sd.ksteps - h : h;
}

// The slot's MMAs have retired: one arrival per consumer warp (lane 0) on its empty barrier; slot < 0: none.
__device__ __forceinline__ void release_slot(uint32_t bar_empty, int slot, bool leader) {
  mbar_arrive_if(bar_empty + 8u * (uint32_t)(slot & (kSlots - 1)), leader && slot >= 0);
}

// ------------------------------------------------------------------------------------------------
// MMA issue.  PTX spells out the accumulator registers, so N is a template argument, and ptxas keeps wgmmas in flight
// only where N and the accumulator array are fixed and nothing between a wgmma and the wait that retires it is a call
// or a divergent branch.  So the issue code is dispatched on N once per half of a step (mma_half_n), and within it
// every slot is one straight-line run of wgmmas.
// ------------------------------------------------------------------------------------------------
// Ring position of the consumer warpgroup: gs = slots consumed so far, prev = the slot whose MMAs are still in flight.
struct RingPos {
  uint32_t gs;
  int prev;
};

// KN K16 steps of D (+)= A * B^T, each PASSES products in the order hi*hi, lo*hi, hi*lo (acc = 0: the first product
// overwrites D), as one committed group.
template <int N, int PASSES, int FMT, int KN>
__device__ __forceinline__ void mma_issue(float (&d)[64], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                          uint32_t acc) {
  constexpr uint32_t a_inc16 = (2u * kOpKCoreBytes) >> 4, b_inc16 = (2u * N * 16u) >> 4;   // 16-byte units
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < KN; ++ks) {
    const uint64_t ao = (uint64_t)(ks * a_inc16), bo = (uint64_t)(ks * b_inc16);
    Wgmma<N, FMT>::run(d, a_hi + ao, b_hi + bo, ks == 0 ? acc : 1u);
    if (PASSES == 3) {
      Wgmma<N, FMT>::run(d, a_lo + ao, b_hi + bo, 1u);
      Wgmma<N, FMT>::run(d, a_hi + ao, b_lo + bo, 1u);
    }
  }
  wgmma_commit();
}

// Slot j of stage sd into the accumulator d: wait for it to land, issue its kn (<= KMAX) K16 steps and release the
// previous slot once they are issued (wait_group 1: the previous slot's MMAs are done).
template <int N, int PASSES, int FMT>
__device__ __forceinline__ void mma_slot(float (&d)[64], const StageDesc& sd, int j, uint32_t acc, uint32_t ring_s,
                                         uint32_t bar_full, uint32_t bar_empty, uint32_t emb_s, uint32_t dir_s,
                                         uint32_t op_s, RingPos& rp, bool leader) {
  constexpr int KMAX = PASSES == 3 ? 2 : 4;   // half of a stage's 64 (x3) or 128 (1-pass) K
  constexpr uint32_t a_inc16 = (2u * kOpKCoreBytes) >> 4;
  uint32_t a_hi, a_lo;
  if (sd.a_kind == A_EMB) {
    a_hi = emb_s; a_lo = emb_s + kEmbPartBytes;
  } else if (sd.a_kind == A_DIR) {
    a_hi = dir_s; a_lo = dir_s + kDirPartBytes;
  } else {
    a_hi = op_s + (uint32_t)((sd.a_off - kColOpBase) / 4) * kOpKCoreBytes;
    a_lo = op_s + (uint32_t)((sd.a_lo_off - kColOpBase) / 4) * kOpKCoreBytes;
  }
  int k0, kn;
  slot_ksteps(sd, j, k0, kn);
  const uint32_t slot = ring_slot(rp.gs), ph = ring_phase(rp.gs);
  const uint32_t b = ring_s + slot * (uint32_t)kSlotBytes;
  const uint64_t ad_hi = make_smem_desc_noswz(a_hi, kOpKCoreBytes, 128) + (uint64_t)(k0 * a_inc16);
  const uint64_t ad_lo = make_smem_desc_noswz(a_lo, kOpKCoreBytes, 128) + (uint64_t)(k0 * a_inc16);
  const uint64_t b_hi = make_smem_desc_noswz(b, N * 16u, 128);
  const uint64_t b_lo = make_smem_desc_noswz(b + (uint32_t)kn * N * 32u, N * 16u, 128);
  mbar_wait(bar_full + 8 * slot, ph);
  // one straight-line branch per K-step count, fence to commit: no join between the wgmmas and their commit
  if (kn == 1) mma_issue<N, PASSES, FMT, 1>(d, ad_hi, ad_lo, b_hi, b_lo, acc);
  else if (KMAX == 2 || kn == 2) mma_issue<N, PASSES, FMT, 2>(d, ad_hi, ad_lo, b_hi, b_lo, acc);
  else if (kn == 3) mma_issue<N, PASSES, FMT, (KMAX < 3 ? KMAX : 3)>(d, ad_hi, ad_lo, b_hi, b_lo, acc);
  else mma_issue<N, PASSES, FMT, KMAX>(d, ad_hi, ad_lo, b_hi, b_lo, acc);
  wgmma_wait<1>();
  release_slot(bar_empty, rp.prev, leader);
  rp.prev = (int)slot;
  ++rp.gs;
}

// The stages [si, si_end) of one half of a step (all of width N) into d.
template <int N, int PASSES, int FMT>
__device__ __forceinline__ void mma_half(float (&d)[64], const MlpProgram& prog, int si, int si_end, uint32_t ring_s,
                                         uint32_t bar_full, uint32_t bar_empty, uint32_t emb_s, uint32_t dir_s,
                                         uint32_t op_s, RingPos& rp, bool leader) {
#pragma unroll 1
  for (; si < si_end; ++si) {
    const StageDesc& sd = prog.st[si];
    const uint32_t acc = (sd.flags & F_FIRST) ? 0u : 1u;
#pragma unroll 1
    for (int j = 0; j < stage_slots(sd); ++j)
      mma_slot<N, PASSES, FMT>(d, sd, j, j == 0 ? acc : 1u, ring_s, bar_full, bar_empty, emb_s, dir_s, op_s, rp, leader);
  }
  // retire the half here: no wgmma may be in flight where the N-dispatch merges (the compiler may move accumulators)
  wgmma_wait<0>();
  release_slot(bar_empty, rp.prev, leader);
  rp.prev = -1;
}

template <int PASSES, int FMT>
__device__ __forceinline__ void mma_half_n(float (&d)[64], int n, const MlpProgram& prog, int si, int si_end, uint32_t ring_s,
                                           uint32_t bar_full, uint32_t bar_empty, uint32_t emb_s, uint32_t dir_s,
                                           uint32_t op_s, RingPos& rp, bool leader) {
#define PNR_MMA_N(NN) \
  case NN / 8: mma_half<NN, PASSES, FMT>(d, prog, si, si_end, ring_s, bar_full, bar_empty, emb_s, dir_s, op_s, rp, leader); break;
  switch (n >> 3) {
    PNR_MMA_N(8) PNR_MMA_N(16) PNR_MMA_N(24) PNR_MMA_N(32) PNR_MMA_N(40) PNR_MMA_N(48) PNR_MMA_N(56) PNR_MMA_N(64)
    PNR_MMA_N(72) PNR_MMA_N(80) PNR_MMA_N(88) PNR_MMA_N(96) PNR_MMA_N(104) PNR_MMA_N(112) PNR_MMA_N(120) PNR_MMA_N(128)
    default: __trap();   // not an MMA width: Builder::add_step refuses such a program
  }
#undef PNR_MMA_N
}

// ------------------------------------------------------------------------------------------------
// Trunk steps in registers.  A trunk step (ReLU hand-over without the sigma head, N = 256 as two N = 128 halves, output
// to the activation columns; 7 of the 9 steps of an 8 x 256 network's tile) runs its epilogue straight from the
// accumulator fragments: no staging tile, no barrier per 128-column window, no column shares.  The values and the
// bytes stored are those of the staged epilogue (epi_group_act + epi_group_store): the same fp32 operations on the same
// elements, the same range check.
// ------------------------------------------------------------------------------------------------
// Half HALF of a trunk step, held in `d` (its output always goes to the activation columns kColAHi / kColALo) ->
// relu(acc + bias), split, stored.  Each thread holds rows r0 = 16w + t/4 and r0 + 8, columns 8j + 2(t%4) + {0, 1}:
// one packed 32-bit word per row and part, and a quad of lanes covers one 16-byte core-matrix row (conflict-free: a
// warp stores 8 consecutive 16-byte rows).  `bias` = the step's bias + 2(t%4), `op_t` = the operand region + this
// thread's byte offset r0 * 16 + (t%4) * 4.
template <int PASSES, int FMT, int HALF>
__device__ __forceinline__ void epi_regs_act(const float (&d)[64], const float* bias, uint8_t* op_t, uint32_t& vmax) {
  constexpr int kHi = ((kColAHi - kColOpBase) / 4 + 16 * HALF) * kOpKCoreBytes;
  constexpr int kLo = ((kColALo - kColOpBase) / 4 + 16 * HALF) * kOpKCoreBytes;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float2 b = *reinterpret_cast<const float2*>(bias + 128 * HALF + 8 * j);
    uint32_t h0, l0, h1, l1;
    split_x2<FMT>(relu_nan(d[4 * j + 0] + b.x), relu_nan(d[4 * j + 1] + b.y), h0, l0);
    split_x2<FMT>(relu_nan(d[4 * j + 2] + b.x), relu_nan(d[4 * j + 3] + b.y), h1, l1);
#ifndef PNR_ABL_NOVMAX
    vmax = __vimax3_u16x2(vmax, h0, h1);   // range check, as in epi_group_act
#endif
    *reinterpret_cast<uint32_t*>(op_t + kHi + j * kOpKCoreBytes) = h0;
    *reinterpret_cast<uint32_t*>(op_t + kHi + j * kOpKCoreBytes + 8 * 16) = h1;
    if (PASSES == 3) {
      *reinterpret_cast<uint32_t*>(op_t + kLo + j * kOpKCoreBytes) = l0;
      *reinterpret_cast<uint32_t*>(op_t + kLo + j * kOpKCoreBytes + 8 * 16) = l1;
    }
  }
}

// Can step `ed` run its epilogue in registers?  (Its halves are N = 128 whenever ed.n = 256 and ed.n0 = 128.)
__device__ __forceinline__ bool trunk_in_regs(const EpiDesc& ed) {
  return ed.kind == EPI_RELU_TO_A && !ed.sigma && ed.n == 256 && ed.n0 == 128 && ed.dst_col == kColAHi &&
         ed.dst_lo_col == kColALo;
}

// Accumulator columns [c_base, c_base + n_h) of the step held in `d` (wgmma fragment: thread t of warp w holds rows
// 16w + t/4 and 16w + t/4 + 8, columns 8j + 2(t%4) + {0, 1} in d[4j .. 4j+3]) -> the staging tile, for the columns
// that fall into the window [w0, w0 + 128).
__device__ __forceinline__ void stage_acc(const float (&d)[64], int c_base, int n_h, int w0, float* stg, int warp, int lane) {
  const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = c_base + 8 * j + 2 * (lane & 3) - w0;
    if (8 * j < n_h && c >= 0 && c < 128) {
      *reinterpret_cast<float2*>(stg + r0 * kStageLd + c) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * kStageLd + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  }
}

// Ablation builds (timing only, garbage outputs): the weight stream alone; no embeddings; no epilogue math or stores on
// the trunk steps (the staged path with its barriers, forward kernels).  (Skipping every epilogue is no ablation: with
// no accumulator ever read, ptxas serializes the wgmmas.)
#ifdef PNR_ABL_STREAM_ONLY
constexpr bool kStreamOnly = true;
#else
constexpr bool kStreamOnly = false;
#endif
#ifdef PNR_ABL_NO_PROLOGUE
constexpr bool kAblNoPrologue = true;
#else
constexpr bool kAblNoPrologue = false;
#endif
#ifdef PNR_ABL_NO_TRUNK_EPILOGUE
constexpr bool kAblNoTrunkEpi = true;
#else
constexpr bool kAblNoTrunkEpi = false;
#endif

// Embeddings of the tile from s_base: threads 0-63 gamma(x) of row t, threads 64-127 gamma(d) of row t - 64.  A
// hash-grid trunk input (p.hash_table set) replaces gamma(x) by h(x): both threads of a row form its point, the xyz
// thread gathers the first half of the feature core rows, the dir thread (after gamma(d), if any) the second half.
template <int PASSES, int FMT, bool BWD>
__device__ __forceinline__ void tile_prologue(const MlpParams& p, const MlpProgram& prog, uint8_t* smem, int64_t s_base,
                                              uint32_t& vmax) {
  named_bar_sync(1, kConsumerThreads);    // the previous tile's end-of-tile reads are done
  const int erow = threadIdx.x & (kRows - 1);
  const bool dir_thread = threadIdx.x >= kRows;
  const bool hashgrid = p.hash_table != nullptr;
  if (!kAblNoPrologue && (!(BWD && dir_thread) || hashgrid)) {
    int64_t se = s_base + erow;
    if (se >= p.S) se = p.S - 1;  // clamp: tail rows compute on a valid sample, results are discarded
    float x[3], d[3];
    if (p.pts != nullptr) {
#pragma unroll
      for (int c = 0; c < 3; ++c) { x[c] = p.pts[se * 3 + c]; d[c] = BWD ? 0.f : p.viewdirs[se * 3 + c]; }
    } else {
      const int64_t ray = se / p.N;
      const float zi = p.z[se];
      const float* rr = p.rays + ray * 6;
      float dn2 = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float dc = rr[3 + c];
        x[c] = __fadd_rn(rr[c], __fmul_rn(dc, zi));  // pts = o + d*z, separately rounded like the oracle
        dn2 = (c == 0) ? __fmul_rn(dc, dc) : __fadd_rn(dn2, __fmul_rn(dc, dc));
        d[c] = dc;
      }
      const float nrm = sqrtf(dn2);
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c] = __fdiv_rn(d[c], nrm);
    }
    if (dir_thread) {
      if (!BWD) encode_row<PASSES, FMT, 4, 32>(d, prog.Ld, smem + kSmemDir, smem + kSmemDir + kDirPartBytes, erow, vmax);
    } else if (!hashgrid) {
      encode_row<PASSES, FMT, 10, 64>(x, prog.Lx, smem + kSmemEmb, smem + kSmemEmb + kEmbPartBytes, erow, vmax);
    }
    if (hashgrid) {
      // a non-finite point is flagged here: the clamp below sends a NaN to the corner (0,0,0), whose features are
      // finite (the clamp stays: a NaN must never become a table index)
      if (!(isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]))) vmax |= 0xFFFFu;
      float v[3];
      hash_normalize(x, p.hash_aabb, v);
      const int nc = ((p.hash_L * p.hash_F + 15) & ~15) / 8, half = (nc + 1) / 2;   // core rows the MMAs read
      hash_rows_f<PASSES, FMT>(p, v, dir_thread ? half : 0, dir_thread ? nc : half, smem + kSmemEmb,
                               smem + kSmemEmb + kEmbPartBytes, erow, vmax);
    }
  }
  fence_proxy_async_smem();   // generic-proxy stores -> visible to the MMAs' async proxy
  named_bar_sync(1, kConsumerThreads);
}

// The MMAs of step `ed` from stage si on: its stages up to the one that closes it, those of the first half (accumulator
// column ed.acc_col) into acc0, the rest into acc1; a ring slot is released when the MMAs that read it have retired.
// Returns the next step's first stage.
template <int PASSES, int FMT>
__device__ __forceinline__ int step_mmas(float (&acc0)[64], float (&acc1)[64], const MlpProgram& prog, const EpiDesc& ed,
                                         int si, uint32_t ring_s, uint32_t bar_full, uint32_t bar_empty, uint32_t emb_s,
                                         uint32_t dir_s, uint32_t op_s, RingPos& rp, bool leader) {
  int h1 = si, end = si;
  for (;;) {
    const uint32_t flags = prog.st[end].flags;
    if (prog.st[end].acc_col == ed.acc_col) h1 = end + 1;
    ++end;
    if (flags & (F_COMMIT_ACC1 | F_COMMIT_VIEW)) break;
  }
  // each half's first stage (F_FIRST) overwrites its accumulator, so the old values are dead: clearing them (before
  // any of the step's wgmmas) says so to the compiler, which can then use those registers between steps without moving
  // live accumulators - a move in a divergent path would serialize every wgmma
#pragma unroll
  for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.f;
  mma_half_n<PASSES, FMT>(acc0, prog.st[si].n, prog, si, h1, ring_s, bar_full, bar_empty, emb_s, dir_s, op_s, rp, leader);
  if (h1 < end)
    mma_half_n<PASSES, FMT>(acc1, prog.st[h1].n, prog, h1, end, ring_s, bar_full, bar_empty, emb_s, dir_s, op_s, rp, leader);
  return end;
}

// A trunk step's epilogue in registers: both halves through epi_regs_act (bias_t, op_t as there) between two barriers.
template <int PASSES, int FMT>
__device__ __forceinline__ void trunk_epilogue(const float (&acc0)[64], const float (&acc1)[64], const float* bias_t,
                                               uint8_t* op_t, uint32_t& vmax) {
  named_bar_sync(1, kConsumerThreads);   // every warp's MMAs of the step have retired: its input is dead
  epi_regs_act<PASSES, FMT, 0>(acc0, bias_t, op_t, vmax);
  epi_regs_act<PASSES, FMT, 1>(acc1, bias_t, op_t, vmax);
  fence_proxy_async_smem();              // the next step's MMAs read what was just stored
  named_bar_sync(1, kConsumerThreads);
}

// End of a COMP tile (one warp, lanes stride channels): fold its per-quarter sums (qsum half `par`) into the open ray's
// running sums racc, in ray order; a ray is written out when the next one starts or the CTA's range ends.
__device__ __forceinline__ void comp_flush_tile(const MlpParams& p, float* racc, const float* qsum, int nch, int par,
                                                int64_t s_base, int64_t s_end, int64_t cta_first, int lane) {
  auto flush = [&](int64_t r) {
    const float depth = racc[3], acc = racc[4];
    __syncwarp();
    for (int c = lane; c < nch; c += 32) {
      const float v = racc[c];
      if (c < 3) { if (p.rgb_map) p.rgb_map[r * 3 + c] = v + (p.white_bkgd ? (1.0f - acc) : 0.f); }
      else if (c == 3) {
        if (p.depth_map) p.depth_map[r] = v;
        if (p.disp_map) p.disp_map[r] = comp_disp(depth, acc);
      }
      else if (c == 4) { if (p.acc_map) p.acc_map[r] = v; }
      else if (c < 5 + p.C) { if (p.sem_map) p.sem_map[r * p.C + (c - 5)] = v; }
      else { if (p.inst_map) p.inst_map[r * p.K + (c - 5 - p.C)] = v; }
      racc[c] = 0.f;
    }
    __syncwarp();
  };
#pragma unroll 1
  for (int qq = 0; qq < kQuarters; ++qq) {
    const int64_t sq = s_base + 32 * qq;
    if (sq >= s_end) break;
    if (sq > cta_first && sq % p.N == 0) flush(sq / p.N - 1);    // the previous ray ended right before sq
    const float* src = qsum + (par * kQuarters + qq) * kCompChPad;
    for (int c = lane; c < nch; c += 32) racc[c] += src[c];
    __syncwarp();
  }
  if (s_base < s_end && s_base + kRows >= s_end) flush(s_end / p.N - 1);   // the CTA's last ray
}

// COMP = false: tiles are dealt round-robin to the CTAs and the network outputs go to `raw`.
// COMP = true : every CTA owns a contiguous range of whole rays and walks it tile by tile; the epilogue composites
// on chip - per-sample alpha / transmittance / weight right after the sigma-producing layer (warp scan over aligned
// groups of 32 samples, carried across groups and tiles through shared memory), logits and colours reduced per group
// with a fixed shuffle tree and accumulated per ray in ray order - and only weights and the per-ray maps leave the
// SM: `raw` (456 B per sample with both heads) is never written.
//
// BWD = true  : the program is a backward program (mlp_program.h): the forward trunk with its ReLU sign patterns kept
// in shared memory, then the layers in reverse with transposed weights; input `grad_in`, output `raw`.
template <int PASSES, int FMT, bool COMP, bool BWD = false>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_fused_kernel(const __grid_constant__ MlpLaunch L) {
  static_assert(!(COMP && BWD), "the compositing epilogue belongs to forward programs");
  extern __shared__ __align__(1024) uint8_t smem[];
  const MlpParams& p = L.p;
  const MlpProgram& prog = L.prog;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_iter = COMP ? (int)((p.rays_per_cta * p.N + kRows - 1) / kRows)
                          : (p.num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  // first sample of this CTA's tile `it`, and the end of the samples it owns
  auto cta_first = [&]() -> int64_t { return COMP ? (int64_t)blockIdx.x * p.rays_per_cta * p.N : 0; };
  auto tile_base = [&](int it) -> int64_t {
    return COMP ? cta_first() + (int64_t)it * kRows : (int64_t)((int)blockIdx.x + it * (int)gridDim.x) * kRows;
  };
  auto cta_end = [&]() -> int64_t {
    if (!COMP) return p.S;
    const int64_t e = cta_first() + p.rays_per_cta * p.N;
    return e < p.S ? e : p.S;
  };

  const float* consts = p.consts;   // (read through L1: a few KB, the same words for every tile)
  float* part = reinterpret_cast<float*>(smem + kSmemPart);   // [2 column shares][kRows][4]: partial sigma / rgb sums
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kSmemBars);
  const uint32_t bar_full = smem_u32(&bars[0]);          // [kSlots] weight slot landed
  const uint32_t bar_empty = smem_u32(&bars[kSlots]);    // [kSlots] its MMAs retired (one arrival per consumer warp)
  uint32_t* absmax = reinterpret_cast<uint32_t*>(bars + 2 * kSlots);   // BWD: [kMaxSteps] this CTA's stash maxima
  static_assert(2 * kSlots * 8 + kMaxSteps * 4 <= 256, "barrier area");
  const uint32_t ring_s = smem_u32(smem + kSmemRing);

  if (BWD) for (int i = threadIdx.x; i < kMaxSteps; i += blockDim.x) absmax[i] = 0u;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kSlots; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kConsumerThreads / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int n_stages = prog.n_stages, n_steps = prog.n_steps;

  if (warp == kConsumerThreads / 32) {
    // =============================================================== weight stream (one elected thread)
    if (elect_one()) {
      uint32_t gs = 0;  // global slot counter
      for (int it = 0; it < n_iter; ++it) {
        for (int si = 0; si < n_stages; ++si) {
          const StageDesc& sd = prog.st[si];
          const uint32_t step_bytes = (uint32_t)sd.n * 32u;   // one K16 step of one image
          const int nslots = stage_slots(sd);
          for (int j = 0; j < nslots; ++j, ++gs) {
            int k0, kn;
            slot_ksteps(sd, j, k0, kn);
            const uint32_t slot = ring_slot(gs), ph = ring_phase(gs);
            const uint32_t part = (uint32_t)kn * step_bytes;   // bytes of one image in this slot
            const uint32_t dst = ring_s + slot * (uint32_t)kSlotBytes, bar = bar_full + 8 * slot;
            const uint8_t* hi = p.wpacked + sd.gofs + (uint32_t)k0 * step_bytes;
            const uint8_t* lo = p.wpacked + sd.gofs + (uint32_t)sd.lo_off16 * 16u + (uint32_t)k0 * step_bytes;
            mbar_wait_backoff(bar_empty + 8 * slot, ph ^ 1);
            mbar_arrive_expect_tx(bar, PASSES == 3 ? 2 * part : part);
            bulk_g2s(dst, hi, part, bar);
            if (PASSES == 3) bulk_g2s(dst + part, lo, part, bar);
          }
        }
      }
    }
  } else {
    // =============================================================== consumer warpgroup
    const int q = warp & 1, ch = warp >> 1;     // 32-row group (a "quarter" of the compositing code) ; column share
    const int row = q * 32 + lane;
    uint8_t* op = smem + kSmemOp;
    uint8_t* op_t = op + (warp * 16 + (lane >> 2)) * 16 + (lane & 3) * 4;   // this thread's word of a trunk epilogue
    float* stg = reinterpret_cast<float*>(smem + kSmemStage);
    const uint32_t op_s = smem_u32(op), emb_s = smem_u32(smem + kSmemEmb), dir_s = smem_u32(smem + kSmemDir);
    RingPos rp{0u, -1};
    uint32_t vmax = 0;                         // largest hi-part bit patterns this thread produced (16x2)
    float acc0[64], acc1[64];                   // the step's two N-halves
    // compositing state (COMP): see mlp_program.h for the shared-memory map
    float* w_row = reinterpret_cast<float*>(smem + kSmemCompW);
    float* qprod = reinterpret_cast<float*>(smem + kSmemCompQ);   // [2][kQuarters]
    float* carry = qprod + 2 * kQuarters;                          // [2]
    float* qsum = reinterpret_cast<float*>(smem + kSmemCompS);     // [2][kQuarters][kCompChPad]
    float* racc = reinterpret_cast<float*>(smem + kSmemCompR);     // [kCompChPad]
    const int nch = 5 + p.C + p.K;
    if (COMP) {
      for (int c = threadIdx.x; c < kCompChPad; c += kConsumerThreads) racc[c] = 0.f;
      if (threadIdx.x == 0) carry[0] = 1.0f;
    }
    for (int it = 0; it < n_iter; ++it) {
      const int64_t s_base = tile_base(it);
      const int64_t s = s_base + row;
      const int64_t s_end = cta_end();
      const bool valid = s < s_end;
      if (kStreamOnly || s_base >= s_end) {
        // no sample of this CTA in the tile: take the weight slots, compute nothing
#pragma unroll 1
        for (int si = 0; si < n_stages; ++si) {
#pragma unroll 1
          for (int j = 0; j < stage_slots(prog.st[si]); ++j, ++rp.gs) {
            mbar_wait(bar_full + 8 * ring_slot(rp.gs), ring_phase(rp.gs));
            release_slot(bar_empty, (int)ring_slot(rp.gs), lane == 0);
          }
        }
        continue;
      }
      const int par = it & 1;
      float* qsum_q = qsum + (par * kQuarters + q) * kCompChPad;     // this quarter's partial sums of this tile
      float w_mine = 0.f;                                            // this row's compositing weight (COMP)
      float sig = 0.f;

      tile_prologue<PASSES, FMT, BWD>(p, prog, smem, s_base, vmax);
      int si = 0;
      for (int st = 0; st < n_steps; ++st) {
        const EpiDesc ed = prog.ep[st];
        si = step_mmas<PASSES, FMT>(acc0, acc1, prog, ed, si, ring_s, bar_full, bar_empty, emb_s, dir_s, op_s, rp, lane == 0);
        if (!BWD && !kAblNoTrunkEpi && trunk_in_regs(ed)) {
          trunk_epilogue<PASSES, FMT>(acc0, acc1, consts + ed.bias_off + 2 * (lane & 3), op_t, vmax);
          continue;
        }

        // ---- epilogue: accumulator columns [0, n0) are in acc0, [n0, n) in acc1
        const float* bias = consts + ed.bias_off;
        const float* aux = consts + ed.aux_off;
        const bool to_a = BWD ? epi_writes_a(ed.kind) : ed.kind == EPI_RELU_TO_A;
        const int ng = ed.n >> 4;
        float c0 = 0.f, c1 = 0.f, c2 = 0.f;
        uint32_t smax = 0;   // backward programs: largest hi-part magnitudes of the A operand this step produces (16x2)
        // backward programs: this row's sign patterns and its row of the incoming gradient (tail rows read row S-1)
        uint16_t* mask_row = reinterpret_cast<uint16_t*>(smem + kSmemMask) + row;
        const float* gin = (BWD && ed.kind == EPI_LOADG_TO_A) ? p.grad_in + (valid ? s : p.S - 1) * (int64_t)ed.n : nullptr;
        float* stash_row = (BWD && p.stash != nullptr && ed.out_off1 != 0 && valid)
                               ? p.stash + ((int64_t)(ed.out_off1 - 1) * p.S + s) * (int64_t)ed.n : nullptr;
        if (BWD && st == 0 && p.grad_in != nullptr) {   // this row of the incoming gradient is needed D-1 steps from now: bring it into L2
          const float* g0 = p.grad_in + (valid ? s : p.S - 1) * (int64_t)prog.ep[0].n;
          for (int c = ch * 32; c < (int)prog.ep[0].n; c += 2 * 32) prefetch_l2(g0 + c);
        }
        for (int w0 = 0; w0 < (int)ed.n; w0 += 128) {
          if (kAblNoTrunkEpi && !BWD && trunk_in_regs(ed)) {
            named_bar_sync(1, kConsumerThreads);
            named_bar_sync(1, kConsumerThreads);
            continue;
          }
          stage_acc(acc0, 0, ed.n0, w0, stg, warp, lane);
          if (ed.n0 < ed.n) stage_acc(acc1, ed.n0, ed.n - ed.n0, w0, stg, warp, lane);
          named_bar_sync(1, kConsumerThreads);
          // this thread's share of the window's 16-column groups: share 0 the first half, share 1 the rest
          const int g_lo = w0 >> 4, g_hi = (ng < g_lo + 8) ? ng : g_lo + 8, g_mid = g_lo + (g_hi - g_lo + 1) / 2;
          const int ga = ch == 0 ? g_lo : g_mid, gb = ch == 0 ? g_mid : g_hi;
#pragma unroll 1
          for (int g = ga; g < gb; ++g) {
            uint32_t r[16];
            const float4* src = reinterpret_cast<const float4*>(stg + row * kStageLd + (g * 16 - w0));
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float4 v = src[k];
              r[4 * k] = __float_as_uint(v.x); r[4 * k + 1] = __float_as_uint(v.y);
              r[4 * k + 2] = __float_as_uint(v.z); r[4 * k + 3] = __float_as_uint(v.w);
            }
            if (to_a) {
              uint32_t hi[8], lo[8];
              if (BWD) epi_group_bwd<PASSES, FMT>(r, g, ed, bias, mask_row, gin, stash_row, p.grad_scale, p.grad_unscale, smax, hi, lo);
              else epi_group_act<PASSES, FMT>(r, g, ed, bias, aux, sig, vmax, hi, lo);
              epi_group_store<PASSES>(g, ed, op, row, hi, lo);
            } else {
              // EPI_LOGITS: where this group's columns go (the columns from n0 on may be a logit layer of its own)
              const bool own_half = !BWD && ed.n_valid1 > 0 && g * 16 >= (int)ed.n0;
              float* out_row = p.raw + (valid ? s : 0) * p.CH + (own_half ? ed.out_off1 : ed.out_off);
              const int out_c0 = own_half ? (int)ed.n0 : 0, out_valid = own_half ? (int)ed.n_valid1 : (int)ed.n_valid;
              const int out_ch = (own_half ? (int)ed.out_off1 : (int)ed.out_off) + 1;   // composited channel of column out_c0
              const bool out_vec = BWD && (p.CH & 3) == 0 && (int)ed.n <= p.CH && (reinterpret_cast<uintptr_t>(p.raw) & 15) == 0 &&
                                   (ed.out_off & 3) == 0;
              if (BWD) {
                if (valid && ed.kind == EPI_ACT_OUT) epi_group_actout(r, g, bias, out_row);
                else if (valid) epi_group_gradout(r, g, ed.n_valid, ed.n_valid1 != 0, out_vec, p.grad_unscale, out_row);
              } else if (ed.kind == EPI_VIEW_RGB) {
                epi_group_rgb(r, g, ed, bias, aux, c0, c1, c2);
              } else if (COMP) {
                epi_group_logits_comp(r, g, out_c0, out_valid, out_ch, bias, w_mine, lane, qsum_q);
              } else if (valid) {
                epi_group_logits(r, g, out_c0, out_valid, bias, out_row);
              }
            }
          }
          if (to_a) fence_proxy_async_smem();   // the next step's MMAs read what was just stored
          named_bar_sync(1, kConsumerThreads);  // (and the staging tile is free again)
        }
        if (!BWD) {
          if (ed.sigma) {
            part[(ch * kRows + row) * 4 + 3] = sig;
            sig = 0.f;
          }
          if (ed.kind == EPI_VIEW_RGB) {
            float* mine = part + (ch * kRows + row) * 4;
            mine[0] = c0; mine[1] = c1; mine[2] = c2;
            named_bar_sync(1, kConsumerThreads);
            if (ch == 0 && (COMP || valid)) {
              const float* b3 = consts + prog.rgb_bias_off;
              const float* other = part + (kRows + row) * 4;   // fixed order: deterministic sums
              float o0 = c0 + other[0], o1 = c1 + other[1], o2 = c2 + other[2], o3 = mine[3] + other[3];
              o0 += b3[0]; o1 += b3[1]; o2 += b3[2]; o3 += consts[prog.sigma_bias_off];
              if (COMP) {   // colours weighted and summed over this aligned group of 32 samples (w = 0 on dummy rows)
                const float r0 = warp_sum32(w_mine * comp_sigmoid(o0));
                const float r1 = warp_sum32(w_mine * comp_sigmoid(o1));
                const float r2 = warp_sum32(w_mine * comp_sigmoid(o2));
                if (lane == 0) { qsum_q[0] = r0; qsum_q[1] = r1; qsum_q[2] = r2; }
              } else {
                float* dst = p.raw + s * p.CH;
                if (p.CH == 4) {
                  *reinterpret_cast<float4*>(dst) = make_float4(o0, o1, o2, o3);
                } else {
                  dst[0] = o0; dst[1] = o1; dst[2] = o2; dst[3] = o3;
                }
              }
            }
          }
        }
        if (BWD) {
          vmax = __vimax3_u16x2(vmax, smax, 0u);          // the range check sees every step
          if (p.stash_absmax != nullptr && to_a && ed.out_off1 != 0) {   // per-step maximum of what went to the stash
            uint32_t m = smax & 0xFFFFu;
            if ((smax >> 16) > m) m = smax >> 16;
            m = __reduce_max_sync(0xffffffffu, m);
            if (lane == 0) atomicMax(absmax + st, m);
          }
        }
        if (COMP && ed.sigma) {
          // ---- per-sample weights of this tile, right after the sigma-producing layer.  sigma = the two column
          // shares' partial dot products + bias, in the order the raw-writing kernel uses.  One warp per quarter =
          // one aligned group of 32 samples.
          named_bar_sync(1, kConsumerThreads);          // both shares of every row's sigma are in shared memory
          if (ch == 0) {
            const int64_t sq = s_base + q * 32;         // first sample of this quarter; live or dummy as a whole
            const bool live = sq < s_end;
            float alpha = 0.f, zi = 0.f, t = 1.0f;
            if (live) {
              const int64_t r = sq / p.N;
              const int i = (int)(sq - r * p.N) + lane;
              zi = p.z[sq + lane];
              const bool has_next = i + 1 < p.N;
              const float z_next = has_next ? p.z[sq + lane + 1] : 0.f;
              const float* rr = p.rays + r * 6;
              const float dist = comp_dist(zi, z_next, has_next, comp_dnorm(rr[3], rr[4], rr[5]));
              float sraw = part[row * 4 + 3];
              sraw += part[(kRows + row) * 4 + 3];
              sraw += consts[prog.sigma_bias_off];
              const bool masked = p.mask_outside && p.sample_box != nullptr && p.sample_box[sq + lane] < 0;
              alpha = comp_alpha(sraw, dist, masked);
              t = 1.0f - alpha + 1e-10f;
            }
            float total;
            const float excl = comp_scan32(t, lane, &total);
            if (lane == 0) qprod[par * kQuarters + q] = total;
            named_bar_sync(3, kQuarters * 32);          // the quarter products
            // transmittance at this quarter's first sample: carried in from the previous tile, restarted where a
            // ray starts, multiplied through the earlier quarters in order (the order is fixed by the sample index)
            float prefix = carry[par];
#pragma unroll
            for (int qq = 0; qq < kQuarters; ++qq) {
              if (qq <= q) {
                if ((s_base + 32 * qq) % p.N == 0) prefix = 1.0f;
                if (qq < q) prefix *= qprod[par * kQuarters + qq];
              }
            }
            const float wi = live ? alpha * (prefix * excl) : 0.f;
            w_row[row] = wi;
            if (live) p.weights[sq + lane] = wi;
            const float sd = warp_sum32(wi * zi), sa = warp_sum32(wi);
            if (lane == 0) {
              qsum_q[3] = sd;
              qsum_q[4] = sa;
              if (q == kQuarters - 1) carry[par ^ 1] = prefix * total;   // transmittance behind the tile's last sample
            }
          }
          named_bar_sync(1, kConsumerThreads);          // w_row is visible to both column shares
          w_mine = w_row[row];
        }
      }
      if (COMP) {
        named_bar_sync(1, kConsumerThreads);            // every quarter's partial sums are in shared memory
        if (warp == 0) comp_flush_tile(p, racc, qsum, nch, par, s_base, s_end, cta_first(), lane);
      }
    }
    if (p.status != nullptr && ((vmax & 0xFFFFu) >= inf_bits16<FMT>() || (vmax >> 16) >= inf_bits16<FMT>()))
      atomicOr(p.status, 1u);
  }
  __syncthreads();
  if (BWD && p.stash_absmax != nullptr && (int)threadIdx.x < prog.n_steps) {   // this CTA's maxima -> the launch's
    const EpiDesc& e = prog.ep[threadIdx.x];
    const uint32_t m = absmax[threadIdx.x];
    if (epi_writes_a(e.kind) && e.out_off1 != 0 && m != 0u) atomicMax(p.stash_absmax + (e.out_off1 - 1), m);
  }
}

template <int PASSES, int FMT, bool COMP, bool BWD = false>
static int launch_one(const MlpLaunch& L, int dev, int grid, cudaStream_t stream) {
  constexpr int kSmem = COMP ? kSmemTotalComp : kSmemTotal;
  const int rc = opt_in_smem((const void*)mlp_fused_kernel<PASSES, FMT, COMP, BWD>, kSmem, dev);
  if (rc != PNR_OK) return rc;
  mlp_fused_kernel<PASSES, FMT, COMP, BWD><<<grid, kMlpThreads, kSmem, stream>>>(L);
  PNR_LAUNCH_CHECK("mlp_fused_kernel");
  return PNR_OK;
}

// Launches on the CURRENT device (the caller has made the context's device current).  mode 1: the
// compositing-epilogue variant; the launch's rays_per_cta is set here (whole rays per CTA, so that every CTA's range
// starts on a 32-sample boundary).  mode 2: L.prog is a backward program (x3 precisions only).
int launch_mlp(MlpLaunch& L, int passes, int fmt, int mode, cudaStream_t stream) {
  const bool composite = mode == kMlpComposite;
  int dev = 0;
  const int rc = current_device("launch_mlp", &dev);
  if (rc != PNR_OK) return rc;
  const int sms = num_sms(dev);
  const int64_t tiles = (L.p.S + kRows - 1) / kRows;
  PNR_CHECK_ARG(tiles < ((int64_t)1 << 31), "launch_mlp: too many samples");
  L.p.num_tiles = (int32_t)tiles;
  const int grid = L.p.num_tiles < sms ? L.p.num_tiles : sms;
  if (grid <= 0) return PNR_OK;
  if (composite) {
    const int64_t R = L.p.S / L.p.N;
    L.p.rays_per_cta = (R + grid - 1) / grid;
  }
  if (mode == kMlpBackward) {
    if (passes != 3) return set_error(PNR_ERR_UNSUPPORTED, "backward programs run in the x3 precisions only");
    return fmt == kFmtF16 ? launch_one<3, kFmtF16, false, true>(L, dev, grid, stream)
                          : launch_one<3, kFmtBF16, false, true>(L, dev, grid, stream);
  }
#define PNR_LAUNCH(P, F) (composite ? launch_one<P, F, true>(L, dev, grid, stream) : launch_one<P, F, false>(L, dev, grid, stream))
  if (fmt == kFmtF16) return passes == 3 ? PNR_LAUNCH(3, kFmtF16) : PNR_LAUNCH(1, kFmtF16);
  return passes == 3 ? PNR_LAUNCH(3, kFmtBF16) : PNR_LAUNCH(1, kFmtBF16);
#undef PNR_LAUNCH
}

}  // namespace pnr
