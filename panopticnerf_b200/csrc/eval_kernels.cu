// eval_kernels.cu — evaluation of rendered frames against their ground truth (the step after panoptic fusion):
//   * semantic confusion matrix (mIoU, pixel accuracy): per-block shared-memory histogram, integer flush,
//   * panoptic quality (PQ / SQ / RQ): (gt id, pred id) pair histogram in an open-addressing table, segment areas and
//     void / crowd overlaps derived from it, matching and per-channel tallies,
//   * image and depth error sums (PSNR, MAE / RMSE / abs-rel): fixed-shape double reductions.
// The reference's evaluator is not in the mount: the metric rules are chosen here (include/pnr.h, DESIGN.md 3.4) and
// restated on the CPU in oracle/reference_eval.py, which the kernels are held to.
//
// Determinism: every count is an integer atomic (order-free, exact).  The matched IoUs of a frame are summed EXACTLY:
// a correctly rounded double IoU in (0.5, 1] is an integer multiple of 2^-53, so each one is added as that integer to a
// 128-bit per-channel accumulator and the frame's sum is rounded to double once (= math.fsum of the frame's IoUs).  No
// float atomics anywhere, and no sort: the result cannot depend on the order the pairs are visited in.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include "../../include/pnr.h"
#include "common.cuh"

namespace pnr {
namespace {

constexpr int kEvalMaxClasses = 64;
constexpr int kThreads = 256;
constexpr uint32_t kVoidId = 0xFFFFFFFFu;              // empty segment slot / void side of a pair (ids are >= 0)
constexpr unsigned long long kEmptyPair = ~0ull;       // (void, void): never inserted
constexpr int kImageBlocks = 256;                      // fixed grid of the image reduction (fixed summation tree)
constexpr int kImageSums = 6;

// dataset id p / 1000 -> class channel in [0, C), or -1 (void): negative ids, ids past the table, table entries
// outside [0, C); without a table the dataset id is the channel when it is below C
struct IdMap {
  const int32_t* table; int32_t n_ids; int32_t C;
};
__device__ __forceinline__ int channel_of(int32_t id, const IdMap& m) {
  if (id < 0) return -1;
  const int32_t d = id / 1000;
  if (m.table == nullptr) return d < m.C ? d : -1;
  if (d >= m.n_ids) return -1;
  const int32_t c = __ldg(m.table + d);
  return (c >= 0 && c < m.C) ? c : -1;
}

int grid_for(int64_t work) {
  const int64_t b = (work + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)num_sms() * 8;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

// ------------------------------------------------------------------------------------------------ semantic
// conf [C, C+1] += pixels with gt channel g (non-void) and prediction channel p (column C: void / unmapped).  One
// grid-stride pass; a warp adds equal bins once (__match_any_sync); the block's uint32 histogram is flushed with one
// 64-bit atomic per non-zero bin.  A block sees fewer than 2^31 pixels (n < 2^31), so its bins cannot wrap.
__global__ void __launch_bounds__(kThreads) eval_semantic_kernel(const int32_t* __restrict__ pred,
                                                                 const int32_t* __restrict__ gt, int64_t n, IdMap m,
                                                                 unsigned long long* conf) {
  extern __shared__ uint32_t hist[];
  const int bins = m.C * (m.C + 1);
  for (int i = threadIdx.x; i < bins; i += blockDim.x) hist[i] = 0u;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x - lane; i0 < n; i0 += stride) {   // warp-uniform
    const int64_t i = i0 + lane;
    int bin = -1;
    if (i < n) {
      const int g = channel_of(gt[i], m);
      if (g >= 0) {
        const int p = channel_of(pred[i], m);
        bin = g * (m.C + 1) + (p < 0 ? m.C : p);
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(hist + bin, (uint32_t)__popc(peers));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bins; i += blockDim.x)
    if (hist[i] != 0u) atomicAdd(conf + i, (unsigned long long)hist[i]);
}

// ------------------------------------------------------------------------------------------------ panoptic
// Workspace: three open-addressing tables of S slots each (S = a power of two >= 2n: at most n keys go into any of
// them, so none is ever more than half full and every probe ends):
//   pairs    key (gt id or void) << 32 | (pred id or void) -> pixel count
//   gt segs  gt id   -> area, matched
//   pr segs  pred id -> area, |p ∩ void|, |p ∩ crowd of its class|, matched
// then the 128-bit IoU accumulators [C][2] (lo, hi) of the frame.
struct PanTables {
  uint32_t mask;                                   // S - 1
  unsigned long long* pair_key; uint32_t* gt_key; uint32_t* pr_key;         // cleared to all-ones
  uint32_t* pair_cnt; uint32_t* gt_area; uint32_t* gt_matched;              // cleared to zero ...
  uint32_t* pr_area; uint32_t* pr_void; uint32_t* pr_crowd; uint32_t* pr_matched;
  unsigned long long* iou_acc;
};

struct PanArgs {
  const int32_t* pred; const int32_t* gt; int64_t n; IdMap m; const uint8_t* is_thing;
  PanTables t;
  unsigned long long* tp; unsigned long long* fp; unsigned long long* fn; double* iou_sum;
};

__device__ __forceinline__ uint32_t mix64(unsigned long long k) {   // murmur3 finaliser
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (uint32_t)k;
}

// Slot of `key`, inserted if absent.  A non-empty slot never changes, so a key read through L2 is final; an empty one
// is claimed with atomicCAS, whose return value decides.
template <class Key>
__device__ __forceinline__ uint32_t slot_of(Key* keys, uint32_t mask, Key key, Key empty) {
  uint32_t s = mix64((unsigned long long)key) & mask;
  while (true) {
    Key k = __ldcg(keys + s);
    if (k == empty) k = atomicCAS(keys + s, empty, key);
    if (k == empty || k == key) return s;
    s = (s + 1u) & mask;
  }
}

// Slot of a key known to be present.
template <class Key>
__device__ __forceinline__ uint32_t find_slot(const Key* keys, uint32_t mask, Key key) {
  uint32_t s = mix64((unsigned long long)key) & mask;
  while (keys[s] != key) s = (s + 1u) & mask;
  return s;
}

__device__ __forceinline__ bool is_crowd(int32_t id, int c, const uint8_t* is_thing) {
  return c >= 0 && is_thing[c] != 0 && id % 1000 == 0;
}

__global__ void __launch_bounds__(kThreads) eval_pairs_kernel(PanArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x - lane; i0 < a.n; i0 += stride) {
    const int64_t i = i0 + lane;
    unsigned long long key = kEmptyPair;
    if (i < a.n) {
      const int32_t g = a.gt[i], p = a.pred[i];
      const uint32_t gk = channel_of(g, a.m) < 0 ? kVoidId : (uint32_t)g;
      const uint32_t pk = channel_of(p, a.m) < 0 ? kVoidId : (uint32_t)p;
      key = ((unsigned long long)gk << 32) | pk;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key != kEmptyPair && lane == __ffs(peers) - 1)
      atomicAdd(a.t.pair_cnt + slot_of(a.t.pair_key, a.t.mask, key, kEmptyPair), (uint32_t)__popc(peers));
  }
}

// per pair: gt area, pred area, the pred's void and same-class crowd overlaps
__global__ void __launch_bounds__(kThreads) eval_segments_kernel(PanArgs a) {
  const PanTables& t = a.t;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= t.mask; s += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = t.pair_key[s];
    if (key == kEmptyPair) continue;
    const uint32_t cnt = t.pair_cnt[s];
    const uint32_t gk = (uint32_t)(key >> 32), pk = (uint32_t)key;
    if (gk != kVoidId) atomicAdd(t.gt_area + slot_of(t.gt_key, t.mask, gk, kVoidId), cnt);
    if (pk != kVoidId) {
      const uint32_t ps = slot_of(t.pr_key, t.mask, pk, kVoidId);
      atomicAdd(t.pr_area + ps, cnt);
      if (gk == kVoidId) {
        atomicAdd(t.pr_void + ps, cnt);
      } else {
        const int cg = channel_of((int32_t)gk, a.m);
        if (is_crowd((int32_t)gk, cg, a.is_thing) && cg == channel_of((int32_t)pk, a.m)) atomicAdd(t.pr_crowd + ps, cnt);
      }
    }
  }
}

// per pair of the same channel (crowd excluded): IoU = inter / (area_p + area_g - inter - |p ∩ void|) > 0.5 is a match
// (2 inter > union in integers; at most one per segment on either side).  tp += 1, IoU added exactly (see the top).
__global__ void __launch_bounds__(kThreads) eval_match_kernel(PanArgs a) {
  const PanTables& t = a.t;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= t.mask; s += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = t.pair_key[s];
    if (key == kEmptyPair) continue;
    const uint32_t gk = (uint32_t)(key >> 32), pk = (uint32_t)key;
    if (gk == kVoidId || pk == kVoidId) continue;
    const int c = channel_of((int32_t)gk, a.m);
    if (c != channel_of((int32_t)pk, a.m) || is_crowd((int32_t)gk, c, a.is_thing)) continue;
    const uint64_t inter = t.pair_cnt[s];
    const uint32_t gs = find_slot(t.gt_key, t.mask, gk), ps = find_slot(t.pr_key, t.mask, pk);
    const uint64_t uni = (uint64_t)t.pr_area[ps] + t.gt_area[gs] - inter - t.pr_void[ps];
    if (2 * inter <= uni) continue;
    t.gt_matched[gs] = 1u;
    t.pr_matched[ps] = 1u;
    atomicAdd(a.tp + c, 1ull);
    const double iou = (double)inter / (double)uni;                         // in (0.5, 1]: a multiple of 2^-53
    const unsigned long long q = (unsigned long long)(iou * 9007199254740992.0);
    const unsigned long long old = atomicAdd(t.iou_acc + 2 * c, q);
    if (old + q < old) atomicAdd(t.iou_acc + 2 * c + 1, 1ull);              // carry into the high word
  }
}

// unmatched segments: a non-crowd gt is a false negative; a prediction is a false positive unless more than half of
// it lies on void or on a crowd region of its class
__global__ void __launch_bounds__(kThreads) eval_unmatched_kernel(PanArgs a) {
  const PanTables& t = a.t;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= t.mask; s += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t gk = t.gt_key[s];
    if (gk != kVoidId && t.gt_matched[s] == 0u) {
      const int c = channel_of((int32_t)gk, a.m);
      if (!is_crowd((int32_t)gk, c, a.is_thing)) atomicAdd(a.fn + c, 1ull);
    }
    const uint32_t pk = t.pr_key[s];
    if (pk != kVoidId && t.pr_matched[s] == 0u) {
      const uint64_t ignored = (uint64_t)t.pr_void[s] + t.pr_crowd[s];
      if (2 * ignored <= (uint64_t)t.pr_area[s]) atomicAdd(a.fp + channel_of((int32_t)pk, a.m), 1ull);
    }
  }
}

// 128-bit unsigned (hi, lo) -> double, rounded to nearest even once: the top 64 significant bits with the rest folded
// into a sticky bit (bit 0 lies below the rounding position of a 53-bit significand).  n < 2^31 matches of at most
// 2^53 each keep hi below 2^31, so 1 <= sh <= 31.
__device__ __forceinline__ double u128_to_double(unsigned long long hi, unsigned long long lo) {
  if (hi == 0ull) return __ull2double_rn(lo);
  const int sh = 64 - __clzll((long long)hi);
  const unsigned long long top = (hi << (64 - sh)) | (lo >> sh) | ((lo & ((1ull << sh) - 1ull)) != 0ull ? 1ull : 0ull);
  return ldexp(__ull2double_rn(top), sh);
}

__global__ void eval_iou_finish_kernel(const unsigned long long* __restrict__ acc, int C, double* iou_sum) {
  const int c = threadIdx.x;
  if (c < C) iou_sum[c] += ldexp(u128_to_double(acc[2 * c + 1], acc[2 * c]), -53);
}

// ------------------------------------------------------------------------------------------------ image / depth
struct ImageArgs {
  const float* rgb; const float* rgb_gt; const float* depth; const float* depth_gt; int64_t n;
};

// fixed tree over the block's threads: the sum's order depends on blockDim only
__device__ __forceinline__ void block_sum(double (*sh)[kThreads], double (&v)[kImageSums]) {
#pragma unroll
  for (int k = 0; k < kImageSums; ++k) sh[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w)
#pragma unroll
      for (int k = 0; k < kImageSums; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + w];
    __syncthreads();
  }
}

// partials[block][6] = {sum (rgb - gt)^2 over 3 channels, rgb pixels, sum |d|, sum d^2, sum |d| / gt, depth pixels}
// (d = depth - depth_gt over depth_gt > 0), in double from the fp32 inputs; each thread visits its pixels in order
__global__ void __launch_bounds__(kThreads) eval_image_kernel(ImageArgs a, double* __restrict__ partials) {
  __shared__ double sh[kImageSums][kThreads];
  double v[kImageSums] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    if (a.rgb != nullptr) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double d = (double)a.rgb[i * 3 + c] - (double)a.rgb_gt[i * 3 + c];
        v[0] += d * d;
      }
      v[1] += 1.0;
    }
    if (a.depth != nullptr) {
      const double g = (double)a.depth_gt[i];
      if (g > 0.0) {
        const double d = (double)a.depth[i] - g;
        v[2] += fabs(d);
        v[3] += d * d;
        v[4] += fabs(d) / g;
        v[5] += 1.0;
      }
    }
  }
  block_sum(sh, v);
  if (threadIdx.x < kImageSums) partials[blockIdx.x * kImageSums + threadIdx.x] = sh[threadIdx.x][0];
}

__global__ void __launch_bounds__(kThreads) eval_image_finish_kernel(const double* __restrict__ partials, int blocks,
                                                                      double* frame_sums) {
  __shared__ double sh[kImageSums][kThreads];
  double v[kImageSums];
#pragma unroll
  for (int k = 0; k < kImageSums; ++k) v[k] = (int)threadIdx.x < blocks ? partials[threadIdx.x * kImageSums + k] : 0.0;
  block_sum(sh, v);
  if (threadIdx.x < kImageSums) frame_sums[threadIdx.x] += sh[threadIdx.x][0];
}

// ------------------------------------------------------------------------------------------------ workspace
constexpr size_t kAlign = 256;
constexpr size_t align_up(size_t b) { return (b + kAlign - 1) / kAlign * kAlign; }
constexpr size_t kImageBytes = align_up(sizeof(double) * kImageBlocks * kImageSums);
constexpr size_t kIouBytes = align_up(sizeof(unsigned long long) * 2 * kEvalMaxClasses);

uint64_t table_slots(int64_t n) {
  uint64_t s = 1024;
  while (s < 2 * (uint64_t)n) s <<= 1;
  return s;
}
// [image partials][pair_key u64 | gt_key | pr_key  (all-ones)][pair_cnt | gt_area | gt_matched | pr_area | pr_void |
//  pr_crowd | pr_matched (zero) | iou_acc]
size_t key_bytes(uint64_t S) { return align_up(S * (8 + 4 + 4)); }
size_t count_bytes(uint64_t S) { return align_up(S * 4 * 7) + kIouBytes; }

PanTables carve(void* ws, uint64_t S) {
  char* p = static_cast<char*>(ws) + kImageBytes;
  PanTables t;
  t.mask = (uint32_t)(S - 1);
  t.pair_key = reinterpret_cast<unsigned long long*>(p);
  t.gt_key = reinterpret_cast<uint32_t*>(p + S * 8);
  t.pr_key = t.gt_key + S;
  uint32_t* c = reinterpret_cast<uint32_t*>(p + key_bytes(S));
  t.pair_cnt = c; t.gt_area = c + S; t.gt_matched = c + 2 * S;
  t.pr_area = c + 3 * S; t.pr_void = c + 4 * S; t.pr_crowd = c + 5 * S; t.pr_matched = c + 6 * S;
  t.iou_acc = reinterpret_cast<unsigned long long*>(p + key_bytes(S) + align_up(S * 4 * 7));
  return t;
}

}  // namespace
}  // namespace pnr

using namespace pnr;

extern "C" size_t pnr_eval_workspace_bytes(int64_t n) {
  const uint64_t S = table_slots(n < 0 ? 0 : n);
  return kImageBytes + key_bytes(S) + count_bytes(S);
}

extern "C" int pnr_eval_semantic(const int32_t* pred_pan, const int32_t* gt_pan, int64_t n, int32_t C,
                                 const int32_t* id_to_channel, int32_t n_ids, uint64_t* conf, void* stream) {
  PNR_CHECK_ARG(C >= 1 && C <= kEvalMaxClasses, "pnr_eval_semantic: C=%d outside [1, %d]", C, kEvalMaxClasses);
  PNR_CHECK_ARG(n >= 0 && n < ((int64_t)1 << 31), "pnr_eval_semantic: n=%lld outside [0, 2^31)", (long long)n);
  PNR_CHECK_ARG(pred_pan && gt_pan && conf, "pnr_eval_semantic: null pred_pan / gt_pan / conf");
  PNR_CHECK_ARG(!id_to_channel || n_ids > 0, "pnr_eval_semantic: id_to_channel needs n_ids > 0");
  if (n == 0) return PNR_OK;
  const IdMap m{id_to_channel, n_ids, C};
  const size_t smem = sizeof(uint32_t) * C * (C + 1);
  eval_semantic_kernel<<<grid_for(n), kThreads, smem, (cudaStream_t)stream>>>(
      pred_pan, gt_pan, n, m, reinterpret_cast<unsigned long long*>(conf));
  PNR_LAUNCH_CHECK("eval_semantic_kernel");
  return PNR_OK;
}

extern "C" int pnr_eval_panoptic(const int32_t* pred_pan, const int32_t* gt_pan, int64_t n, int32_t C,
                                 const int32_t* id_to_channel, int32_t n_ids, const uint8_t* is_thing, void* workspace,
                                 size_t workspace_bytes, uint64_t* tp, uint64_t* fp, uint64_t* fn, double* iou_sum,
                                 void* stream) {
  PNR_CHECK_ARG(C >= 1 && C <= kEvalMaxClasses, "pnr_eval_panoptic: C=%d outside [1, %d]", C, kEvalMaxClasses);
  PNR_CHECK_ARG(n >= 0 && n < ((int64_t)1 << 31), "pnr_eval_panoptic: n=%lld outside [0, 2^31)", (long long)n);
  PNR_CHECK_ARG(pred_pan && gt_pan && is_thing && workspace && tp && fp && fn && iou_sum,
                "pnr_eval_panoptic: null pred_pan / gt_pan / is_thing / workspace / tp / fp / fn / iou_sum");
  PNR_CHECK_ARG(!id_to_channel || n_ids > 0, "pnr_eval_panoptic: id_to_channel needs n_ids > 0");
  PNR_CHECK_ARG(workspace_bytes >= pnr_eval_workspace_bytes(n),
                "pnr_eval_panoptic: workspace of %zu bytes, pnr_eval_workspace_bytes(%lld) = %zu", workspace_bytes,
                (long long)n, pnr_eval_workspace_bytes(n));
  PNR_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "pnr_eval_panoptic: workspace not 16-byte aligned");
  if (n == 0) return PNR_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  const uint64_t S = table_slots(n);
  char* tables = static_cast<char*>(workspace) + kImageBytes;
  PNR_CUDA(cudaMemsetAsync(tables, 0xFF, key_bytes(S), st));
  PNR_CUDA(cudaMemsetAsync(tables + key_bytes(S), 0, count_bytes(S), st));
  PanArgs a{pred_pan, gt_pan, n, IdMap{id_to_channel, n_ids, C}, is_thing, carve(workspace, S),
            reinterpret_cast<unsigned long long*>(tp), reinterpret_cast<unsigned long long*>(fp),
            reinterpret_cast<unsigned long long*>(fn), iou_sum};
  eval_pairs_kernel<<<grid_for(n), kThreads, 0, st>>>(a);
  PNR_LAUNCH_CHECK("eval_pairs_kernel");
  eval_segments_kernel<<<grid_for((int64_t)S), kThreads, 0, st>>>(a);
  PNR_LAUNCH_CHECK("eval_segments_kernel");
  eval_match_kernel<<<grid_for((int64_t)S), kThreads, 0, st>>>(a);
  PNR_LAUNCH_CHECK("eval_match_kernel");
  eval_unmatched_kernel<<<grid_for((int64_t)S), kThreads, 0, st>>>(a);
  PNR_LAUNCH_CHECK("eval_unmatched_kernel");
  eval_iou_finish_kernel<<<1, kEvalMaxClasses, 0, st>>>(a.t.iou_acc, C, iou_sum);
  PNR_LAUNCH_CHECK("eval_iou_finish_kernel");
  return PNR_OK;
}

extern "C" int pnr_eval_image(const float* rgb_map, const float* rgb_gt, const float* depth_map, const float* depth_gt,
                              int64_t n, double* frame_sums, void* workspace, size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(n >= 0, "pnr_eval_image: n=%lld < 0", (long long)n);
  PNR_CHECK_ARG(frame_sums && workspace, "pnr_eval_image: null frame_sums / workspace");
  PNR_CHECK_ARG(!rgb_map == !rgb_gt, "pnr_eval_image: rgb_map and rgb_gt go together");
  PNR_CHECK_ARG(!depth_map == !depth_gt, "pnr_eval_image: depth_map and depth_gt go together");
  PNR_CHECK_ARG(workspace_bytes >= kImageBytes, "pnr_eval_image: workspace of %zu bytes, needs %zu (pnr_eval_workspace_bytes)",
                workspace_bytes, kImageBytes);
  if (n == 0 || (!rgb_map && !depth_map)) return PNR_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  const int64_t want = (n + kThreads - 1) / kThreads;
  const int blocks = (int)(want < kImageBlocks ? want : kImageBlocks);   // depends on n only: a fixed summation tree
  double* partials = static_cast<double*>(workspace);
  eval_image_kernel<<<blocks, kThreads, 0, st>>>(ImageArgs{rgb_map, rgb_gt, depth_map, depth_gt, n}, partials);
  PNR_LAUNCH_CHECK("eval_image_kernel");
  eval_image_finish_kernel<<<1, kThreads, 0, st>>>(partials, blocks, frame_sums);
  PNR_LAUNCH_CHECK("eval_image_finish_kernel");
  return PNR_OK;
}
