// weight_kernels.cu — per-pixel weights of a frame set for weighted training draws (include/pnr.h, DESIGN 3.4).
//   weights : pnr_pixel_weights, blockIdx.y strides over frames, x over the frame's pixels; each pixel is
//             pnr_weight_of_pixel of ray_math.h (also compiled for the host by the CPU tests).
//   counts  : pnr_label_counts, a shared-memory histogram per block, then one 64-bit atomic per non-zero bin.
//   cdf     : pnr_pixel_cdf, reduce-then-scan over tiles of 2^15 pixels: the tile sums, one block's scan of them, then
//             per tile its 1024 group sums scanned on top of the tile's prefix.  Integer sums: every schedule gives
//             the same bits.  A warp reads 1024 contiguous pixels (2 KB) as four coalesced 16-byte loads per lane and
//             forms the 32 group sums of the chunk by two xor shuffles and one transposing shuffle per load.
#include "common.cuh"
#include "ray_math.h"

#include <algorithm>

namespace pnr {

constexpr int kWeightThreads = 256;

__global__ void __launch_bounds__(kWeightThreads) pixel_weights_kernel(const __grid_constant__ pnr_pixel_weights_args a) {
  for (int f = blockIdx.y; f < a.F; f += gridDim.y) {
    int64_t lo, hi;
    const int cam = pnr_depth_frame(a.frame_cam, a.pix_offset, a.num_cameras, a.P, f, &lo, &hi);
    for (int64_t q = (int64_t)blockIdx.x * kWeightThreads + threadIdx.x; q < hi - lo;
         q += (int64_t)gridDim.x * kWeightThreads)
      a.weight[lo + q] = pnr_weight_of_pixel(a, f, cam, lo, q);
  }
}

__global__ void __launch_bounds__(kWeightThreads) label_counts_kernel(const int16_t* __restrict__ label, int64_t P,
                                                                      int C, unsigned long long* __restrict__ counts) {
  extern __shared__ uint32_t hist[];   // [C + 1]; a block counts at most 2^31 + 256 pixels (the grid sees to it)
  for (int i = threadIdx.x; i <= C; i += kWeightThreads) hist[i] = 0;
  __syncthreads();
  for (int64_t p = (int64_t)blockIdx.x * kWeightThreads + threadIdx.x; p < P; p += (int64_t)gridDim.x * kWeightThreads)
    atomicAdd(hist + pnr_weight_slot(__ldg(label + p), C), 1u);
  __syncthreads();
  for (int i = threadIdx.x; i <= C; i += kWeightThreads)
    if (hist[i] != 0) atomicAdd(counts + i, (unsigned long long)hist[i]);
}

constexpr int kCdfWarps = 8;
constexpr int kCdfChunk = 1024;                                   // pixels per warp step: 32 groups
constexpr int kCdfChunksPerWarp = 4;
constexpr int64_t kCdfTile = (int64_t)kCdfWarps * kCdfChunksPerWarp * kCdfChunk;   // 2^15 pixels, 1024 groups

// The sum of group c0 / 32 + lane of the chunk of 1024 pixels at c0 (c0 < P, a multiple of 1024), and in *nz the
// non-zero weights among the pixels this lane read.  Lane l's load k holds pixels c0 + 256 k + 8 l .. + 8, a quarter of
// group 8 k + l / 4.
__device__ __forceinline__ uint32_t chunk_group_sum(const uint16_t* __restrict__ w, int64_t P, int64_t c0, int lane,
                                                    uint32_t* nz) {
  uint32_t s[4];
  uint32_t n = 0;
  if (c0 + kCdfChunk <= P) {
    const uint4* v = reinterpret_cast<const uint4*>(w + c0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint4 x = __ldg(v + k * 32 + lane);
      const uint32_t words[4] = {x.x, x.y, x.z, x.w};
      uint32_t t = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t lo16 = words[j] & 0xFFFFu, hi16 = words[j] >> 16;
        t += lo16 + hi16;
        n += (lo16 != 0) + (hi16 != 0);
      }
      s[k] = t;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t b = c0 + k * 256 + lane * 8;
      uint32_t t = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t x = b + j < P ? (uint32_t)__ldg(w + b + j) : 0u;
        t += x;
        n += x != 0;
      }
      s[k] = t;
    }
  }
  *nz = n;
  uint32_t out = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    s[k] += __shfl_xor_sync(0xffffffffu, s[k], 1);
    s[k] += __shfl_xor_sync(0xffffffffu, s[k], 2);
    const uint32_t t = __shfl_sync(0xffffffffu, s[k], 4 * (lane & 7));   // group 8 k + (lane & 7)
    if (k == (lane >> 3)) out = t;
  }
  return out;
}

__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// ws[2 t] = the sum of tile t's weights, ws[2 t + 1] = its non-zero count
__global__ void __launch_bounds__(kCdfWarps * 32) cdf_tile_sums_kernel(const uint16_t* __restrict__ w, int64_t P,
                                                                       uint64_t* __restrict__ ws) {
  __shared__ uint32_t s_sum[kCdfWarps], s_nz[kCdfWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t t0 = (int64_t)blockIdx.x * kCdfTile;
  uint32_t sum = 0, nz = 0;   // a warp's 4096 pixels: < 2^28
  for (int i = 0; i < kCdfChunksPerWarp; ++i) {
    const int64_t c0 = t0 + (int64_t)(warp * kCdfChunksPerWarp + i) * kCdfChunk;
    if (c0 >= P) break;
    uint32_t n;
    sum += chunk_group_sum(w, P, c0, lane, &n);
    nz += n;
  }
  sum = warp_sum_u32(sum);
  nz = warp_sum_u32(nz);
  if (lane == 0) { s_sum[warp] = sum; s_nz[warp] = nz; }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t a = 0, b = 0;
    for (int k = 0; k < kCdfWarps; ++k) { a += s_sum[k]; b += s_nz[k]; }
    ws[2 * blockIdx.x] = a;
    ws[2 * blockIdx.x + 1] = b;
  }
}

// one block: ws[2 t] <- the exclusive prefix of the tile sums; totals = {T, non-zero count}
constexpr int kCdfScanThreads = 1024;
__global__ void __launch_bounds__(kCdfScanThreads) cdf_scan_tiles_kernel(uint64_t* __restrict__ ws, int64_t tiles,
                                                                         uint64_t* __restrict__ totals) {
  __shared__ uint64_t s_warp[kCdfScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t carry = 0, nz = 0;
  for (int64_t b = 0; b < tiles; b += kCdfScanThreads) {
    const int64_t t = b + threadIdx.x;
    const uint64_t v = t < tiles ? ws[2 * t] : 0;
    if (t < tiles) nz += ws[2 * t + 1];
    uint64_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint64_t o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint64_t before = carry, all = carry;
    for (int k = 0; k < kCdfScanThreads / 32; ++k) {
      if (k < warp) before += s_warp[k];
      all += s_warp[k];
    }
    if (t < tiles) ws[2 * t] = before + incl - v;
    carry = all;
    __syncthreads();   // s_warp is rewritten by the next round
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) nz += __shfl_xor_sync(0xffffffffu, nz, d);
  if (lane == 0) s_warp[warp] = nz;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t n = 0;
    for (int k = 0; k < kCdfScanThreads / 32; ++k) n += s_warp[k];
    totals[0] = carry;
    totals[1] = n;
  }
}

// cum[g] for the 1024 groups of tile blockIdx.x: its prefix (ws) plus the inclusive scan of its group sums
__global__ void __launch_bounds__(kCdfWarps * 32) cdf_tile_scan_kernel(const uint16_t* __restrict__ w, int64_t P,
                                                                       const uint64_t* __restrict__ ws,
                                                                       uint64_t* __restrict__ cum) {
  __shared__ uint32_t s_tot[kCdfWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t t0 = (int64_t)blockIdx.x * kCdfTile;
  uint32_t incl[kCdfChunksPerWarp];
  uint32_t run = 0;   // the warp's running sum: < 2^28
#pragma unroll
  for (int i = 0; i < kCdfChunksPerWarp; ++i) {
    incl[i] = 0;
    const int64_t c0 = t0 + (int64_t)(warp * kCdfChunksPerWarp + i) * kCdfChunk;
    if (c0 < P) {
      uint32_t n;
      uint32_t v = chunk_group_sum(w, P, c0, lane, &n);
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += o;
      }
      incl[i] = run + v;
      run += __shfl_sync(0xffffffffu, v, 31);
    }
  }
  if (lane == 0) s_tot[warp] = run;
  __syncthreads();
  uint64_t base = ws[2 * blockIdx.x];
  for (int k = 0; k < warp; ++k) base += s_tot[k];
  const int64_t G = (P + PNR_WEIGHT_GROUP - 1) / PNR_WEIGHT_GROUP;
#pragma unroll
  for (int i = 0; i < kCdfChunksPerWarp; ++i) {
    const int64_t g = (t0 + (int64_t)(warp * kCdfChunksPerWarp + i) * kCdfChunk) / PNR_WEIGHT_GROUP + lane;
    if (g < G) cum[g] = base + incl[i];
  }
}

}  // namespace pnr

using namespace pnr;

extern "C" int pnr_pixel_weights(const pnr_pixel_weights_args* args, void* stream) {
  PNR_CHECK_ARG(args, "pnr_pixel_weights: null args");
  const pnr_pixel_weights_args& a = *args;
  PNR_CHECK_ARG(a.F >= 1 && a.F < INT32_MAX, "pnr_pixel_weights: F=%d outside [1, 2^31 - 1)", a.F);
  PNR_CHECK_ARG(a.P >= 1, "pnr_pixel_weights: P=%lld < 1", (long long)a.P);
  PNR_CHECK_ARG(a.C >= 0 && a.C <= 32767, "pnr_pixel_weights: C=%d outside [0, 32767]", a.C);
  int rc = check_cameras("pnr_pixel_weights", a.cams, a.num_cameras, 31);
  if (rc != PNR_OK) return rc;
  PNR_CHECK_ARG(a.frame_cam && a.pix_offset && a.weight,
                "pnr_pixel_weights: null pointer (frame_cam, pix_offset and weight are required)");
  PNR_CHECK_ARG(isfinite(a.scale) && a.scale > 0.f, "pnr_pixel_weights: scale=%g is not finite and > 0",
                (double)a.scale);
  int dev = 0;
  rc = current_device("pnr_pixel_weights", &dev);
  if (rc != PNR_OK) return rc;
  int64_t max_hw = 1;
  for (int k = 0; k < a.num_cameras; ++k) max_hw = std::max(max_hw, (int64_t)a.cams[k].H * a.cams[k].W);
  const int64_t ny = std::min<int64_t>(a.F, 65535);
  const int64_t want = (max_hw + kWeightThreads - 1) / kWeightThreads;
  const int64_t cap = std::max<int64_t>(1, (int64_t)num_sms(dev) * 16 / ny);
  pixel_weights_kernel<<<dim3((unsigned)std::min(want, cap), (unsigned)ny), kWeightThreads, 0, (cudaStream_t)stream>>>(a);
  PNR_LAUNCH_CHECK("pixel_weights_kernel");
  return PNR_OK;
}

extern "C" int pnr_label_counts(const int16_t* label, int64_t P, int32_t C, uint64_t* counts, void* stream) {
  PNR_CHECK_ARG(P >= 1, "pnr_label_counts: P=%lld < 1", (long long)P);
  PNR_CHECK_ARG(C >= 0 && C <= 8191, "pnr_label_counts: C=%d outside [0, 8191]", C);
  PNR_CHECK_ARG(label && counts, "pnr_label_counts: null pointer (label and counts are required)");
  int dev = 0;
  int rc = current_device("pnr_label_counts", &dev);
  if (rc != PNR_OK) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  PNR_CUDA(cudaMemsetAsync(counts, 0, (size_t)(C + 1) * sizeof(uint64_t), st));
  const int64_t want = (P + kWeightThreads - 1) / kWeightThreads;
  const int64_t least = (P + (int64_t(1) << 31) - 1) >> 31;   // no block counts more than 2^31 + 256 pixels
  const int64_t blocks = std::max(least, std::min(want, (int64_t)num_sms(dev) * 8));
  label_counts_kernel<<<(unsigned)blocks, kWeightThreads, (size_t)(C + 1) * sizeof(uint32_t), st>>>(
      label, P, C, (unsigned long long*)counts);
  PNR_LAUNCH_CHECK("label_counts_kernel");
  return PNR_OK;
}

extern "C" size_t pnr_pixel_cdf_workspace_bytes(int64_t P) {
  if (P < 1 || P >= (int64_t(1) << 47)) return 0;
  return (size_t)((P + kCdfTile - 1) / kCdfTile) * 2 * sizeof(uint64_t);
}

extern "C" int pnr_pixel_cdf(const uint16_t* weight, int64_t P, uint64_t* cum, uint64_t* totals, void* workspace,
                             size_t workspace_bytes, void* stream) {
  PNR_CHECK_ARG(P >= 1 && P < (int64_t(1) << 47), "pnr_pixel_cdf: P=%lld outside [1, 2^47)", (long long)P);
  PNR_CHECK_ARG(weight && cum && totals, "pnr_pixel_cdf: null pointer (weight, cum and totals are required)");
  PNR_CHECK_ARG(((uintptr_t)weight & 15) == 0, "pnr_pixel_cdf: weight is not 16-byte aligned");
  const size_t need = pnr_pixel_cdf_workspace_bytes(P);
  PNR_CHECK_ARG(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 15) == 0,
                "pnr_pixel_cdf: workspace of %zu bytes at %p; it needs %zu bytes, 16-byte aligned", workspace_bytes,
                workspace, need);
  const int64_t tiles = (P + kCdfTile - 1) / kCdfTile;
  PNR_CHECK_ARG(tiles < INT32_MAX, "pnr_pixel_cdf: %lld tiles", (long long)tiles);
  const cudaStream_t st = (cudaStream_t)stream;
  uint64_t* ws = (uint64_t*)workspace;
  cdf_tile_sums_kernel<<<(unsigned)tiles, kCdfWarps * 32, 0, st>>>(weight, P, ws);
  PNR_LAUNCH_CHECK("cdf_tile_sums_kernel");
  cdf_scan_tiles_kernel<<<1, kCdfScanThreads, 0, st>>>(ws, tiles, totals);
  PNR_LAUNCH_CHECK("cdf_scan_tiles_kernel");
  cdf_tile_scan_kernel<<<(unsigned)tiles, kCdfWarps * 32, 0, st>>>(weight, P, ws, cum);
  PNR_LAUNCH_CHECK("cdf_tile_scan_kernel");
  return PNR_OK;
}
