// stereo_kernels.cu — pnr_stereo_depth: semi-global matching of rectified stereo pairs into the frame store's depth
// (include/pnr.h, DESIGN 3.4).  Per chunk of frames, a fixed sequence of launches:
//   census    : grey and 9 x 7 census of both images, a tile of rows staged in shared memory.
//   aggregate : one launch per direction, one warp per path line.  Lane l holds the disparities
//               [2 K2 l, 2 K2 (l + 1)) as K2 packed u16 pairs (K2 = ceil(D / 64)); the step is pnr_sgm_step (DPX),
//               the neighbours across lanes come by one shuffle each way and m_r by __reduce_min_sync.  Costs are
//               recomputed from the census words at each step.  S is accumulated in the workspace by direction: the
//               first direction stores L_r, the other seven add theirs (u16 adds, exact; launch order on the stream
//               keeps them apart).  At every step a warp reads and writes the D contiguous u16 of one pixel, so
//               vertical and diagonal paths are as coalesced as horizontal ones.
//   right     : d_R of the left-right check, one thread per pixel (the diagonal of S along the row).
//   select    : winner, uniqueness, left-right check, subpixel and depth, one thread per pixel
//               (pnr_stereo_select / pnr_stereo_depth_of of stereo_math.h), straight into the store's depth rows.
// S was chosen over eight per-direction volumes because it moves the fewest bytes: 2 N D of stores for the first
// direction and 4 N D of loads and stores for each other one, against 16 N D of stores and 16 N D of loads to sum
// eight volumes afterwards.
#include "common.cuh"
#include "stereo_math.h"

#include <algorithm>

namespace pnr {

constexpr int kStereoFramesPerLaunch = 256;
constexpr int kCensusTX = 128, kCensusTY = 8;
constexpr int kAggWarps = 4;
constexpr int kPixThreads = 256;

struct StereoParams {
  const uint8_t* rgb8;
  const int64_t* pix_offset;
  int64_t P;
  const uint8_t* right;
  int32_t H, W, D, P1, P2, U;
  float B16, min_depth, max_depth;
  float* depth;
  int16_t* disparity;
  uint64_t* census_l;
  uint64_t* census_r;
  uint16_t* S;
  int16_t* d_right;
  int32_t base;   // the call's index of this launch's first frame
  int32_t frames[kStereoFramesPerLaunch];
};

// the store's pixels of frame f, or false when its range is not H W pixels inside [0, P]
__device__ __forceinline__ bool stereo_frame(const StereoParams& p, int f, int64_t* lo) {
  const int64_t a = p.pix_offset[f], b = p.pix_offset[f + 1];
  *lo = a;
  return a >= 0 && b <= p.P && b - a == (int64_t)p.H * p.W;
}

// blockIdx.z = 2 i + side (side 0: the store's left image, 1: right[i])
__global__ void __launch_bounds__(kCensusTX) stereo_census_kernel(const __grid_constant__ StereoParams p) {
  __shared__ uint8_t g[kCensusTY + 6][kCensusTX + 8];
  const int i = blockIdx.z >> 1, side = blockIdx.z & 1;
  const int64_t fi = p.base + i, HW = (int64_t)p.H * p.W;
  const uint8_t* img;
  if (side == 0) {
    int64_t lo;
    if (!stereo_frame(p, p.frames[i], &lo)) return;
    img = p.rgb8 + lo * 3;
  } else {
    img = p.right + fi * HW * 3;
  }
  const int x0 = blockIdx.x * kCensusTX, y0 = blockIdx.y * kCensusTY;
  for (int k = threadIdx.x; k < (kCensusTY + 6) * (kCensusTX + 8); k += kCensusTX) {
    const int r = k / (kCensusTX + 8), c = k % (kCensusTX + 8);
    const int yy = min(max(y0 - 3 + r, 0), p.H - 1), xx = min(max(x0 - 4 + c, 0), p.W - 1);
    const uint8_t* px = img + ((int64_t)yy * p.W + xx) * 3;
    g[r][c] = (uint8_t)pnr_grey(px[0], px[1], px[2]);
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= p.W) return;
  uint64_t* out = (side == 0 ? p.census_l : p.census_r) + fi * HW;
  for (int r = 0; r < kCensusTY && y0 + r < p.H; ++r)
    out[(int64_t)(y0 + r) * p.W + x] = pnr_census(&g[r][threadIdx.x], kCensusTX + 8);
}

// blockIdx.y = frame of the launch; warp w of block b walks path b kAggWarps + w of direction (dx, dy)
template <int K2>
__global__ void __launch_bounds__(kAggWarps * 32) stereo_aggregate_kernel(const __grid_constant__ StereoParams p,
                                                                          int dx, int dy, int first) {
  const int lane = threadIdx.x & 31;
  const int path = blockIdx.x * kAggWarps + (threadIdx.x >> 5);
  const int H = p.H, W = p.W, D = p.D;
  if (path >= pnr_sgm_num_paths(dx, dy, H, W)) return;   // the whole warp
  const int64_t fi = p.base + blockIdx.y, HW = (int64_t)H * W;
  const uint64_t* cl = p.census_l + fi * HW;
  const uint64_t* cr = p.census_r + fi * HW;
  uint32_t* S = reinterpret_cast<uint32_t*>(p.S + fi * HW * D);
  int x, y;
  pnr_sgm_path_start(dx, dy, H, W, path, &x, &y);
  const int d_lane = lane * 2 * K2;
  uint32_t L[K2];
#pragma unroll
  for (int j = 0; j < K2; ++j) L[j] = d_lane + 2 * j < D ? 0u : PNR_STEREO_ABSENT;
  uint32_t m = 0;
  const uint32_t p1x2 = pnr_u16x2_splat(p.P1);
  while (x >= 0 && x < W && y >= 0 && y < H) {
    const int64_t q = (int64_t)y * W + x;
    const uint64_t l = cl[q];
    const uint64_t* crow = cr + (int64_t)y * W;
    uint32_t c[K2];
#pragma unroll
    for (int j = 0; j < K2; ++j) {
      const int d = d_lane + 2 * j;
      const uint32_t c0 = (d < D && x - d >= 0) ? pnr_census_cost(l, crow[x - d]) : PNR_STEREO_COST_NONE;
      const uint32_t c1 = (d < D && x - d - 1 >= 0) ? pnr_census_cost(l, crow[x - d - 1]) : PNR_STEREO_COST_NONE;
      c[j] = c0 | (c1 << 16);
    }
    uint32_t below = __shfl_up_sync(0xffffffffu, L[K2 - 1], 1);
    uint32_t above = __shfl_down_sync(0xffffffffu, L[0], 1);
    if (lane == 0) below = PNR_STEREO_ABSENT;
    if (lane == 31) above = PNR_STEREO_ABSENT;
    const uint32_t m2 = pnr_u16x2_splat(m), mp2 = pnr_u16x2_splat(m + p.P2);
    uint32_t n[K2];
#pragma unroll
    for (int j = 0; j < K2; ++j)
      n[j] = d_lane + 2 * j < D ? pnr_sgm_step(L[j], j > 0 ? L[j - 1] : below, j + 1 < K2 ? L[j + 1] : above, c[j],
                                               m2, p1x2, mp2)
                                : PNR_STEREO_ABSENT;
    uint32_t mm = n[0];
#pragma unroll
    for (int j = 0; j < K2; ++j) {
      L[j] = n[j];
      if (j > 0) mm = pnr_u16x2_min3(mm, n[j], n[j]);
    }
    m = __reduce_min_sync(0xffffffffu, pnr_u16_min(mm & 0xFFFFu, mm >> 16));
    uint32_t* s = S + q * (D / 2) + lane * K2;
#pragma unroll
    for (int j = 0; j < K2; ++j)
      if (d_lane + 2 * j < D) s[j] = first ? L[j] : pnr_u16x2_add(s[j], L[j]);
    x += dx;
    y += dy;
  }
}

// blockIdx.y = frame of the launch, x over its pixels
__global__ void __launch_bounds__(kPixThreads) stereo_right_kernel(const __grid_constant__ StereoParams p) {
  const int64_t HW = (int64_t)p.H * p.W, q = (int64_t)blockIdx.x * kPixThreads + threadIdx.x;
  if (q >= HW) return;
  const int64_t fi = p.base + blockIdx.y, y = q / p.W;
  const uint16_t* srow = p.S + (fi * HW + y * p.W) * p.D;
  p.d_right[fi * HW + q] = (int16_t)pnr_stereo_right_argmin(srow, p.W, p.D, (int)(q - y * p.W));
}

__global__ void __launch_bounds__(kPixThreads) stereo_select_kernel(const __grid_constant__ StereoParams p) {
  const int64_t HW = (int64_t)p.H * p.W, q = (int64_t)blockIdx.x * kPixThreads + threadIdx.x;
  if (q >= HW) return;
  const int64_t fi = p.base + blockIdx.y, y = q / p.W;
  int64_t lo;
  const bool ok = stereo_frame(p, p.frames[blockIdx.y], &lo);
  const int d16 = ok ? pnr_stereo_select(p.S + (fi * HW + q) * p.D, p.D, p.U, (int)(q - y * p.W),
                                         p.d_right + fi * HW + y * p.W)
                     : -1;
  if (p.disparity) p.disparity[fi * HW + q] = (int16_t)d16;
  if (p.depth && ok) p.depth[lo + q] = pnr_stereo_depth_of(d16, p.B16, p.min_depth, p.max_depth);
}

static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

static bool stereo_sizes_ok(int32_t n, int32_t H, int32_t W, int32_t D) {
  return n >= 1 && H >= 1 && H <= 65535 && W >= 1 && W <= 65535 && D >= 32 && D <= 256 && D % 32 == 0;
}

}  // namespace pnr

using namespace pnr;

extern "C" size_t pnr_stereo_workspace_bytes(int32_t n, int32_t H, int32_t W, int32_t D) {
  if (!stereo_sizes_ok(n, H, W, D)) return 0;
  const size_t N = (size_t)n * H * W;
  return 2 * align16(8 * N) + align16(2 * N * D) + align16(2 * N);
}

extern "C" int pnr_stereo_depth(const pnr_stereo_args* args, void* stream) {
  PNR_CHECK_ARG(args, "pnr_stereo_depth: null args");
  const pnr_stereo_args& a = *args;
  PNR_CHECK_ARG(a.n >= 1, "pnr_stereo_depth: n=%d < 1", a.n);
  PNR_CHECK_ARG(a.H >= 1 && a.H <= 65535 && a.W >= 1 && a.W <= 65535,
                "pnr_stereo_depth: H=%d W=%d outside [1, 65535]", a.H, a.W);
  PNR_CHECK_ARG(a.D >= 32 && a.D <= 256 && a.D % 32 == 0, "pnr_stereo_depth: D=%d not in {32, 64, .., 256}", a.D);
  PNR_CHECK_ARG(a.P1 >= 0 && a.P1 <= a.P2 && a.P2 <= 2048, "pnr_stereo_depth: P1=%d P2=%d outside 0 <= P1 <= P2 <= 2048",
                a.P1, a.P2);
  PNR_CHECK_ARG(a.U >= 0 && a.U <= 99, "pnr_stereo_depth: U=%d outside [0, 99]", a.U);
  PNR_CHECK_ARG(a.F >= 1 && a.F < INT32_MAX, "pnr_stereo_depth: F=%d outside [1, 2^31 - 1)", a.F);
  PNR_CHECK_ARG(a.P >= 1, "pnr_stereo_depth: P=%lld < 1", (long long)a.P);
  PNR_CHECK_ARG(a.rgb8 && a.pix_offset && a.right && a.frames,
                "pnr_stereo_depth: null input pointer (rgb8, pix_offset, right and frames are required)");
  PNR_CHECK_ARG(a.depth || a.disparity, "pnr_stereo_depth: null outputs (depth and disparity are both null)");
  for (int i = 0; i < a.n; ++i)
    PNR_CHECK_ARG(a.frames[i] >= 0 && a.frames[i] < a.F, "pnr_stereo_depth: frames[%d]=%d outside [0, F=%d)", i,
                  a.frames[i], a.F);
  if (a.depth) {
    PNR_CHECK_ARG(isfinite(a.B16) && a.B16 > 0.f, "pnr_stereo_depth: B16=%g is not finite and > 0", (double)a.B16);
    PNR_CHECK_ARG(isfinite(a.min_depth) && a.min_depth > 0.f, "pnr_stereo_depth: min_depth=%g is not finite and > 0",
                  (double)a.min_depth);
    PNR_CHECK_ARG(isfinite(a.max_depth) && a.max_depth > a.min_depth,
                  "pnr_stereo_depth: max_depth=%g is not finite and > min_depth=%g", (double)a.max_depth,
                  (double)a.min_depth);
  }
  const size_t need = pnr_stereo_workspace_bytes(a.n, a.H, a.W, a.D);
  PNR_CHECK_ARG(a.workspace && a.workspace_bytes >= need && ((uintptr_t)a.workspace & 15) == 0,
                "pnr_stereo_depth: workspace of %zu bytes at %p; the call needs %zu bytes, 16-byte aligned",
                a.workspace_bytes, a.workspace, need);
  int dev = 0;
  int rc = current_device("pnr_stereo_depth", &dev);
  if (rc != PNR_OK) return rc;
  const cudaStream_t st = (cudaStream_t)stream;

  const size_t N = (size_t)a.n * a.H * a.W;
  char* ws = (char*)a.workspace;
  StereoParams sp;
  sp.rgb8 = a.rgb8; sp.pix_offset = a.pix_offset; sp.P = a.P; sp.right = a.right;
  sp.H = a.H; sp.W = a.W; sp.D = a.D; sp.P1 = a.P1; sp.P2 = a.P2; sp.U = a.U;
  sp.B16 = a.B16; sp.min_depth = a.min_depth; sp.max_depth = a.max_depth;
  sp.depth = a.depth; sp.disparity = a.disparity;
  sp.census_l = (uint64_t*)ws;
  sp.census_r = (uint64_t*)(ws + align16(8 * N));
  sp.S = (uint16_t*)(ws + 2 * align16(8 * N));
  sp.d_right = (int16_t*)(ws + 2 * align16(8 * N) + align16(2 * N * a.D));

  static const int kDirs[8][2] = {{1, 0}, {-1, 0}, {0, 1}, {0, -1}, {1, 1}, {-1, -1}, {1, -1}, {-1, 1}};
  const int K2 = (a.D + 63) / 64;
  const unsigned pix_blocks = (unsigned)(((int64_t)a.H * a.W + kPixThreads - 1) / kPixThreads);
  for (int f0 = 0; f0 < a.n; f0 += kStereoFramesPerLaunch) {
    const int nf = std::min(kStereoFramesPerLaunch, a.n - f0);
    sp.base = f0;
    for (int i = 0; i < nf; ++i) sp.frames[i] = a.frames[f0 + i];
    stereo_census_kernel<<<dim3((a.W + kCensusTX - 1) / kCensusTX, (a.H + kCensusTY - 1) / kCensusTY, 2 * nf),
                           kCensusTX, 0, st>>>(sp);
    PNR_LAUNCH_CHECK("stereo_census_kernel");
    for (int r = 0; r < 8; ++r) {
      const int dx = kDirs[r][0], dy = kDirs[r][1];
      const dim3 grid((pnr_sgm_num_paths(dx, dy, a.H, a.W) + kAggWarps - 1) / kAggWarps, nf);
      const int first = r == 0;
      switch (K2) {
        case 1: stereo_aggregate_kernel<1><<<grid, kAggWarps * 32, 0, st>>>(sp, dx, dy, first); break;
        case 2: stereo_aggregate_kernel<2><<<grid, kAggWarps * 32, 0, st>>>(sp, dx, dy, first); break;
        case 3: stereo_aggregate_kernel<3><<<grid, kAggWarps * 32, 0, st>>>(sp, dx, dy, first); break;
        default: stereo_aggregate_kernel<4><<<grid, kAggWarps * 32, 0, st>>>(sp, dx, dy, first); break;
      }
      PNR_LAUNCH_CHECK("stereo_aggregate_kernel");
    }
    stereo_right_kernel<<<dim3(pix_blocks, nf), kPixThreads, 0, st>>>(sp);
    PNR_LAUNCH_CHECK("stereo_right_kernel");
    stereo_select_kernel<<<dim3(pix_blocks, nf), kPixThreads, 0, st>>>(sp);
    PNR_LAUNCH_CHECK("stereo_select_kernel");
  }
  return PNR_OK;
}
