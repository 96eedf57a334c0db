// stereo_math.h — the per-pixel and per-step rules of pnr_stereo_depth (include/pnr.h, DESIGN 3.4): grey, census,
// matching cost, one step of a semi-global aggregation path over packed u16 pairs, the left-right minimum and the
// per-pixel selection.  Shared by the kernels (stereo_kernels.cu) and the host build the CPU tests hold against the
// numpy oracle (tests/host_emu.cpp); the kernels keep only layout here (staging, shuffles, the path walk).
// Everything is integer arithmetic until the one fp32 division of the depth, so both builds give the same bits.
#pragma once
#include <stdint.h>
#include "../../include/pnr.h"

#if defined(__CUDACC__)
#define PNR_SHD __host__ __device__ __forceinline__
#else
#define PNR_SHD inline
#endif

#define PNR_STEREO_COST_NONE 63u        // the cost of a disparity whose right pixel x - d is outside the image
#define PNR_STEREO_ABSENT 0x7FFF7FFFu   // both halves of a packed pair that takes no part (d - 1 < 0, d + 1 >= D, d >= D)

// Packed unsigned 16-bit pairs.  On sm_90a the add-min and three-way min are the DPX instructions VIADDMNMX.U16x2 /
// VIMNMX3.U16x2; the host build spells out the same per-halfword operation.  Every value the step forms stays below
// 2^16 (L <= 63 + P2 <= 2111, ABSENT + P1 <= 34815), so no halfword wraps.
PNR_SHD uint32_t pnr_u16x2_add(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __vadd2(a, b);
#else
  return ((a + b) & 0xFFFFu) | ((((a >> 16) + (b >> 16)) & 0xFFFFu) << 16);
#endif
}
PNR_SHD uint32_t pnr_u16x2_sub(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __vsub2(a, b);
#else
  return ((a - b) & 0xFFFFu) | ((((a >> 16) - (b >> 16)) & 0xFFFFu) << 16);
#endif
}
PNR_SHD uint32_t pnr_u16_min(uint32_t a, uint32_t b) { return a < b ? a : b; }
// min(a + b, c) per halfword
PNR_SHD uint32_t pnr_u16x2_addmin(uint32_t a, uint32_t b, uint32_t c) {
#if defined(__CUDA_ARCH__)
  return __viaddmin_u16x2(a, b, c);
#else
  const uint32_t s = pnr_u16x2_add(a, b);
  return pnr_u16_min(s & 0xFFFFu, c & 0xFFFFu) | (pnr_u16_min(s >> 16, c >> 16) << 16);
#endif
}
// min(a, b, c) per halfword
PNR_SHD uint32_t pnr_u16x2_min3(uint32_t a, uint32_t b, uint32_t c) {
#if defined(__CUDA_ARCH__)
  return __vimin3_u16x2(a, b, c);
#else
  return pnr_u16_min(pnr_u16_min(a & 0xFFFFu, b & 0xFFFFu), c & 0xFFFFu) |
         (pnr_u16_min(pnr_u16_min(a >> 16, b >> 16), c >> 16) << 16);
#endif
}
PNR_SHD uint32_t pnr_u16x2_splat(uint32_t v) { return (v & 0xFFFFu) * 0x10001u; }
// the pair (hi half of a, lo half of b): the neighbours one disparity down of b's pair, or one up of a's
PNR_SHD uint32_t pnr_u16x2_funnel(uint32_t a, uint32_t b) { return (a >> 16) | (b << 16); }

// Grey: g = (4899 R + 9617 G + 1868 B + 8192) >> 14
PNR_SHD uint32_t pnr_grey(uint32_t r, uint32_t g, uint32_t b) { return (4899u * r + 9617u * g + 1868u * b + 8192u) >> 14; }

// Census of the pixel at the centre of a 9 x 7 window of grey values (9 wide, 7 high; row k at win + k * pitch, edge
// pixels already repeated where the window leaves the image): bit k of the 62, in raster order with the centre
// skipped, is 1 iff g(q_k) < g(p).
PNR_SHD uint64_t pnr_census(const uint8_t* win, int pitch) {
  const uint32_t c = win[3 * pitch + 4];
  uint64_t bits = 0;
  int k = 0;
  for (int dy = 0; dy < 7; ++dy)
    for (int dx = 0; dx < 9; ++dx) {
      if (dy == 3 && dx == 4) continue;
      bits |= (uint64_t)(win[dy * pitch + dx] < c) << k;
      ++k;
    }
  return bits;
}

PNR_SHD uint32_t pnr_census_cost(uint64_t l, uint64_t r) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__popcll(l ^ r);
#else
  return (uint32_t)__builtin_popcountll(l ^ r);
#endif
}

// One step of a path, for the packed pair L of disparities (d, d + 1), d even:
//   L_r(p, d) = C(p, d) + min(L_r(p-r, d), L_r(p-r, d-1) + P1, L_r(p-r, d+1) + P1, m + P2) - m
// L: the pair at p - r; below / above: the packed pairs holding d - 1 (in its hi half) and d + 2 (in its lo half),
// PNR_STEREO_ABSENT where those disparities do not exist; c: the costs at p; m2 / p1x2 / mp2: m, P1 and m + P2 in both
// halves.  A path starts from L = 0 for every d < D and m = 0, which gives L_r = C at its first pixel.
PNR_SHD uint32_t pnr_sgm_step(uint32_t L, uint32_t below, uint32_t above, uint32_t c, uint32_t m2, uint32_t p1x2,
                              uint32_t mp2) {
  const uint32_t lm1 = pnr_u16x2_funnel(below, L);   // (d - 1, d)
  const uint32_t lp1 = pnr_u16x2_funnel(L, above);   // (d + 1, d + 2)
  const uint32_t a = pnr_u16x2_addmin(lm1, p1x2, L);
  const uint32_t b = pnr_u16x2_addmin(lp1, p1x2, mp2);
  return pnr_u16x2_add(pnr_u16x2_sub(pnr_u16x2_min3(a, b, mp2), m2), c);
}

// The first pixel of path i of direction (dx, dy) (each in {-1, 0, 1}, not both 0) of an H x W image, the pixels
// whose p - r is outside it: for dy = 0 column x0 (H paths), for dx = 0 row y0 (W paths), else column x0 for every
// row and then row y0 for the other columns (H + W - 1 paths); x0 = 0 for dx > 0 else W - 1, y0 likewise.
PNR_SHD int pnr_sgm_num_paths(int dx, int dy, int H, int W) { return dx == 0 ? W : (dy == 0 ? H : H + W - 1); }
PNR_SHD void pnr_sgm_path_start(int dx, int dy, int H, int W, int i, int* x, int* y) {
  const int x0 = dx > 0 ? 0 : W - 1, y0 = dy > 0 ? 0 : H - 1;
  if (dx == 0) { *x = i; *y = y0; return; }
  if (i < H) { *x = x0; *y = i; return; }
  const int j = i - H + 1;   // the other columns, 1 .. W - 1 away from x0
  *x = dx > 0 ? j : W - 1 - j;
  *y = y0;
}

// The left-right check's right disparity d_R(xr) = argmin_d S(xr + d, y, d) over d < D with xr + d < W, the lowest d
// on ties; srow = S of row y, [W, D].
PNR_SHD int pnr_stereo_right_argmin(const uint16_t* srow, int W, int D, int xr) {
  int best = 0;
  uint32_t bs = srow[(int64_t)xr * D];
  for (int d = 1; d < D && xr + d < W; ++d) {
    const uint32_t s = srow[(int64_t)(xr + d) * D + d];
    if (s < bs) { bs = s; best = d; }
  }
  return best;
}

// The disparity of pixel x in sixteenths, or -1: s = S(x, y, 0 .. D), drow = d_R of row y.  Winner d* = argmin S, the
// lowest d on ties; invalid if some |d - d*| > 1 has S(d) (100 - U) < S(d*) 100, or unless x - d* >= 0 and
// |d* - d_R(x - d*)| <= 1; subpixel for 0 < d* < D - 1: den = max(S(d*-1) + S(d*+1) - 2 S(d*), 1),
// 16 d* + ((S(d*-1) - S(d*+1)) 16 + den) / (2 den), C's division (toward zero).
PNR_SHD int pnr_stereo_select(const uint16_t* s, int D, int U, int x, const int16_t* drow) {
  int best = 0;
  int32_t bs = s[0];
  for (int d = 1; d < D; ++d)
    if ((int32_t)s[d] < bs) { bs = s[d]; best = d; }
  const int32_t lim = bs * 100;
  for (int d = 0; d < D; ++d)
    if ((d < best - 1 || d > best + 1) && (int32_t)s[d] * (100 - U) < lim) return -1;
  if (x - best < 0) return -1;
  const int dr = drow[x - best];
  if (dr - best > 1 || best - dr > 1) return -1;
  if (best == 0 || best == D - 1) return 16 * best;
  const int32_t lo = s[best - 1], hi = s[best + 1];
  int32_t den = lo + hi - 2 * bs;
  den = den < 1 ? 1 : den;
  return 16 * best + ((lo - hi) * 16 + den) / (2 * den);
}

// Depth from a disparity in sixteenths: t = B16 / fp32(d16) (one IEEE division), kept when d16 > 0 and
// min_depth < t <= max_depth, else 0.
PNR_SHD float pnr_stereo_depth_of(int d16, float b16, float min_depth, float max_depth) {
  if (d16 <= 0) return 0.f;
#if defined(__CUDA_ARCH__)
  const float t = __fdiv_rn(b16, (float)d16);
#else
  const float t = b16 / (float)d16;
#endif
  return (t > min_depth && t <= max_depth) ? t : 0.f;
}
