// host_emu_stereo.cpp — host build of the semi-global matching routines of csrc/stereo_math.h (pnr_grey, pnr_census,
// pnr_census_cost, pnr_sgm_step, pnr_sgm_path_start, pnr_stereo_right_argmin, pnr_stereo_select,
// pnr_stereo_depth_of), so the CPU tests can hold pnr_stereo_depth's rule against the numpy oracle
// (tests/oracle_stereo.py) bit for bit, and the GPU tests can hold the kernels against this build.
// Built by tests/oracle_stereo.py with: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include <vector>
#include "../panopticnerf_b200/csrc/stereo_math.h"

extern "C" {

// The selection alone over a given S [H, W, D] u16 -> d16 [H, W]: d_R of every pixel, then pnr_stereo_select.
void emu_select(const uint16_t* S, int H, int W, int D, int U, int16_t* d16) {
  std::vector<int16_t> dr((size_t)W);
  for (int y = 0; y < H; ++y) {
    const uint16_t* srow = S + (size_t)y * W * D;
    for (int x = 0; x < W; ++x) dr[x] = (int16_t)pnr_stereo_right_argmin(srow, W, D, x);
    for (int x = 0; x < W; ++x) d16[(size_t)y * W + x] = (int16_t)pnr_stereo_select(srow + (size_t)x * D, D, U, x, dr.data());
  }
}

// One pair of H x W RGB8 images -> d16 [H, W] and depth [H, W] (depth may be NULL), S [H, W, D] u16 when S_out is not
// NULL.  The aggregation walks every path of every direction with the disparities in packed pairs, as the kernel's
// lanes hold them laid end to end.
void emu_stereo(const uint8_t* left, const uint8_t* right, int H, int W, int D, int P1, int P2, int U, float b16,
                float min_depth, float max_depth, int16_t* d16, float* depth, uint16_t* S_out) {
  const int PW = W + 8, PH = H + 6;
  std::vector<uint64_t> cen[2];
  const uint8_t* img[2] = {left, right};
  std::vector<uint8_t> g((size_t)PW * PH);
  for (int s = 0; s < 2; ++s) {
    for (int r = 0; r < PH; ++r)
      for (int c = 0; c < PW; ++c) {
        const int yy = r - 3 < 0 ? 0 : (r - 3 >= H ? H - 1 : r - 3), xx = c - 4 < 0 ? 0 : (c - 4 >= W ? W - 1 : c - 4);
        const uint8_t* px = img[s] + ((size_t)yy * W + xx) * 3;
        g[(size_t)r * PW + c] = (uint8_t)pnr_grey(px[0], px[1], px[2]);
      }
    cen[s].resize((size_t)H * W);
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) cen[s][(size_t)y * W + x] = pnr_census(&g[(size_t)y * PW + x], PW);
  }
  const int NW = D / 2;   // packed pairs per pixel
  std::vector<uint32_t> S((size_t)H * W * NW, 0u);
  static const int kDirs[8][2] = {{1, 0}, {-1, 0}, {0, 1}, {0, -1}, {1, 1}, {-1, -1}, {1, -1}, {-1, 1}};
  std::vector<uint32_t> L(NW), n(NW);
  const uint32_t p1x2 = pnr_u16x2_splat((uint32_t)P1);
  for (int r = 0; r < 8; ++r) {
    const int dx = kDirs[r][0], dy = kDirs[r][1];
    for (int path = 0; path < pnr_sgm_num_paths(dx, dy, H, W); ++path) {
      int x, y;
      pnr_sgm_path_start(dx, dy, H, W, path, &x, &y);
      for (int j = 0; j < NW; ++j) L[j] = 0;
      uint32_t m = 0;
      while (x >= 0 && x < W && y >= 0 && y < H) {
        const size_t q = (size_t)y * W + x;
        const uint64_t l = cen[0][q];
        const uint32_t m2 = pnr_u16x2_splat(m), mp2 = pnr_u16x2_splat(m + (uint32_t)P2);
        uint32_t mm = 0xFFFFu;
        for (int j = 0; j < NW; ++j) {
          const int d = 2 * j;
          const uint32_t c0 = x - d >= 0 ? pnr_census_cost(l, cen[1][q - d]) : PNR_STEREO_COST_NONE;
          const uint32_t c1 = x - d - 1 >= 0 ? pnr_census_cost(l, cen[1][q - d - 1]) : PNR_STEREO_COST_NONE;
          n[j] = pnr_sgm_step(L[j], j > 0 ? L[j - 1] : PNR_STEREO_ABSENT, j + 1 < NW ? L[j + 1] : PNR_STEREO_ABSENT,
                              c0 | (c1 << 16), m2, p1x2, mp2);
          mm = pnr_u16_min(mm, pnr_u16_min(n[j] & 0xFFFFu, n[j] >> 16));
        }
        for (int j = 0; j < NW; ++j) {
          L[j] = n[j];
          S[q * NW + j] = pnr_u16x2_add(S[q * NW + j], n[j]);
        }
        m = mm;
        x += dx;
        y += dy;
      }
    }
  }
  const uint16_t* S16 = reinterpret_cast<const uint16_t*>(S.data());
  if (S_out)
    for (size_t k = 0; k < (size_t)H * W * D; ++k) S_out[k] = S16[k];
  std::vector<int16_t> dr((size_t)H * W);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x)
      dr[(size_t)y * W + x] = (int16_t)pnr_stereo_right_argmin(S16 + (size_t)y * W * D, W, D, x);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t q = (size_t)y * W + x;
      const int v = pnr_stereo_select(S16 + q * D, D, U, x, dr.data() + (size_t)y * W);
      d16[q] = (int16_t)v;
      if (depth) depth[q] = pnr_stereo_depth_of(v, b16, min_depth, max_depth);
    }
}
}
