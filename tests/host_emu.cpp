// host_emu.cpp — host build of csrc/ray_math.h and csrc/stereo_math.h, so CPU tests can prove that the kernels' fp32
// operation order equals the oracle's bit for bit without a GPU.  Each emu_* is a loop over rays, pixels or points
// around the routines that intersect_kernel, stratified_kernel, interval_kernel, sample_pdf_kernel, rays_kernel,
// ray_batch_kernel, the depth kernels of pnr_project_depth and the stereo kernels of pnr_stereo_depth call.  One piece
// stays written out in both places: stratified_kernel's interval test (pnr_tag here), because a predicate shared with
// pnr_tag changes the SASS of pnr_tag's callers.
// Built by __graft_entry__.build() and the `emu` fixture through tests/host_emu.py's build_host_emu().
#include <cstdint>
#include <vector>
#include "../panopticnerf_b200/csrc/ray_math.h"
#include "../panopticnerf_b200/csrc/stereo_math.h"

// primitive b of ray o, read as intersect_kernel reads it: the box as 15 floats and the clamped triangle range
// (tri_start null: every primitive is a cuboid)
static void prim_step(const float* o, const float* bc, const float* bh, const float* br, const int32_t* tri_start,
                      const float* tris, int64_t T, int b, int M, PnrHitList* L) {
  float q[15];
  for (int e = 0; e < 3; ++e) { q[e] = bc[b * 3 + e]; q[3 + e] = bh[b * 3 + e]; }
  for (int e = 0; e < 9; ++e) q[6 + e] = br[b * 9 + e];
  int k0 = 0, k1 = 0;
  if (tri_start) pnr_tri_range(tri_start, b, T, &k0, &k1);
  pnr_prim_step(o[0], o[1], o[2], o[3], o[4], o[5], q, k0, k1, tris, M, b, L);
}

extern "C" {

// intersect_kernel's loop on a sequence table of B primitives (DESIGN 3.2): the static primitives [0, S), then the
// block of the ray's frame.  ray_frame null (and F = 0): every primitive is static.  No argument checks: the tests
// pass valid tables.
void emu_intersect_frames(const float* rays, int64_t R, const float* bc, const float* bh, const float* br,
                          const int32_t* tri_start, const float* tris, int64_t T, int B, int S,
                          const int32_t* frame_boxes, int F, const int32_t* ray_frame, int M, uint8_t* hit,
                          int32_t* box_id, float* t_in, float* t_out) {
  for (int64_t r = 0; r < R; ++r) {
    PnrHitList L;
    pnr_hits_init(&L);
    for (int b = 0; b < S; ++b) prim_step(rays + r * 6, bc, bh, br, tri_start, tris, T, b, M, &L);
    int b0, b1;
    pnr_frame_range(ray_frame ? ray_frame[r] : -1, frame_boxes, F, S, B, &b0, &b1);
    for (int b = b0; b < b1; ++b) prim_step(rays + r * 6, bc, bh, br, tri_start, tris, T, b, M, &L);
    pnr_hits_store(&L, M, r, hit, box_id, t_in, t_out);
  }
}

// a single table of B primitives, as pnr_intersect / pnr_intersect_meshes
void emu_intersect(const float* rays, int64_t R, const float* bc, const float* bh, const float* br,
                   const int32_t* tri_start, const float* tris, int64_t T, int B, int M, uint8_t* hit,
                   int32_t* box_id, float* t_in, float* t_out) {
  emu_intersect_frames(rays, R, bc, bh, br, tri_start, tris, T, B, B, nullptr, 0, nullptr, M, hit, box_id, t_in,
                       t_out);
}

void emu_stratified(const float* near, const float* far, const float* t_vals, const float* u, int64_t R, int N,
                    float perturb, const int32_t* box_id, const float* t_in, const float* t_out, int M, float* z,
                    int32_t* sb) {
  for (int64_t r = 0; r < R; ++r)
    for (int i = 0; i < N; ++i) {
      z[r * N + i] = pnr_sample_z(near[r], far[r], t_vals, u + r * N, i, N, perturb);
      if (sb) sb[r * N + i] = pnr_tag(z[r * N + i], box_id + r * M, t_in + r * M, t_out + r * M, M);
    }
}

void emu_intervals(const float* near, const float* far, const float* t_vals, const float* u, int64_t R, int N,
                   float perturb, const int32_t* box_id, const float* t_in, const float* t_out, int M, float* z,
                   int32_t* sb) {
  for (int64_t r = 0; r < R; ++r) {
    PnrIntervalPlan P;
    pnr_interval_plan(near[r], far[r], box_id + r * M, t_in + r * M, t_out + r * M, M, N, &P);
    float* zr = z + r * N;
    if (P.kept == 0) {   // no kept interval: the uniform rule, untagged
      for (int i = 0; i < N; ++i) {
        zr[i] = pnr_sample_z(near[r], far[r], t_vals, u + r * N, i, N, perturb);
        sb[r * N + i] = -1;
      }
      continue;
    }
    for (int k = 0; k < N; ++k) zr[k] = pnr_interval_slot_z(&P, u + r * N, k, perturb);
    for (int i = 1; i < N; ++i) {   // insertion sort: the kernel's bitonic network yields the same sorted array
      const float v = zr[i];
      int j = i - 1;
      while (j >= 0 && zr[j] > v) { zr[j + 1] = zr[j]; --j; }
      zr[j + 1] = v;
    }
    for (int i = 0; i < N; ++i) sb[r * N + i] = pnr_tag(zr[i], box_id + r * M, t_in + r * M, t_out + r * M, M);
  }
}

void emu_sample_pdf(const float* z, const float* w, int64_t R, int N, int Ni, const float* u, float* z_f,
                    int64_t* idx) {
  float cdf[256];
  for (int64_t r = 0; r < R; ++r) {
    pnr_pdf_cdf(w + r * N, N, cdf);
    for (int j = 0; j < Ni; ++j) {
      int id;
      z_f[r * Ni + j] = pnr_pdf_sample(z + r * N, cdf, N - 1, u[r * Ni + j], &id);
      idx[r * Ni + j] = id;
    }
  }
}

// camera 0 (pinhole, intr = fx, fy, cx, cy) or 2 (fisheye, + xi, k1, k2), as pnr_generate_rays; returns -1 for any
// other camera: the equirect camera is device-only, because host and device sincosf round differently
int emu_generate_rays(int H, int W, int row0, int rows, int camera, const float* intr, const float* c2w,
                      float* rays) {
  if (camera != 0 && camera != 2) return -1;
  for (int64_t i = 0; i < (int64_t)rows * W; ++i) {
    const int v = row0 + (int)(i / W), u = (int)(i % W);
    float x, y, z;
    if (camera == 0)
      pnr_pinhole_dir((float)u, (float)v, intr[0], intr[1], intr[2], intr[3], &x, &y, &z);
    else
      pnr_fisheye_dir((float)u, (float)v, intr[0], intr[1], intr[2], intr[3], intr[4], intr[5], intr[6], &x, &y, &z);
    float* o = rays + i * 6;
    o[0] = c2w[3]; o[1] = c2w[7]; o[2] = c2w[11];
    pnr_cam_to_world(c2w, x, y, z, o + 3, o + 4, o + 5);
  }
  return 0;
}

// ray_batch_kernel's loop over pnr_ray_batch_row: rows r0 .. r1-1 with host pointers (no argument checks: the tests
// pass valid sets)
void emu_sample_ray_batch(const pnr_ray_batch_args* a) {
  for (int64_t r = a->r0; r < a->r1; ++r) pnr_ray_batch_row(*a, a->pix_offset, r);
}

// one Philox4x32-10 block
void emu_philox4x32_10(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  pnr_philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1], out);
}

uint64_t emu_mulhi64(uint64_t a, uint64_t b) { return pnr_mulhi64(a, b); }

// one point: 1 and (*pix, *t) when it lands, else 0
int emu_project_point(const pnr_ray_camera* cam, const float* M, float x, float y, float z, float min_depth,
                      float max_depth, int64_t* pix, float* t) {
  return pnr_project_point(*cam, M, x, y, z, min_depth, max_depth, pix, t) ? 1 : 0;
}

// the whole of pnr_project_depth with host pointers (points, frame_cam, pix_offset and depth on the host; no argument
// checks: the tests pass valid tables): fill the named frames with +Inf, every (pair, point) in order, a plain
// minimum on the bits, then the final pass into depth
void emu_project_depth(const pnr_project_depth_args* a) {
  std::vector<uint32_t> z((size_t)a->P, PNR_DEPTH_NONE);
  std::vector<char> named((size_t)a->F, 0);
  for (int k = 0; k < a->Q; ++k) named[a->pair_frame[k]] = 1;
  for (int k = 0; k < a->Q; ++k) {
    const int f = a->pair_frame[k], s = a->pair_scan[k];
    int64_t lo, hi;
    const pnr_ray_camera& c = a->cams[pnr_depth_frame(a->frame_cam, a->pix_offset, a->num_cameras, a->P, f, &lo, &hi)];
    for (int64_t i = a->scan_offset[s]; i < a->scan_offset[s + 1]; ++i) {
      const float* p = a->points + i * 4;
      int64_t pix;
      float t;
      if (pnr_project_point(c, a->pair_M + (int64_t)k * 12, p[0], p[1], p[2], a->min_depth, a->max_depth, &pix, &t) &&
          lo + pix < hi) {
        const uint32_t b = pnr_float_bits(t);
        if (b < z[lo + pix]) z[lo + pix] = b;
      }
    }
  }
  for (int f = 0; f < a->F; ++f) {
    if (!named[f]) continue;
    int64_t lo, hi;
    const pnr_ray_camera& c = a->cams[pnr_depth_frame(a->frame_cam, a->pix_offset, a->num_cameras, a->P, f, &lo, &hi)];
    for (int64_t q = 0; q < hi - lo; ++q)
      a->depth[lo + q] = pnr_depth_pixel(z.data() + lo, hi - lo, c.W, c.H, q, a->occlusion_radius, a->occlusion_margin);
  }
}

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
