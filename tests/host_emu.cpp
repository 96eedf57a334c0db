// host_emu.cpp — host build of csrc/ray_math.h, so CPU tests can prove that the ray kernels' fp32 operation order
// equals the oracle's bit for bit without a GPU.  Each emu_* is a loop over rays or pixels around the ray_math.h
// routines that intersect_kernel, stratified_kernel, interval_kernel, sample_pdf_kernel, rays_kernel and
// ray_batch_kernel call.  One piece stays written out in both places: stratified_kernel's interval test (pnr_tag here),
// because a predicate shared with pnr_tag changes the SASS of pnr_tag's callers.
// Built by __graft_entry__.build() and tests/host_emu.py with: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include "../panopticnerf_b200/csrc/ray_math.h"

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
}
