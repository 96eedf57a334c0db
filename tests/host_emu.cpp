// host_emu.cpp — host build of csrc/ray_math.h, so CPU tests can prove that the ray kernels' fp32 operation order
// equals the oracle's bit for bit without a GPU.  Each emu_* is a loop over rays or pixels around the ray_math.h
// routines that intersect_kernel, stratified_kernel, interval_kernel, sample_pdf_kernel and rays_kernel call.  Two
// pieces stay written out in both places, because sharing them changes the kernels' SASS: intersect_kernel's
// per-primitive step (below) and stratified_kernel's interval test (pnr_tag here).
// Built by __graft_entry__.build() and tests/host_emu.py with: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include "../panopticnerf_b200/csrc/ray_math.h"

extern "C" {

// tri_start / tris null (and T = 0): every primitive is a cuboid, as in pnr_intersect
void emu_intersect(const float* rays, int64_t R, const float* bc, const float* bh, const float* br,
                   const int32_t* tri_start, const float* tris, int64_t T, int B, int M, uint8_t* hit,
                   int32_t* box_id, float* t_in, float* t_out) {
  for (int64_t r = 0; r < R; ++r) {
    const float* q = rays + r * 6;
    PnrHitList L;
    pnr_hits_init(&L);
    for (int b = 0; b < B; ++b) {
      int k0 = 0, k1 = 0;
      if (tri_start) pnr_tri_range(tri_start, b, T, &k0, &k1);
      // intersect_kernel's per-primitive step, restated: moved into a shared function, it changes the kernel's SASS
      float tmin, tmax;
      if (!pnr_slab(q[0], q[1], q[2], q[3], q[4], q[5], bc + b * 3, bh + b * 3, br + b * 9, &tmin, &tmax)) continue;
      if (k0 == k1) {
        pnr_hits_insert(&L, M, tmin, tmax, b);
        continue;
      }
      const PnrShear S = pnr_shear(q[3], q[4], q[5]);
      PnrMeshCross X;
      pnr_cross_init(&X);
      for (int k = k0; k < k1; ++k) {
        float t;
        if (pnr_tri_cross(q[0], q[1], q[2], S, tris + (int64_t)k * 9, &t)) pnr_cross_add(&X, M, t);
      }
      pnr_cross_emit(&X, &L, M, b);
    }
    pnr_hits_store(&L, M, r, hit, box_id, t_in, t_out);
  }
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
}
