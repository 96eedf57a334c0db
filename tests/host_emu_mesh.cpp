// host_emu_mesh.cpp — host build of the mesh-primitive routines of csrc/ray_math.h (pnr_shear, pnr_tri_cross,
// PnrMeshCross) in the order intersect_kernel<true> calls them, so CPU tests can prove the fp32 operation order equals
// the oracle's bit for bit without a GPU.  Built by tests/test_cpu_mesh_primitives.py with:
// g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include "../panopticnerf_b200/csrc/ray_math.h"

extern "C" {

void emu_intersect_meshes(const float* rays, int64_t R, const float* bc, const float* bh, const float* br,
                          const int32_t* tri_start, const float* tris, int64_t T, int B, int M, uint8_t* hit,
                          int32_t* box_id, float* t_in, float* t_out) {
  for (int64_t r = 0; r < R; ++r) {
    const float* q = rays + r * 6;
    PnrHitList L;
    pnr_hits_init(&L);
    for (int b = 0; b < B; ++b) {
      int64_t k0 = tri_start[b] < 0 ? 0 : tri_start[b];
      if (k0 > T) k0 = T;
      int64_t k1 = tri_start[b + 1] < k0 ? k0 : tri_start[b + 1];
      if (k1 > T) k1 = T;
      float tmin, tmax;
      const bool h = pnr_slab(q[0], q[1], q[2], q[3], q[4], q[5], bc + b * 3, bh + b * 3, br + b * 9, &tmin, &tmax);
      if (!h) continue;
      if (k0 == k1) {
        pnr_hits_insert(&L, M, tmin, tmax, b);
        continue;
      }
      const PnrShear S = pnr_shear(q[3], q[4], q[5]);
      PnrMeshCross X;
      pnr_cross_init(&X);
      for (int64_t k = k0; k < k1; ++k) {
        float t;
        if (pnr_tri_cross(q[0], q[1], q[2], S, tris + k * 9, &t)) pnr_cross_add(&X, M, t);
      }
      pnr_cross_emit(&X, &L, M, b);
    }
    hit[r] = L.n > 0;
    for (int m = 0; m < M; ++m) {
      const bool v = m < L.n;
      box_id[r * M + m] = v ? L.id[m] : -1;
      t_in[r * M + m] = v ? pnr_max_nan(L.key[m], 0.f) : 0.f;
      t_out[r * M + m] = v ? L.tout[m] : 0.f;
    }
  }
}
}
