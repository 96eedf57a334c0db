// host_emu_sequence.cpp — host build of pnr_intersect_frames (csrc/ray_math.h; DESIGN 3.2), so the CPU tests can
// compare a sequence table's intersection with the per-frame oracle (tests/oracle_sequence.py) bit for bit without a
// GPU.  emu_intersect_frames is intersect_kernel<kMeshes, true>'s loop: the static primitives [0, S), then the block of
// the ray's frame (pnr_frame_range).  The per-primitive step is written out again here, as in tests/host_emu.cpp,
// because moving it into a function the kernel shares changes the kernel's SASS.
// Built by the `emu_seq` fixture of tests/oracle_sequence.py with: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include "../panopticnerf_b200/csrc/ray_math.h"

// intersect_kernel's per-primitive step for primitive b (tri_start null: every primitive is a cuboid)
static void step(const float* q, const float* bc, const float* bh, const float* br, const int32_t* tri_start,
                 const float* tris, int64_t T, int b, int M, PnrHitList* L) {
  int k0 = 0, k1 = 0;
  if (tri_start) pnr_tri_range(tri_start, b, T, &k0, &k1);
  float tmin, tmax;
  if (!pnr_slab(q[0], q[1], q[2], q[3], q[4], q[5], bc + b * 3, bh + b * 3, br + b * 9, &tmin, &tmax)) return;
  if (k0 == k1) {
    pnr_hits_insert(L, M, tmin, tmax, b);
    return;
  }
  const PnrShear S = pnr_shear(q[3], q[4], q[5]);
  PnrMeshCross X;
  pnr_cross_init(&X);
  for (int k = k0; k < k1; ++k) {
    float t;
    if (pnr_tri_cross(q[0], q[1], q[2], S, tris + (int64_t)k * 9, &t)) pnr_cross_add(&X, M, t);
  }
  pnr_cross_emit(&X, L, M, b);
}

extern "C" {

// a sequence table of B primitives, S of them static, F >= 1 frames (no argument checks: the tests pass valid tables)
void emu_intersect_frames(const float* rays, int64_t R, const float* bc, const float* bh, const float* br,
                          const int32_t* tri_start, const float* tris, int64_t T, int B, int S,
                          const int32_t* frame_boxes, int F, const int32_t* ray_frame, int M, uint8_t* hit,
                          int32_t* box_id, float* t_in, float* t_out) {
  for (int64_t r = 0; r < R; ++r) {
    PnrHitList L;
    pnr_hits_init(&L);
    for (int b = 0; b < S; ++b) step(rays + r * 6, bc, bh, br, tri_start, tris, T, b, M, &L);
    int b0, b1;
    pnr_frame_range(ray_frame[r], frame_boxes, F, S, B, &b0, &b1);
    for (int b = b0; b < b1; ++b) step(rays + r * 6, bc, bh, br, tri_start, tris, T, b, M, &L);
    pnr_hits_store(&L, M, r, hit, box_id, t_in, t_out);
  }
}
}
