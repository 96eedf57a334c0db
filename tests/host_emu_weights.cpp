// host_emu_weights.cpp — host build of the weighted-draw routines of csrc/ray_math.h (pnr_pixel_weight,
// pnr_weight_of_pixel, pnr_weighted_pixel, pnr_ray_batch_row<true>), so the CPU tests can hold the kernels of
// pnr_pixel_weights and pnr_sample_ray_batch_weighted against the numpy oracle (tests/oracle_pixel_weights.py) bit for
// bit without a GPU.  Each emu_* is the kernel's loop around the same routine.  Built with the flags of host_emu.cpp
// (-ffp-contract=off) by __graft_entry__.build() and tests/oracle_pixel_weights.py's host_lib() through
// _build.build_host_emu_weights().
#include <cstdint>
#include "../panopticnerf_b200/csrc/ray_math.h"

extern "C" {

// ray_batch_weighted_kernel's loop: the pixel drawn through the weight table (pnr_ray_batch_row<true>; the tests pass
// a table that agrees with its sums, and no argument checks are made)
void emu_sample_ray_batch_weighted(const pnr_ray_batch_args* a, const pnr_ray_batch_weights* w) {
  for (int64_t r = a->r0; r < a->r1; ++r) pnr_ray_batch_row<true>(*a, a->pix_offset, r, w);
}

// the weighted pick alone, for one x
int64_t emu_weighted_pixel(const uint16_t* weight, const uint64_t* cum, int64_t P, uint64_t x) {
  return pnr_weighted_pixel(weight, cum, P, x);
}

// the composition rule alone, for n (keep, frame factor, class factor) triples
void emu_pixel_weight(const uint8_t* keep, float scale, const float* ff, const float* cf, int64_t n, uint16_t* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = pnr_pixel_weight(keep[i] != 0, scale, ff[i], cf[i]);
}

// pixel_weights_kernel's loop with host pointers: every frame, each of its clamped pixels
void emu_pixel_weights(const pnr_pixel_weights_args* a) {
  for (int f = 0; f < a->F; ++f) {
    int64_t lo, hi;
    const int cam = pnr_depth_frame(a->frame_cam, a->pix_offset, a->num_cameras, a->P, f, &lo, &hi);
    for (int64_t q = 0; q < hi - lo; ++q) a->weight[lo + q] = pnr_weight_of_pixel(*a, f, cam, lo, q);
  }
}
}
