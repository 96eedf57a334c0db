// host_emu_lidar.cpp — host build of the LiDAR depth routines of csrc/ray_math.h (pnr_project_point, pnr_depth_frame,
// pnr_depth_pixel), so the CPU tests can hold pnr_project_depth's operation order against the numpy oracle
// (tests/oracle_lidar.py) bit for bit, and the GPU tests can hold the kernels against this build.
// Built by tests/test_cpu_lidar_depth.py's fixture with: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include <vector>
#include "../panopticnerf_b200/csrc/ray_math.h"

extern "C" {

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
}
