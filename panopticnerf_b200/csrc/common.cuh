// common.cuh — error plumbing, launch accounting and per-device launch facts shared by the libpnr translation units.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <mutex>
#include <set>
#include <utility>
#include <cuda_runtime.h>
#include "../../include/pnr.h"

namespace pnr {

int set_error(int code, const char* fmt, ...);   // stores a thread-local message, returns code
void count_launch(int n = 1);
// fixed (bounding-box) one-hot maps from per-sample weights (stream_kernels.cu; used by pnr_mlp_composite)
int launch_fixed_maps(const float* weights, const int32_t* sample_box, const int32_t* box_sem, const int32_t* box_inst,
                      int64_t R, int N, int C, int K, int B, float* fsem, float* finst, cudaStream_t stream);
// pnr_sample_pdf with an explicit row stride for u (ray_kernels.cu; used by pnr_render_fused)
int sample_pdf_strided(const float* z, const float* weights, int64_t R, int32_t N, int32_t Ni, const float* u,
                       int64_t u_stride, float* z_fine, int64_t* idx, float* z_all, void* stream);
// the host checks of a sequence table's frame fields against B primitives (ray_kernels.cu; pnr_intersect_frames and
// pnr_render_fused_frames name themselves with fn)
int check_frame_table(const char* fn, const pnr_frame_table* fr, int32_t B);
// a5 on B primitives, with their meshes (mesh_tri_start / mesh_tris null and T = 0: cuboids only) and frame table
// (fr null: every primitive static) (ray_kernels.cu; the pnr_intersect* entry points and pnr_render_fused*).  fn: the
// entry point's name in the error messages.
int intersect_rays(const char* fn, const float* rays, int64_t R, const float* box_center, const float* box_half,
                   const float* box_rot, const int32_t* mesh_tri_start, const float* mesh_tris, int64_t T, int32_t B,
                   int32_t M, uint8_t* hit_mask, int32_t* box_id, float* t_in, float* t_out, const pnr_frame_table* fr,
                   void* stream);

#define PNR_CHECK_ARG(cond, ...) \
  do { if (!(cond)) return ::pnr::set_error(PNR_ERR_ARG, __VA_ARGS__); } while (0)

#define PNR_CUDA(call)                                                                         \
  do {                                                                                         \
    cudaError_t e__ = (call);                                                                  \
    if (e__ != cudaSuccess)                                                                    \
      return ::pnr::set_error(PNR_ERR_CUDA, "%s failed: %s (%s:%d)", #call,                    \
                              cudaGetErrorString(e__), __FILE__, __LINE__);                    \
  } while (0)

#define PNR_LAUNCH_CHECK(name)                                                                 \
  do {                                                                                         \
    cudaError_t e__ = cudaGetLastError();                                                      \
    if (e__ != cudaSuccess)                                                                    \
      return ::pnr::set_error(PNR_ERR_CUDA, "launch of %s failed: %s", name,                   \
                              cudaGetErrorString(e__));                                        \
    ::pnr::count_launch();                                                                     \
  } while (0)

constexpr int kMaxDevices = 64;

// SM count of device `dev` (cached per device; every per-device fact in this library is indexed by ordinal).
inline int num_sms(int dev) {
  static int n[kMaxDevices] = {0};
  if (dev < 0 || dev >= kMaxDevices) return 132;
  if (n[dev] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev] = v > 0 ? v : 132;
  }
  return n[dev];
}
inline int num_sms() {   // of the current device
  int dev = 0;
  cudaGetDevice(&dev);
  return num_sms(dev);
}

// The current device into *out; refused (`what` names the entry point) when its ordinal is past the per-device tables.
inline int current_device(const char* what, int* out) {
  int dev = 0;
  PNR_CUDA(cudaGetDevice(&dev));
  PNR_CHECK_ARG(dev >= 0 && dev < kMaxDevices, "%s: device ordinal %d >= %d", what, dev, kMaxDevices);
  *out = dev;
  return PNR_OK;
}

// The camera table of a frame-set call (pnr_sample_ray_batch, pnr_project_depth; fn names it): 1..MAX cameras, each a
// pinhole (0) or fisheye (2) of H, W in [1, 2^size_bits) (size_bits = 31: any positive int32).
inline int check_cameras(const char* fn, const pnr_ray_camera* cams, int32_t n, int size_bits) {
  PNR_CHECK_ARG(n >= 1 && n <= PNR_RAY_BATCH_MAX_CAMERAS, "%s: num_cameras=%d outside [1,%d]", fn, n,
                PNR_RAY_BATCH_MAX_CAMERAS);
  for (int k = 0; k < n; ++k) {
    const pnr_ray_camera& c = cams[k];
    PNR_CHECK_ARG(c.model != 1, "%s: camera %d is equirect (model 1): its rays are device-only (sincosf), so frame "
                  "sets take pinhole (0) and fisheye (2) cameras", fn, k);
    PNR_CHECK_ARG(c.model == 0 || c.model == 2, "%s: camera %d model %d (0 pinhole, 2 fisheye)", fn, k, c.model);
    PNR_CHECK_ARG(c.H >= 1 && c.W >= 1 && (int64_t)c.H < (int64_t(1) << size_bits) &&
                  (int64_t)c.W < (int64_t(1) << size_bits),
                  "%s: camera %d size H=%d W=%d outside [1, 2^%d)", fn, k, c.H, c.W, size_bits);
  }
  return PNR_OK;
}

// Lets `kernel` use `bytes` (> 48 KB) of dynamic shared memory on device `dev`.  The opt-in is a per-device function
// attribute: it is set once per (kernel, device).
inline int opt_in_smem(const void* kernel, int bytes, int dev) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  std::lock_guard<std::mutex> lock(mu);
  if (done.count({kernel, dev}) == 0) {
    PNR_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done.insert({kernel, dev});
  }
  return PNR_OK;
}

// Makes `dev` current for a scope and restores the caller's device afterwards (the library never leaves the
// process on a different device than it found it - PyTorch's notion of the current device stays intact).
struct DeviceGuard {
  int prev = -1;
  bool changed = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) changed = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    if (changed) cudaSetDevice(prev);
  }
};

}  // namespace pnr
