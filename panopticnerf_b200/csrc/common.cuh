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
