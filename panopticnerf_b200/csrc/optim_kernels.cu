// optim_kernels.cu — the optimiser of the training path: pnr_adam_step, Adam over one flat fp32 parameter vector whose
// gradient is the rank-ordered sum of G gradient slices (the all-gathered gradients of G data-parallel ranks).
//
// Every operation is an explicitly rounded intrinsic (__fadd_rn, __fmul_rn, __fdiv_rn, __fsqrt_rn), which nvcc never
// contracts into an FMA: a float32 host restatement of the same order (tests/test_gpu_data_parallel.py) reproduces the
// kernel bit for bit, and so does every rank that runs it on the same gathered slices.
#include <cmath>
#include "common.cuh"

namespace pnr {
namespace {

struct AdamConsts {
  float w1, w1c;      // lerp weight 1 - beta1 as torch receives it, and 1 - w1 (torch's lerp rule for w1 >= 0.5)
  float beta2, w2;    // beta2 and 1 - beta2
  float eps, wd, neg_step, bc2;
};

// torch.optim.Adam's single-tensor update of one element, operation for operation (see include/pnr.h).
__device__ __forceinline__ void adam_element(float g, float& p, float& m, float& v, const AdamConsts& k) {
  if (k.wd != 0.0f) g = __fadd_rn(g, __fmul_rn(k.wd, p));
  const float d = __fsub_rn(g, m);
  m = k.w1 < 0.5f ? __fadd_rn(m, __fmul_rn(k.w1, d)) : __fsub_rn(g, __fmul_rn(d, k.w1c));
  v = __fadd_rn(__fmul_rn(v, k.beta2), __fmul_rn(__fmul_rn(k.w2, g), g));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), k.bc2), k.eps);
  p = __fadd_rn(p, __fmul_rn(k.neg_step, __fdiv_rn(m, denom)));
}

struct AdamPtrs {
  const float* grads; float* p; float* m; float* v; float* grad_sum;
  int64_t P, ld; int G;
};

constexpr int kAdamThreads = 256;
constexpr int64_t kAdamMaxBlocks = 8192;

// 16-byte path: element quads [0, P/4) by float4, the P % 4 tail elements by the first threads of the grid.
__global__ void __launch_bounds__(kAdamThreads) adam_vec4_kernel(AdamPtrs a, AdamConsts k) {
  const int64_t nq = a.P >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int64_t q = t0; q < nq; q += stride) {
    float4 g = __ldg(reinterpret_cast<const float4*>(a.grads) + q);
    for (int s = 1; s < a.G; ++s) {
      const float4 h = __ldg(reinterpret_cast<const float4*>(a.grads + s * a.ld) + q);
      g.x = __fadd_rn(g.x, h.x); g.y = __fadd_rn(g.y, h.y); g.z = __fadd_rn(g.z, h.z); g.w = __fadd_rn(g.w, h.w);
    }
    if (a.grad_sum) reinterpret_cast<float4*>(a.grad_sum)[q] = g;
    float4 p = reinterpret_cast<const float4*>(a.p)[q];
    float4 m = reinterpret_cast<const float4*>(a.m)[q];
    float4 v = reinterpret_cast<const float4*>(a.v)[q];
    adam_element(g.x, p.x, m.x, v.x, k);
    adam_element(g.y, p.y, m.y, v.y, k);
    adam_element(g.z, p.z, m.z, v.z, k);
    adam_element(g.w, p.w, m.w, v.w, k);
    reinterpret_cast<float4*>(a.p)[q] = p;
    reinterpret_cast<float4*>(a.m)[q] = m;
    reinterpret_cast<float4*>(a.v)[q] = v;
  }
  const int64_t i = 4 * nq + t0;
  if (i < a.P) {
    float g = a.grads[i];
    for (int s = 1; s < a.G; ++s) g = __fadd_rn(g, a.grads[s * a.ld + i]);
    if (a.grad_sum) a.grad_sum[i] = g;
    adam_element(g, a.p[i], a.m[i], a.v[i], k);
  }
}

// Any alignment (a slice stride that is not a multiple of four floats, or a buffer offset by a partial quad).
__global__ void __launch_bounds__(kAdamThreads) adam_scalar_kernel(AdamPtrs a, AdamConsts k) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.P; i += stride) {
    float g = a.grads[i];
    for (int s = 1; s < a.G; ++s) g = __fadd_rn(g, a.grads[s * a.ld + i]);
    if (a.grad_sum) a.grad_sum[i] = g;
    adam_element(g, a.p[i], a.m[i], a.v[i], k);
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace
}  // namespace pnr

using namespace pnr;

extern "C" int pnr_adam_step(const float* grads, float* param, float* exp_avg, float* exp_avg_sq,
                             const pnr_adam_args* a, float* grad_sum, void* stream) {
  PNR_CHECK_ARG(a, "pnr_adam_step: null args");
  PNR_CHECK_ARG(a->G >= 1, "pnr_adam_step: G=%d < 1", a->G);
  PNR_CHECK_ARG(a->P >= 0, "pnr_adam_step: P=%lld < 0", (long long)a->P);
  PNR_CHECK_ARG(a->ld_grad >= a->P, "pnr_adam_step: ld_grad=%lld < P=%lld", (long long)a->ld_grad, (long long)a->P);
  PNR_CHECK_ARG(a->ld_grad <= INT64_MAX / a->G, "pnr_adam_step: G * ld_grad overflows");
  PNR_CHECK_ARG(std::isfinite(a->beta1) && a->beta1 >= 0.0 && a->beta1 < 1.0, "pnr_adam_step: beta1=%g outside [0,1)", a->beta1);
  PNR_CHECK_ARG(std::isfinite(a->beta2) && a->beta2 >= 0.0 && a->beta2 < 1.0, "pnr_adam_step: beta2=%g outside [0,1)", a->beta2);
  PNR_CHECK_ARG(std::isfinite(a->eps) && a->eps >= 0.0f, "pnr_adam_step: eps=%g (finite, >= 0)", (double)a->eps);
  PNR_CHECK_ARG(std::isfinite(a->weight_decay) && a->weight_decay >= 0.0f,
                "pnr_adam_step: weight_decay=%g (finite, >= 0)", (double)a->weight_decay);
  PNR_CHECK_ARG(std::isfinite(a->step_size) && a->step_size >= 0.0f, "pnr_adam_step: step_size=%g (finite, >= 0)",
                (double)a->step_size);
  PNR_CHECK_ARG(std::isfinite(a->bc2_sqrt) && a->bc2_sqrt > 0.0f, "pnr_adam_step: bc2_sqrt=%g (finite, > 0)",
                (double)a->bc2_sqrt);
  if (a->P == 0) return PNR_OK;
  PNR_CHECK_ARG(grads, "pnr_adam_step: null grads");
  PNR_CHECK_ARG(param, "pnr_adam_step: null param");
  PNR_CHECK_ARG(exp_avg, "pnr_adam_step: null exp_avg");
  PNR_CHECK_ARG(exp_avg_sq, "pnr_adam_step: null exp_avg_sq");

  AdamConsts k;
  k.w1 = (float)(1.0 - a->beta1);
  k.w1c = 1.0f - k.w1;
  k.beta2 = (float)a->beta2;
  k.w2 = (float)(1.0 - a->beta2);
  k.eps = a->eps; k.wd = a->weight_decay; k.neg_step = -a->step_size; k.bc2 = a->bc2_sqrt;
  const AdamPtrs p{grads, param, exp_avg, exp_avg_sq, grad_sum, a->P, a->ld_grad, a->G};
  const bool vec = (a->ld_grad & 3) == 0 && aligned16(grads) && aligned16(param) && aligned16(exp_avg) &&
                   aligned16(exp_avg_sq) && (!grad_sum || aligned16(grad_sum));
  const int64_t items = vec ? (a->P + 3) / 4 : a->P;
  const unsigned blocks = (unsigned)std::min<int64_t>((items + kAdamThreads - 1) / kAdamThreads, kAdamMaxBlocks);
  if (vec) {
    adam_vec4_kernel<<<blocks, kAdamThreads, 0, (cudaStream_t)stream>>>(p, k);
    PNR_LAUNCH_CHECK("adam_vec4_kernel");
  } else {
    adam_scalar_kernel<<<blocks, kAdamThreads, 0, (cudaStream_t)stream>>>(p, k);
    PNR_LAUNCH_CHECK("adam_scalar_kernel");
  }
  return PNR_OK;
}
