// stream_kernels.cu — the floating-point HBM-bound stages: standalone positional encoding
// (SURVEY.md 8(a) a7) and alpha compositing / raw2outputs (a9).
//   encode    : 128 samples per CTA, each thread encodes one sample into a shared tile, the CTA then
//               streams the contiguous [128, 3+6L] tile out with fully coalesced stores.
//   composite : one warp per ray; lanes stride the sample axis; transmittance is an exclusive
//               product scan done with warp shuffles; per-class logits are accumulated with lanes
//               striding the (contiguous) channel axis so every raw row is read once, coalesced.
#include "common.cuh"
#include "composite_math.cuh"
#include "ray_math.h"

namespace pnr {

// ------------------------------------------------------------------------------------ a7 encode
constexpr int kEncTile = 128;

__global__ void __launch_bounds__(kEncTile) encode_kernel(const float* __restrict__ x, int64_t n, int L,
                                                          float* __restrict__ out) {
  extern __shared__ float tile[];  // [kEncTile][E]
  const int E = 3 + 6 * L;
  const int64_t s0 = (int64_t)blockIdx.x * kEncTile;
  const int64_t s = s0 + threadIdx.x;
  if (s < n) {
    float* row = tile + threadIdx.x * E;
    float p[3] = {x[s * 3 + 0], x[s * 3 + 1], x[s * 3 + 2]};
    row[0] = p[0]; row[1] = p[1]; row[2] = p[2];
    float f = 1.0f;
    for (int k = 0; k < L; ++k) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float sn, cs;
        sincosf(p[c] * f, &sn, &cs);  // exact power-of-two scaling, accurate sin/cos
        row[3 + 6 * k + c] = sn;
        row[3 + 6 * k + 3 + c] = cs;
      }
      f *= 2.0f;
    }
  }
  __syncthreads();
  const int64_t cnt = (int64_t)min((int64_t)kEncTile, n - s0) * E;
  float* dst = out + s0 * E;
  for (int64_t i = threadIdx.x; i < cnt; i += kEncTile) dst[i] = tile[i];
}

// ------------------------------------------------------------------------------------ ray generation
struct CamArgs { float fx, fy, cx, cy; float xi, k1, k2; float c2w[12]; int H, W, row0, rows, camera; };

__global__ void __launch_bounds__(256) rays_kernel(CamArgs a, float* __restrict__ rays) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)a.rows * a.W) return;
  const int v = a.row0 + (int)(i / a.W), u = (int)(i % a.W);
  float x, y, z;
  if (a.camera == 0) {  // pinhole; every op separately rounded so the result equals the oracle's bit for bit
    x = __fdiv_rn(__fsub_rn((float)u, a.cx), a.fx);
    y = __fdiv_rn(__fsub_rn((float)v, a.cy), a.fy);
    z = 1.0f;
  } else if (a.camera == 2) {   // KITTI-360 fisheye (MEI): ray_math.h, also compiled for the host by the CPU tests
    pnr_fisheye_dir((float)u, (float)v, a.fx, a.fy, a.cx, a.cy, a.xi, a.k1, a.k2, &x, &y, &z);
  } else {
    const float lon = __fmul_rn(__fsub_rn(__fdiv_rn((float)u, (float)a.W), 0.5f), 6.2831853071795864769f);
    const float lat = __fmul_rn(__fsub_rn(0.5f, __fdiv_rn((float)v, (float)a.H)), 3.14159265358979323846f);
    float sl, cl, so, co;
    sincosf(lat, &sl, &cl);
    sincosf(lon, &so, &co);
    x = cl * so; y = -sl; z = cl * co;
  }
  float2* o = reinterpret_cast<float2*>(rays + i * 6);
  const float d0 = __fadd_rn(__fadd_rn(__fmul_rn(a.c2w[0], x), __fmul_rn(a.c2w[1], y)), __fmul_rn(a.c2w[2], z));
  const float d1 = __fadd_rn(__fadd_rn(__fmul_rn(a.c2w[4], x), __fmul_rn(a.c2w[5], y)), __fmul_rn(a.c2w[6], z));
  const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(a.c2w[8], x), __fmul_rn(a.c2w[9], y)), __fmul_rn(a.c2w[10], z));
  o[0] = make_float2(a.c2w[3], a.c2w[7]);
  o[1] = make_float2(a.c2w[11], d0);
  o[2] = make_float2(d1, d2);
}

// ------------------------------------------------------------------------------------ a9 composite
constexpr int kCompMaxPerLane = 8;   // N <= 256
constexpr int kCompMaxChan = 4;      // C, K <= 128 each
constexpr int kCompWarps = 4;

struct CompositeArgs {
  const float* raw; const float* z; const float* rays;
  int64_t R; int N, C, K, CH;
  int white_bkgd, sem_softmax, mask_outside;
  const int32_t* sample_box; const int32_t* box_sem; const int32_t* box_inst; int B;
  pnr_composite_out o;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, d));
  return v;
}

__global__ void __launch_bounds__(kCompWarps * 32) composite_kernel(CompositeArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kCompWarps + (threadIdx.x >> 5);
  if (r >= a.R) return;
  const int N = a.N, CH = a.CH;
  const float* raw = a.raw + r * N * CH;
  const float* z = a.z + r * N;
  const float dx = a.rays[r * 6 + 3], dy = a.rays[r * 6 + 4], dz = a.rays[r * 6 + 5];
  const float dnorm = comp_dnorm(dx, dy, dz);

  float w[kCompMaxPerLane];
  float carry = 1.0f;  // product of (1 - alpha + 1e-10) over all earlier groups of 32 samples
  float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_d = 0.f, acc_a = 0.f;
#pragma unroll
  for (int j = 0; j < kCompMaxPerLane; ++j) {
    w[j] = 0.f;
    const int i0 = j * 32;
    if (i0 >= N) continue;
    const int i = i0 + lane;
    float alpha = 0.f, zi = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
    if (i < N) {
      zi = z[i];
      const float dist = comp_dist(zi, (i + 1 < N) ? z[i + 1] : 0.f, i + 1 < N, dnorm);
      const float* q = raw + (int64_t)i * CH;
      const bool masked = a.mask_outside && a.sample_box != nullptr && a.sample_box[r * N + i] < 0;
      alpha = comp_alpha(q[3], dist, masked);
      cr = comp_sigmoid(q[0]);
      cg = comp_sigmoid(q[1]);
      cb = comp_sigmoid(q[2]);
    }
    // exclusive product scan of t = 1 - alpha + 1e-10 across the warp
    const float t = (i < N) ? (1.0f - alpha + 1e-10f) : 1.0f;
    float total;
    const float excl = comp_scan32(t, lane, &total);
    const float T = carry * excl;
    carry *= total;
    const float wi = alpha * T;
    w[j] = wi;
    if (i < N) {
      if (a.o.weights) a.o.weights[r * N + i] = wi;
      acc_r += wi * cr; acc_g += wi * cg; acc_b += wi * cb; acc_d += wi * zi; acc_a += wi;
    }
  }
  acc_r = warp_sum(acc_r); acc_g = warp_sum(acc_g); acc_b = warp_sum(acc_b);
  acc_d = warp_sum(acc_d); acc_a = warp_sum(acc_a);
  if (lane == 0) {
    if (a.o.rgb_map) {
      const float bg = a.white_bkgd ? (1.0f - acc_a) : 0.f;
      a.o.rgb_map[r * 3 + 0] = acc_r + bg;
      a.o.rgb_map[r * 3 + 1] = acc_g + bg;
      a.o.rgb_map[r * 3 + 2] = acc_b + bg;
    }
    if (a.o.depth_map) a.o.depth_map[r] = acc_d;
    if (a.o.acc_map) a.o.acc_map[r] = acc_a;
    if (a.o.disp_map) a.o.disp_map[r] = comp_disp(acc_d, acc_a);
  }

  const int C = a.C, K = a.K;
  const bool want_sem = C > 0 && a.o.semantic_map, want_inst = K > 0 && a.o.instance_map;
  const bool want_fsem = C > 0 && a.o.fixed_semantic_map && a.sample_box && a.box_sem;
  const bool want_finst = K > 0 && a.o.fixed_instance_map && a.sample_box && a.box_inst;
  if (!(want_sem || want_inst || want_fsem || want_finst)) return;

  float sem[kCompMaxChan], ins[kCompMaxChan], fsem[kCompMaxChan], fins[kCompMaxChan];
#pragma unroll
  for (int q = 0; q < kCompMaxChan; ++q) sem[q] = ins[q] = fsem[q] = fins[q] = 0.f;
  for (int i = 0; i < N; ++i) {
    float wi = 0.f;
#pragma unroll
    for (int j = 0; j < kCompMaxPerLane; ++j)
      if (j == (i >> 5)) wi = __shfl_sync(0xffffffffu, w[j], i & 31);
    const float* q = raw + (int64_t)i * CH + 4;
    if (want_sem) {
      float v[kCompMaxChan];
#pragma unroll
      for (int s = 0; s < kCompMaxChan; ++s) {
        const int c = lane + 32 * s;
        v[s] = (c < C) ? q[c] : -INFINITY;
      }
      if (a.sem_softmax) {
        float m = v[0];
#pragma unroll
        for (int s = 1; s < kCompMaxChan; ++s) m = fmaxf(m, v[s]);
        m = warp_max(m);
        float e = 0.f;
#pragma unroll
        for (int s = 0; s < kCompMaxChan; ++s) {
          v[s] = (lane + 32 * s < C) ? expf(v[s] - m) : 0.f;
          e += v[s];
        }
        e = warp_sum(e);
#pragma unroll
        for (int s = 0; s < kCompMaxChan; ++s) v[s] = v[s] / e;
      }
#pragma unroll
      for (int s = 0; s < kCompMaxChan; ++s)
        if (lane + 32 * s < C) sem[s] += wi * v[s];
    }
    if (want_inst) {
#pragma unroll
      for (int s = 0; s < kCompMaxChan; ++s) {
        const int c = lane + 32 * s;
        if (c < K) ins[s] += wi * q[C + c];
      }
    }
    if (want_fsem || want_finst) {
      const int32_t sb = a.sample_box[r * N + i];
      if (sb >= 0 && sb < a.B) {
        if (want_fsem) {
          const int32_t id = a.box_sem[sb];
#pragma unroll
          for (int s = 0; s < kCompMaxChan; ++s)
            if (lane + 32 * s == id) fsem[s] += wi;
        }
        if (want_finst) {
          const int32_t id = a.box_inst[sb];
#pragma unroll
          for (int s = 0; s < kCompMaxChan; ++s)
            if (lane + 32 * s == id) fins[s] += wi;
        }
      }
    }
  }
#pragma unroll
  for (int s = 0; s < kCompMaxChan; ++s) {
    const int c = lane + 32 * s;
    if (want_sem && c < C) a.o.semantic_map[r * C + c] = sem[s];
    if (want_inst && c < K) a.o.instance_map[r * K + c] = ins[s];
    if (want_fsem && c < C) a.o.fixed_semantic_map[r * C + c] = fsem[s];
    if (want_finst && c < K) a.o.fixed_instance_map[r * K + c] = fins[s];
  }
}

// ------------------------------------------------------------------------------------ a9 backward
// d(loss)/d(raw) given d(loss)/d(maps) (SURVEY 8(f) rank 2: the first stage of the backward chain).
// With t_i = 1 - alpha_i + 1e-10, T_i = prod_{j<i} t_j, w_i = alpha_i T_i and
//   G_i = dL/dw_i = g_rgb . c_i + g_depth z_i + g_acc + g_sem . s_i + g_inst . u_i + g_w[i] + fixed-map terms:
//   dL/dalpha_i = G_i T_i - (sum_{j>i} G_j w_j) / t_i,   dalpha/dsigma = delta_i exp(-sigma_i delta_i),
//   dL/dc_i = w_i g_rgb (through the sigmoid), dL/ds_i = w_i g_sem, dL/du_i = w_i g_inst.
// Same work distribution as the forward kernel: one warp per ray, lanes stride samples for the scans and
// channels for the logits; T is recomputed with the forward's arithmetic (composite_math.cuh) so that w matches it
// bit for bit.
struct CompositeBwdArgs {
  const float* raw; const float* z; const float* rays;
  int64_t R; int N, C, K, CH;
  int white_bkgd, mask_outside;
  const int32_t* sample_box; const int32_t* box_sem; const int32_t* box_inst; int B;
  pnr_composite_grads g;
  float* d_raw;
};

__global__ void __launch_bounds__(kCompWarps * 32) composite_backward_kernel(CompositeBwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kCompWarps + (threadIdx.x >> 5);
  if (r >= a.R) return;
  const int N = a.N, CH = a.CH, C = a.C, K = a.K;
  const float* raw = a.raw + r * N * CH;
  float* d_raw = a.d_raw + r * N * CH;
  const float* z = a.z + r * N;
  const float dx = a.rays[r * 6 + 3], dy = a.rays[r * 6 + 4], dz = a.rays[r * 6 + 5];
  const float dnorm = comp_dnorm(dx, dy, dz);
  float g_r = 0.f, g_g = 0.f, g_b = 0.f;
  if (a.g.rgb_map) { g_r = a.g.rgb_map[r * 3 + 0]; g_g = a.g.rgb_map[r * 3 + 1]; g_b = a.g.rgb_map[r * 3 + 2]; }
  const float g_depth = a.g.depth_map ? a.g.depth_map[r] : 0.f;
  float g_acc = a.g.acc_map ? a.g.acc_map[r] : 0.f;
  if (a.white_bkgd) g_acc -= g_r + g_g + g_b;   // rgb_map += 1 - acc_map
  const bool fsem = C > 0 && a.g.fixed_semantic_map && a.sample_box && a.box_sem;
  const bool finst = K > 0 && a.g.fixed_instance_map && a.sample_box && a.box_inst;

  float w[kCompMaxPerLane], T[kCompMaxPerLane], G[kCompMaxPerLane], dsig[kCompMaxPerLane], tv[kCompMaxPerLane];
  float carry = 1.0f;
#pragma unroll
  for (int j = 0; j < kCompMaxPerLane; ++j) {
    w[j] = T[j] = G[j] = dsig[j] = 0.f;
    tv[j] = 1.0f;
    const int i0 = j * 32;
    if (i0 >= N) continue;
    const int i = i0 + lane;
    float alpha = 0.f, Gi = 0.f, ds = 0.f;
    float cr = 0.f, cg = 0.f, cb = 0.f;
    if (i < N) {
      const float zi = z[i];
      const float dist = comp_dist(zi, (i + 1 < N) ? z[i + 1] : 0.f, i + 1 < N, dnorm);
      const float* q = raw + (int64_t)i * CH;
      float sig = fmaxf(q[3], 0.f);
      bool live = q[3] > 0.f;
      int32_t sb = -1;
      if (a.sample_box != nullptr) sb = a.sample_box[r * N + i];
      if (a.mask_outside && a.sample_box != nullptr && sb < 0) { sig = 0.f; live = false; }
      const float e = expf(-sig * dist);   // comp_alpha's exp, kept: 1 - alpha is not e in fp32
      alpha = 1.0f - e;
      ds = live ? dist * e : 0.f;                       // dalpha / draw_sigma
      cr = comp_sigmoid(q[0]);
      cg = comp_sigmoid(q[1]);
      cb = comp_sigmoid(q[2]);
      Gi = g_r * cr + g_g * cg + g_b * cb + g_depth * zi + g_acc;
      if (a.g.weights) Gi += a.g.weights[r * N + i];
      if (sb >= 0 && sb < a.B) {
        if (fsem) { const int32_t id = a.box_sem[sb]; if (id >= 0 && id < C) Gi += a.g.fixed_semantic_map[r * C + id]; }
        if (finst) { const int32_t id = a.box_inst[sb]; if (id >= 0 && id < K) Gi += a.g.fixed_instance_map[r * K + id]; }
      }
    }
    const float t = (i < N) ? (1.0f - alpha + 1e-10f) : 1.0f;
    tv[j] = t;
    float total;
    T[j] = carry * comp_scan32(t, lane, &total);
    carry *= total;
    w[j] = alpha * T[j];
    G[j] = Gi;
    dsig[j] = ds;
    if (i < N) {   // colour gradients need nothing else
      const float wi = w[j];
      float* dq = d_raw + (int64_t)i * CH;
      dq[0] = wi * g_r * cr * (1.0f - cr);
      dq[1] = wi * g_g * cg * (1.0f - cg);
      dq[2] = wi * g_b * cb * (1.0f - cb);
    }
  }

  // logits: G_i += g_sem . s_i + g_inst . u_i ; d_raw[i, 4 + c] = w_i g[c]   (lanes stride channels)
  const bool have_sem = C > 0 && a.g.semantic_map, have_inst = K > 0 && a.g.instance_map;
  if (C + K > 0) {
    float gs[kCompMaxChan], gi[kCompMaxChan];
#pragma unroll
    for (int s = 0; s < kCompMaxChan; ++s) {
      const int c = lane + 32 * s;
      gs[s] = (have_sem && c < C) ? a.g.semantic_map[r * C + c] : 0.f;
      gi[s] = (have_inst && c < K) ? a.g.instance_map[r * K + c] : 0.f;
    }
    for (int i = 0; i < N; ++i) {
      float wi = 0.f;
#pragma unroll
      for (int j = 0; j < kCompMaxPerLane; ++j)
        if (j == (i >> 5)) wi = __shfl_sync(0xffffffffu, w[j], i & 31);
      const float* q = raw + (int64_t)i * CH + 4;
      float* dq = d_raw + (int64_t)i * CH + 4;
      float dot = 0.f;
#pragma unroll
      for (int s = 0; s < kCompMaxChan; ++s) {
        const int c = lane + 32 * s;
        if (c < C) { dot += gs[s] * q[c]; dq[c] = wi * gs[s]; }
        if (c < K) { dot += gi[s] * q[C + c]; dq[C + c] = wi * gi[s]; }
      }
      dot = warp_sum(dot);
#pragma unroll
      for (int j = 0; j < kCompMaxPerLane; ++j)
        if (j == (i >> 5) && lane == (i & 31)) G[j] += dot;
    }
  }

  // suffix sums of G_j w_j, last group of 32 first
  float tail = 0.f;   // sum over all later groups
#pragma unroll
  for (int j = kCompMaxPerLane - 1; j >= 0; --j) {
    const int i0 = j * 32;
    if (i0 >= N) continue;
    const int i = i0 + lane;
    const float v = (i < N) ? G[j] * w[j] : 0.f;
    float incl = v;   // inclusive suffix sum within the group
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const float o = __shfl_down_sync(0xffffffffu, incl, d);
      if (lane + d < 32) incl += o;
    }
    // strictly later samples: the next lane's inclusive sum, not incl - v, which cancels when sample i holds most of
    // the weight (a surface) and would leave S, then S / t with t ~ 1e-10, wrong by ulps of G_i w_i
    float later = __shfl_down_sync(0xffffffffu, incl, 1);
    if (lane == 31) later = 0.f;
    const float S = tail + later;
    tail += __shfl_sync(0xffffffffu, incl, 0);
    if (i < N) {
      const float t = tv[j];
      d_raw[(int64_t)i * CH + 3] = (G[j] * T[j] - S / t) * dsig[j];
    }
  }
}

}  // namespace pnr

using namespace pnr;

// ------------------------------------------------------------------------------------ fixed (bounding-box) maps
// fixed_semantic_map[r,c] = sum_i w_i [box_sem[sample_box_i] == c] (likewise instances) from the per-sample weights
// alone - the companion of the MLP kernel's compositing epilogue, which never sees the id tables.  One warp per ray,
// samples in order (the sum order is the sample order), lanes own channels lane, lane+32, ...
__global__ void __launch_bounds__(kCompWarps * 32) fixed_maps_kernel(
    const float* __restrict__ weights, const int32_t* __restrict__ sample_box, const int32_t* __restrict__ box_sem,
    const int32_t* __restrict__ box_inst, int64_t R, int N, int C, int K, int B, float* __restrict__ fsem,
    float* __restrict__ finst) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kCompWarps + (threadIdx.x >> 5);
  if (r >= R) return;
  float a[kCompMaxChan], b[kCompMaxChan];
#pragma unroll
  for (int q = 0; q < kCompMaxChan; ++q) a[q] = b[q] = 0.f;
  for (int i0 = 0; i0 < N; i0 += 32) {
    const int i = i0 + lane;
    const float wl = i < N ? weights[r * N + i] : 0.f;
    const int32_t sl = i < N ? sample_box[r * N + i] : -1;
    const int32_t id_s = (fsem != nullptr && sl >= 0 && sl < B) ? box_sem[sl] : -1;
    const int32_t id_i = (finst != nullptr && sl >= 0 && sl < B) ? box_inst[sl] : -1;
    // only the samples that lie in a primitive contribute (in sample order, so the sums are unchanged)
    unsigned todo = __ballot_sync(0xffffffffu, id_s >= 0 || id_i >= 0);
    while (todo) {
      const int j = __ffs(todo) - 1;
      todo &= todo - 1;
      const float wj = __shfl_sync(0xffffffffu, wl, j);
      const int32_t cs = __shfl_sync(0xffffffffu, id_s, j), ci = __shfl_sync(0xffffffffu, id_i, j);
#pragma unroll
      for (int q = 0; q < kCompMaxChan; ++q) {
        if (lane + 32 * q == cs) a[q] += wj;
        if (lane + 32 * q == ci) b[q] += wj;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < kCompMaxChan; ++q) {
    const int c = lane + 32 * q;
    if (fsem != nullptr && c < C) fsem[r * C + c] = a[q];
    if (finst != nullptr && c < K) finst[r * K + c] = b[q];
  }
}

int pnr::launch_fixed_maps(const float* weights, const int32_t* sample_box, const int32_t* box_sem,
                           const int32_t* box_inst, int64_t R, int N, int C, int K, int B, float* fsem, float* finst,
                           cudaStream_t stream) {
  if (R == 0 || (!fsem && !finst)) return PNR_OK;
  PNR_CHECK_ARG(C <= 32 * kCompMaxChan && K <= 32 * kCompMaxChan, "fixed maps: C=%d or K=%d > %d", C, K, 32 * kCompMaxChan);
  fixed_maps_kernel<<<(unsigned)((R + kCompWarps - 1) / kCompWarps), kCompWarps * 32, 0, stream>>>(
      weights, sample_box, box_sem, box_inst, R, N, C, K, B, fsem, finst);
  PNR_LAUNCH_CHECK("fixed_maps_kernel");
  return PNR_OK;
}

// ------------------------------------------------------------------------------------ label tiles
// 8(e) / 8(f) rank 4: the per-ray tile a rank contributes to the all-gather when labels, not logits, are wanted:
// rgb as u8, depth as f32, semantic / instance label = argmax over the composited maps (ties -> lowest index)
// as i16.  13 bytes per ray instead of 4*(5+C+K) (cfg3: 456 -> 13).  One warp per ray; lanes stride channels.
struct LabelArgs {
  const float* rgb; const float* depth; const float* sem; const float* inst;
  int64_t R; int C, K;
  uint8_t* rgb8; float* depth_out; int16_t* sem_label; int16_t* inst_label;
};

// argmax over v[0..n) with lanes striding the channels; NaN counts as -inf; ties -> lowest index; -1 when n == 0
__device__ __forceinline__ int warp_argmax(const float* __restrict__ v, int n, int lane) {
  float best = -INFINITY;
  int arg = 0x7fffffff;
  for (int c = lane; c < n; c += 32) {
    float x = v[c];
    if (x != x) x = -INFINITY;
    if (x > best || arg == 0x7fffffff) { best = x; arg = c; }   // ascending c: the first maximum is kept
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, d);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, d);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  return arg == 0x7fffffff ? -1 : arg;
}

__global__ void __launch_bounds__(256) label_tiles_kernel(LabelArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= a.R) return;
  if (a.rgb8 != nullptr && lane < 3) {
    const float c = fminf(fmaxf(a.rgb[r * 3 + lane], 0.f), 1.f);
    a.rgb8[r * 3 + lane] = (uint8_t)__float2int_rn(c * 255.0f);
  }
  if (a.depth_out != nullptr && lane == 3) a.depth_out[r] = a.depth[r];
  if (a.sem_label != nullptr) {
    const int s = warp_argmax(a.sem + r * a.C, a.C, lane);
    if (lane == 0) a.sem_label[r] = (int16_t)s;
  }
  if (a.inst_label != nullptr) {
    const int s = warp_argmax(a.inst + r * a.K, a.K, lane);
    if (lane == 0) a.inst_label[r] = (int16_t)s;
  }
}

extern "C" int pnr_label_tiles(const float* rgb_map, const float* depth_map, const float* semantic_map,
                               const float* instance_map, int64_t R, int32_t C, int32_t K, uint8_t* rgb8,
                               float* depth_out, int16_t* sem_label, int16_t* inst_label, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(R > 0 && C >= 0 && K >= 0 && C < 32768 && K < 32768, "pnr_label_tiles: bad sizes");
  PNR_CHECK_ARG(!rgb8 || rgb_map, "pnr_label_tiles: rgb8 wanted without rgb_map");
  PNR_CHECK_ARG(!depth_out || depth_map, "pnr_label_tiles: depth wanted without depth_map");
  PNR_CHECK_ARG(!sem_label || (semantic_map && C > 0), "pnr_label_tiles: semantic labels wanted without semantic_map");
  PNR_CHECK_ARG(!inst_label || (instance_map && K > 0), "pnr_label_tiles: instance labels wanted without instance_map");
  LabelArgs a{rgb_map, depth_map, semantic_map, instance_map, R, C, K, rgb8, depth_out, sem_label, inst_label};
  label_tiles_kernel<<<(unsigned)((R + 7) / 8), 256, 0, (cudaStream_t)stream>>>(a);
  PNR_LAUNCH_CHECK("label_tiles_kernel");
  return PNR_OK;
}

extern "C" int pnr_composite_backward(const float* raw, const float* z, const float* rays, int64_t R, int32_t N,
                                      int32_t C, int32_t K, int32_t white_bkgd, int32_t sem_softmax,
                                      int32_t mask_outside, const int32_t* sample_box, const int32_t* box_sem,
                                      const int32_t* box_inst, int32_t B, const pnr_composite_grads* g,
                                      float* d_raw, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(R > 0, "pnr_composite_backward: R=%lld < 0", (long long)R);
  PNR_CHECK_ARG(raw && z && rays && g && d_raw, "pnr_composite_backward: null pointer");
  PNR_CHECK_ARG(N >= 1 && N <= 32 * kCompMaxPerLane, "pnr_composite_backward: N=%d outside [1,%d]", N,
                32 * kCompMaxPerLane);
  PNR_CHECK_ARG(C >= 0 && C <= 32 * kCompMaxChan && K >= 0 && K <= 32 * kCompMaxChan,
                "pnr_composite_backward: C=%d or K=%d outside [0,%d]", C, K, 32 * kCompMaxChan);
  if (sem_softmax)
    return set_error(PNR_ERR_UNSUPPORTED, "pnr_composite_backward: sem_activation=softmax is not implemented");
  CompositeBwdArgs a;
  a.raw = raw; a.z = z; a.rays = rays; a.R = R; a.N = N; a.C = C; a.K = K; a.CH = 4 + C + K;
  a.white_bkgd = white_bkgd; a.mask_outside = mask_outside;
  a.sample_box = sample_box; a.box_sem = box_sem; a.box_inst = box_inst; a.B = B; a.g = *g; a.d_raw = d_raw;
  composite_backward_kernel<<<(unsigned)((R + kCompWarps - 1) / kCompWarps), kCompWarps * 32, 0,
                              (cudaStream_t)stream>>>(a);
  PNR_LAUNCH_CHECK("composite_backward_kernel");
  return PNR_OK;
}

extern "C" int pnr_generate_rays(int32_t H, int32_t W, int32_t row0, int32_t rows, int32_t camera,
                                 const float* intr_host, const float* c2w_host, float* rays, void* stream) {
  if (rows == 0 || W == 0) return PNR_OK;
  PNR_CHECK_ARG(intr_host && c2w_host && rays, "pnr_generate_rays: null pointer");
  PNR_CHECK_ARG(H > 0 && W > 0 && rows > 0 && row0 >= 0 && row0 + rows <= H, "pnr_generate_rays: bad image window");
  PNR_CHECK_ARG(camera >= 0 && camera <= 2, "pnr_generate_rays: camera %d (0 pinhole, 1 equirect, 2 fisheye)", camera);
  CamArgs a;
  a.fx = intr_host[0]; a.fy = intr_host[1]; a.cx = intr_host[2]; a.cy = intr_host[3];
  a.xi = a.k1 = a.k2 = 0.f;
  if (camera == 2) { a.xi = intr_host[4]; a.k1 = intr_host[5]; a.k2 = intr_host[6]; }
  for (int i = 0; i < 12; ++i) a.c2w[i] = c2w_host[i];
  a.H = H; a.W = W; a.row0 = row0; a.rows = rows; a.camera = camera;
  const int64_t n = (int64_t)rows * W;
  rays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, rays);
  PNR_LAUNCH_CHECK("rays_kernel");
  return PNR_OK;
}

extern "C" int pnr_encode(const float* x, int64_t n, int32_t L, float* out, void* stream) {
  if (n == 0) return PNR_OK;
  PNR_CHECK_ARG(x && out, "pnr_encode: null pointer");
  PNR_CHECK_ARG(L >= 0 && L <= 16, "pnr_encode: L=%d outside [0,16]", L);
  const size_t smem = (size_t)kEncTile * (3 + 6 * L) * sizeof(float);
  int dev = 0;
  int rc = current_device("pnr_encode", &dev);
  if (rc != PNR_OK) return rc;
  rc = opt_in_smem((const void*)encode_kernel, 64 * 1024, dev);
  if (rc != PNR_OK) return rc;
  encode_kernel<<<(unsigned)((n + kEncTile - 1) / kEncTile), kEncTile, smem, (cudaStream_t)stream>>>(
      x, n, L, out);
  PNR_LAUNCH_CHECK("encode_kernel");
  return PNR_OK;
}

extern "C" int pnr_composite(const float* raw, const float* z, const float* rays, int64_t R, int32_t N,
                             int32_t C, int32_t K, int32_t white_bkgd, int32_t sem_softmax,
                             int32_t mask_outside, const int32_t* sample_box, const int32_t* box_sem,
                             const int32_t* box_inst, int32_t B, const pnr_composite_out* out,
                             void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(R > 0, "pnr_composite: R=%lld < 0", (long long)R);
  PNR_CHECK_ARG(raw && z && rays && out, "pnr_composite: null pointer");
  PNR_CHECK_ARG(N >= 1 && N <= 32 * kCompMaxPerLane, "pnr_composite: N=%d outside [1,%d]", N,
                32 * kCompMaxPerLane);
  PNR_CHECK_ARG(C >= 0 && C <= 32 * kCompMaxChan && K >= 0 && K <= 32 * kCompMaxChan,
                "pnr_composite: C=%d or K=%d outside [0,%d]", C, K, 32 * kCompMaxChan);
  CompositeArgs a;
  a.raw = raw; a.z = z; a.rays = rays; a.R = R; a.N = N; a.C = C; a.K = K; a.CH = 4 + C + K;
  a.white_bkgd = white_bkgd; a.sem_softmax = sem_softmax; a.mask_outside = mask_outside;
  a.sample_box = sample_box; a.box_sem = box_sem; a.box_inst = box_inst; a.B = B; a.o = *out;
  composite_kernel<<<(unsigned)((R + kCompWarps - 1) / kCompWarps), kCompWarps * 32, 0,
                     (cudaStream_t)stream>>>(a);
  PNR_LAUNCH_CHECK("composite_kernel");
  return PNR_OK;
}
