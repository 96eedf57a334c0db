// ray_kernels.cu — the bit-exact integer/compare stages of the render path (SURVEY.md 8(a) a5, a6, a10):
// ray / oriented-box slab intersection with M-nearest selection, scene near/far, stratified depths
// with per-sample primitive ids, and the inverse-CDF fine sampler with merge-sort.
// All are HBM-bound streaming kernels: one thread (or one warp) per ray, box table staged in shared
// memory, coalesced row-major outputs.  Arithmetic order lives in ray_math.h.
#include "common.cuh"
#include "ray_math.h"

namespace pnr {

// ------------------------------------------------------------------------------------ a5 intersect
constexpr int kBoxChunk = 512;  // boxes staged per shared-memory fill (15 floats each = 30 KB; 17 with meshes)

// kMeshes = false: the slab test of every box (pnr_intersect).  kMeshes = true: a box whose triangle range
// [tri_start[b], tri_start[b+1]) is not empty is the cull volume of a closed mesh (ray_math.h: pnr_tri_cross,
// PnrMeshCross); on a cull hit its triangles are read from global memory (the same rows for the whole warp, so
// L1/L2-resident broadcasts).  Every range is clamped into [0, T], so a malformed start table cannot read outside tris.
template <bool kMeshes>
__global__ void __launch_bounds__(256) intersect_kernel(const float* __restrict__ rays, int64_t R,
                                                        const float* __restrict__ bc,
                                                        const float* __restrict__ bh,
                                                        const float* __restrict__ br, int B, int M,
                                                        uint8_t* __restrict__ hit_mask,
                                                        int32_t* __restrict__ box_id,
                                                        float* __restrict__ t_in,
                                                        float* __restrict__ t_out,
                                                        const int32_t* __restrict__ tri_start,
                                                        const float* __restrict__ tris, int64_t T) {
  constexpr int kS = kMeshes ? 17 : 15;   // floats per staged box: center, half, rot (+ the triangle range)
  __shared__ float sb[kBoxChunk * kS];
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 1;
  if (r < R) {
    const float2* p = reinterpret_cast<const float2*>(rays + r * 6);
    const float2 a = p[0], b = p[1], c = p[2];
    ox = a.x; oy = a.y; oz = b.x; dx = b.y; dy = c.x; dz = c.y;
  }
  PnrHitList L;
  pnr_hits_init(&L);
  for (int b0 = 0; b0 < B; b0 += kBoxChunk) {
    const int nb = min(kBoxChunk, B - b0);
    __syncthreads();
    for (int i = threadIdx.x; i < nb * kS; i += blockDim.x) {
      const int b = i / kS, e = i % kS;
      if (kMeshes && e >= 15) {
        const int64_t lo = min(max((int64_t)tri_start[b0 + b], (int64_t)0), T);
        const int64_t hi = min(max((int64_t)tri_start[b0 + b + 1], lo), T);
        sb[i] = __int_as_float((int)(e == 15 ? lo : hi));
      } else {
        sb[i] = e < 3 ? bc[(b0 + b) * 3 + e] : (e < 6 ? bh[(b0 + b) * 3 + e - 3] : br[(b0 + b) * 9 + e - 6]);
      }
    }
    __syncthreads();
    if (r < R) {
      for (int b = 0; b < nb; ++b) {
        const float* q = sb + b * kS;
        float tmin, tmax;
        const bool hit = pnr_slab(ox, oy, oz, dx, dy, dz, q, q + 3, q + 6, &tmin, &tmax);
        if (kMeshes) {
          const int k0 = __float_as_int(q[15]), k1 = __float_as_int(q[16]);
          if (k0 == k1) {
            if (hit) pnr_hits_insert(&L, M, tmin, tmax, b0 + b);
          } else if (hit) {
            const PnrShear S = pnr_shear(dx, dy, dz);
            PnrMeshCross X;
            pnr_cross_init(&X);
            for (int k = k0; k < k1; ++k) {
              float v[9];
#pragma unroll
              for (int e = 0; e < 9; ++e) v[e] = __ldg(tris + (int64_t)k * 9 + e);
              float t;
              if (pnr_tri_cross(ox, oy, oz, S, v, &t)) pnr_cross_add(&X, M, t);
            }
            pnr_cross_emit(&X, &L, M, b0 + b);
          }
        } else if (hit) {
          pnr_hits_insert(&L, M, tmin, tmax, b0 + b);
        }
      }
    }
  }
  if (r < R) {
    hit_mask[r] = L.n > 0 ? 1 : 0;
#pragma unroll
    for (int m = 0; m < PNR_MAX_HITS; ++m)
      if (m < M) {
        const bool v = m < L.n;
        box_id[r * M + m] = v ? L.id[m] : -1;
        t_in[r * M + m] = v ? pnr_max_nan(L.key[m], 0.f) : 0.f;
        t_out[r * M + m] = v ? L.tout[m] : 0.f;
      }
  }
}

struct Aabb { float c[3], h[3]; };

__global__ void __launch_bounds__(256) near_far_kernel(const float* __restrict__ rays, int64_t R,
                                                       Aabb box, float near_min, float far_default,
                                                       float* __restrict__ near,
                                                       float* __restrict__ far) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float2* p = reinterpret_cast<const float2*>(rays + r * 6);
  const float2 a = p[0], b = p[1], c = p[2];
  const float rot[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  float tmin, tmax;
  const bool hit = pnr_slab(a.x, a.y, b.x, b.y, c.x, c.y, box.c, box.h, rot, &tmin, &tmax);
  near[r] = hit ? pnr_max_nan(tmin, near_min) : near_min;
  far[r] = hit ? tmax : far_default;
}

__global__ void __launch_bounds__(256) bound_kernel(const uint8_t* __restrict__ hit,
                                                    const int32_t* __restrict__ box_id,
                                                    const float* __restrict__ t_in,
                                                    const float* __restrict__ t_out, int64_t R, int M,
                                                    float* __restrict__ near, float* __restrict__ far) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R || !hit[r]) return;
  float last = 0.f;  // max over t_out of valid slots (padding slots contribute 0, as in the oracle)
  for (int m = 0; m < M; ++m) last = pnr_max_nan(last, box_id[r * M + m] >= 0 ? t_out[r * M + m] : 0.f);
  near[r] = pnr_max_nan(near[r], t_in[r * M]);
  far[r] = pnr_min_nan(far[r], last);
}

// ------------------------------------------------------------------------------------ a6 sampling
// One warp per ray: the ray's near/far and its <= 8 hit intervals are loaded once (lane m holds interval m,
// broadcast by shuffle), lanes stride the sample axis so z / sample_box stores are fully coalesced.
__global__ void __launch_bounds__(256) stratified_kernel(
    const float* __restrict__ near, const float* __restrict__ far, const float* __restrict__ t_vals,
    const float* __restrict__ u, int64_t R, int N, float perturb, const int32_t* __restrict__ box_id,
    const float* __restrict__ t_in, const float* __restrict__ t_out, int M, float* __restrict__ z,
    int32_t* __restrict__ sample_box) {
  const int lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  const float nr = near[r], fr = far[r];
  int32_t my_id = -1;
  float my_in = 0.f, my_out = 0.f;
  if (box_id != nullptr && lane < M) {
    my_id = box_id[r * M + lane];
    my_in = t_in[r * M + lane];
    my_out = t_out[r * M + lane];
  }
  for (int i0 = 0; i0 < N; i0 += 32) {   // warp-uniform trip count: the shuffles below need all lanes
    const int i = i0 + lane;
    const bool live = i < N;
    float zi = 0.f;
    if (live) {
      const int64_t idx = r * N + i;
      zi = (perturb > 0.f) ? pnr_strat_z_jitter(nr, fr, t_vals, i, N, u[idx]) : pnr_strat_z(nr, fr, t_vals[i]);
      z[idx] = zi;
    }
    if (sample_box != nullptr) {
      int32_t tag = -1;
      for (int m = M - 1; m >= 0; --m) {   // first (nearest) containing interval wins
        const int32_t id = __shfl_sync(0xffffffffu, my_id, m);
        const float a = __shfl_sync(0xffffffffu, my_in, m), b = __shfl_sync(0xffffffffu, my_out, m);
        if (id >= 0 && zi >= a && zi <= b) tag = id;
      }
      if (live) sample_box[r * N + i] = (box_id != nullptr) ? tag : -1;
    }
  }
}

// a6, interval mode (ray_math.h: pnr_interval_plan): one warp per ray; every lane builds the ray's (tiny) plan
// from the same <= 8 intervals, lanes stride the allocation slots, the warp bitonic-sorts the depths in shared
// memory and tags them.
constexpr int kIvWarps = 8;
constexpr int kIvMaxN = 256;

__global__ void __launch_bounds__(kIvWarps * 32) interval_kernel(
    const float* __restrict__ near, const float* __restrict__ far, const float* __restrict__ t_vals,
    const float* __restrict__ u, int64_t R, int N, float perturb, const int32_t* __restrict__ box_id,
    const float* __restrict__ t_in, const float* __restrict__ t_out, int M, float* __restrict__ z,
    int32_t* __restrict__ sample_box) {
  __shared__ float s_all[kIvWarps][kIvMaxN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kIvWarps + warp;
  if (r >= R) return;
  const float nr = near[r], fr = far[r];
  PnrIntervalPlan P;
  pnr_interval_plan(nr, fr, box_id + r * M, t_in + r * M, t_out + r * M, M, N, &P);
  float* all = s_all[warp];
  if (P.kept == 0) {   // no primitive on this ray: the uniform rule (already ascending)
    for (int i = lane; i < N; i += 32) {
      const int64_t idx = r * N + i;
      z[idx] = (perturb > 0.f) ? pnr_strat_z_jitter(nr, fr, t_vals, i, N, u[idx]) : pnr_strat_z(nr, fr, t_vals[i]);
      if (sample_box != nullptr) sample_box[idx] = -1;
    }
    return;
  }
  int Pw = 1;
  while (Pw < N) Pw <<= 1;
  for (int k = lane; k < Pw; k += 32)
    all[k] = k < N ? pnr_interval_z(&P, k, (perturb > 0.f) ? u[r * N + k] : 0.5f) : __int_as_float(0x7f800000);
  __syncwarp();
  for (int k = 2; k <= Pw; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < Pw; i += 32) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool asc = (i & k) == 0;
          const float a = all[i], b = all[ixj];
          if ((a > b) == asc) { all[i] = b; all[ixj] = a; }
        }
      }
      __syncwarp();
    }
  for (int i = lane; i < N; i += 32) {
    const float zi = all[i];
    z[r * N + i] = zi;
    if (sample_box != nullptr) sample_box[r * N + i] = pnr_tag(zi, box_id + r * M, t_in + r * M, t_out + r * M, M);
  }
}

// Re-tag an existing depth array (used after the fine-sample merge).
__global__ void __launch_bounds__(256) tag_kernel(const float* __restrict__ z, int64_t R, int N,
                                                  const int32_t* __restrict__ box_id,
                                                  const float* __restrict__ t_in,
                                                  const float* __restrict__ t_out, int M,
                                                  int32_t* __restrict__ sample_box) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * N) return;
  const int64_t r = idx / N;
  sample_box[idx] = pnr_tag(z[idx], box_id + r * M, t_in + r * M, t_out + r * M, M);
}

// ------------------------------------------------------------------------------------ a10 sample_pdf
// One warp per ray.  Lane 0 runs the two sequential double-accumulated running sums (their order is
// part of the bit-exact contract); all lanes then search / interpolate, and the warp bitonic-sorts
// the merged depths in shared memory.
constexpr int kPdfWarps = 4;
constexpr int kPdfMaxN = 256;     // coarse samples
constexpr int kPdfMaxAll = 512;   // coarse + fine, padded to a power of two

__global__ void __launch_bounds__(kPdfWarps * 32) sample_pdf_kernel(
    const float* __restrict__ z, const float* __restrict__ weights, int64_t R, int N, int Ni,
    const float* __restrict__ u, int64_t u_stride, float* __restrict__ z_fine, int64_t* __restrict__ idx_out,
    float* __restrict__ z_all) {
  __shared__ float s_w[kPdfWarps][kPdfMaxN];
  __shared__ float s_z[kPdfWarps][kPdfMaxN];
  __shared__ float s_cdf[kPdfWarps][kPdfMaxN];
  __shared__ float s_all[kPdfWarps][kPdfMaxAll];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * kPdfWarps + warp;
  if (r >= R) return;
  float* w = s_w[warp];
  float* zz = s_z[warp];
  float* cdf = s_cdf[warp];
  float* all = s_all[warp];
  for (int i = lane; i < N; i += 32) {
    w[i] = weights[r * N + i];
    zz[i] = z[r * N + i];
  }
  __syncwarp();
  {
    // pnr_pdf_cdf (ray_math.h: two sequential running sums in double, rounded to fp32 per element) as a warp scan.
    // Bit-identical to the sequential order because every partial sum is EXACT in double: the addends w + 1e-5 are fp32
    // values in [2^-17, 2^1) (lowest set bit >= 2^-40) and at most 254 of them stay below 2^8 - 49 bits; the pdf values
    // are fp32 in [2^-25, 2) and their sums stay below 2 - 50 bits.  (Weights outside [0, 1] - not produced by the
    // compositing - could round differently in the two orders.)
    const int nw = N - 2, per = (nw + 31) >> 5;
    const int k0 = min(lane * per, nw), k1 = min(k0 + per, nw);
    double part = 0.0;
    for (int k = k0; k < k1; ++k) part = __dadd_rn(part, (double)__fadd_rn(w[k + 1], 1e-5f));
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) part = __dadd_rn(part, __shfl_xor_sync(0xffffffffu, part, d));
    const float total = (float)part;
    double mine = 0.0;
    for (int k = k0; k < k1; ++k) mine = __dadd_rn(mine, (double)__fdiv_rn(__fadd_rn(w[k + 1], 1e-5f), total));
    double incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const double t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl = __dadd_rn(incl, t);
    }
    double acc = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) { acc = 0.0; cdf[0] = 0.f; }
    for (int k = k0; k < k1; ++k) {
      acc = __dadd_rn(acc, (double)__fdiv_rn(__fadd_rn(w[k + 1], 1e-5f), total));
      cdf[k + 1] = (float)acc;
    }
  }
  __syncwarp();
  const int Nb = N - 1;
  int P = 1;
  while (P < N + Ni) P <<= 1;
  for (int j = lane; j < Ni; j += 32) {
    const float uj = u[r * u_stride + j];
    int idx;
    const float zf = pnr_pdf_sample(zz, cdf, Nb, uj, &idx);
    if (z_fine != nullptr) z_fine[r * Ni + j] = zf;
    if (idx_out != nullptr) idx_out[r * Ni + j] = idx;
    all[N + j] = zf;
  }
  if (z_all == nullptr) return;
  __syncwarp();
  // Merge of the coarse depths (ascending by construction) with the fine ones.  When the fine depths are ascending too
  // - they are whenever u is (the deterministic sampler's linspace; the inverse CDF is monotone) - every element's
  // place in the merged row is its own index plus its rank in the other list (strict on one side, non-strict on the
  // other, so ties get distinct places): two binary searches per element instead of a 36-pass bitonic sort of the
  // padded row.  Same values in the same order either way; jittered (unsorted) u takes the sort.
  bool sorted = true;
  for (int j = lane; j + 1 < Ni; j += 32) sorted = sorted && (all[N + j] <= all[N + j + 1]);
  for (int i = lane; i + 1 < N; i += 32) sorted = sorted && (zz[i] <= zz[i + 1]);
  sorted = __all_sync(0xffffffffu, sorted);
  if (sorted) {
    // the merged row goes straight to global memory (each place is written exactly once)
    float* out = z_all + r * (int64_t)(N + Ni);
    const float* fine = all + N;
    for (int i = lane; i < N; i += 32) {      // coarse element i: + number of fine depths strictly below it
      const float v = zz[i];
      int lo = 0, hi = Ni;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (fine[mid] < v) lo = mid + 1; else hi = mid; }
      out[i + lo] = v;
    }
    for (int j = lane; j < Ni; j += 32) {     // fine element j: + number of coarse depths <= it
      const float v = fine[j];
      int lo = 0, hi = N;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (zz[mid] <= v) lo = mid + 1; else hi = mid; }
      out[j + lo] = v;
    }
    return;
  }
  for (int i = lane; i < N; i += 32) all[i] = zz[i];
  for (int i = N + Ni + lane; i < P; i += 32) all[i] = __int_as_float(0x7f800000);
  __syncwarp();
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < P; i += 32) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const bool asc = (i & k) == 0;
          const float a = all[i], b = all[ixj];
          if ((a > b) == asc) { all[i] = b; all[ixj] = a; }
        }
      }
      __syncwarp();
    }
  for (int i = lane; i < N + Ni; i += 32) z_all[r * (N + Ni) + i] = all[i];
}

}  // namespace pnr

using namespace pnr;

static inline unsigned blocks_for(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

// fn: the entry point's name in the error messages
static int intersect_rays(const char* fn, const float* rays, int64_t R, const float* box_center, const float* box_half,
                     const float* box_rot, const int32_t* mesh_tri_start, const float* mesh_tris, int64_t T, int32_t B,
                     int32_t M, uint8_t* hit_mask, int32_t* box_id, float* t_in, float* t_out, void* stream) {
  if (R == 0) return PNR_OK;  // empty input: nothing to do (pointers of empty tensors may be null)
  PNR_CHECK_ARG(R >= 0 && B >= 0, "%s: R=%lld or B=%d < 0", fn, (long long)R, B);
  PNR_CHECK_ARG(M >= 1 && M <= PNR_MAX_HITS, "%s: M=%d outside [1,%d]", fn, M, PNR_MAX_HITS);
  PNR_CHECK_ARG(rays && hit_mask && box_id && t_in && t_out, "%s: null pointer", fn);
  PNR_CHECK_ARG(B == 0 || (box_center && box_half && box_rot), "%s: null box table", fn);
  const bool meshes = mesh_tri_start || mesh_tris || T != 0;
  PNR_CHECK_ARG(!meshes || (mesh_tri_start && mesh_tris && T >= 1 && T < (int64_t(1) << 31)),
                "%s: mesh_tri_start (%s), mesh_tris (%s) and T=%lld: both pointers null with T == 0, or both set "
                "with 1 <= T < 2^31", fn, mesh_tri_start ? "set" : "null", mesh_tris ? "set" : "null", (long long)T);
  if (meshes && B > 0)
    intersect_kernel<true><<<blocks_for(R, 256), 256, 0, (cudaStream_t)stream>>>(
        rays, R, box_center, box_half, box_rot, B, M, hit_mask, box_id, t_in, t_out, mesh_tri_start, mesh_tris, T);
  else
    intersect_kernel<false><<<blocks_for(R, 256), 256, 0, (cudaStream_t)stream>>>(
        rays, R, box_center, box_half, box_rot, B, M, hit_mask, box_id, t_in, t_out, nullptr, nullptr, 0);
  PNR_LAUNCH_CHECK("intersect_kernel");
  return PNR_OK;
}

extern "C" int pnr_intersect_meshes(const float* rays, int64_t R, const float* box_center, const float* box_half,
                                    const float* box_rot, const int32_t* mesh_tri_start, const float* mesh_tris,
                                    int64_t T, int32_t B, int32_t M, uint8_t* hit_mask, int32_t* box_id, float* t_in,
                                    float* t_out, void* stream) {
  return intersect_rays("pnr_intersect_meshes", rays, R, box_center, box_half, box_rot, mesh_tri_start, mesh_tris, T, B, M,
                        hit_mask, box_id, t_in, t_out, stream);
}

extern "C" int pnr_intersect(const float* rays, int64_t R, const float* box_center,
                             const float* box_half, const float* box_rot, int32_t B, int32_t M,
                             uint8_t* hit_mask, int32_t* box_id, float* t_in, float* t_out,
                             void* stream) {
  return intersect_rays("pnr_intersect", rays, R, box_center, box_half, box_rot, nullptr, nullptr, 0, B, M, hit_mask, box_id,
                        t_in, t_out, stream);
}

extern "C" int pnr_scene_near_far(const float* rays, int64_t R, const float* aabb_host, float near_min,
                                  float far_default, float* near, float* far, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(rays && aabb_host && near && far, "pnr_scene_near_far: null pointer");
  if (R == 0) return PNR_OK;
  Aabb box;
  for (int j = 0; j < 3; ++j) {
    // same fp32 expressions as the oracle: (lo+hi)*0.5, (hi-lo)*0.5
    box.c[j] = (aabb_host[j] + aabb_host[3 + j]) * 0.5f;
    box.h[j] = (aabb_host[3 + j] - aabb_host[j]) * 0.5f;
  }
  near_far_kernel<<<blocks_for(R, 256), 256, 0, (cudaStream_t)stream>>>(rays, R, box, near_min,
                                                                         far_default, near, far);
  PNR_LAUNCH_CHECK("near_far_kernel");
  return PNR_OK;
}

extern "C" int pnr_bound_by_primitives(const uint8_t* hit_mask, const int32_t* box_id,
                                       const float* t_in, const float* t_out, int64_t R, int32_t M,
                                       float* near, float* far, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(hit_mask && box_id && t_in && t_out && near && far, "pnr_bound_by_primitives: null");
  PNR_CHECK_ARG(M >= 1 && M <= PNR_MAX_HITS, "pnr_bound_by_primitives: M=%d outside [1,%d]", M, PNR_MAX_HITS);
  if (R == 0) return PNR_OK;
  bound_kernel<<<blocks_for(R, 256), 256, 0, (cudaStream_t)stream>>>(hit_mask, box_id, t_in, t_out, R,
                                                                      M, near, far);
  PNR_LAUNCH_CHECK("bound_kernel");
  return PNR_OK;
}

extern "C" int pnr_sample_stratified(const float* near, const float* far, const float* t_vals,
                                     const float* u, int64_t R, int32_t N, float perturb,
                                     const int32_t* box_id, const float* t_in, const float* t_out,
                                     int32_t M, float* z, int32_t* sample_box, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(near && far && t_vals && z, "pnr_sample_stratified: null pointer");
  PNR_CHECK_ARG(N >= 1, "pnr_sample_stratified: N < 1");
  PNR_CHECK_ARG(!(perturb > 0.f) || u, "pnr_sample_stratified: perturb > 0 needs u");
  PNR_CHECK_ARG(box_id == nullptr || (t_in && t_out), "pnr_sample_stratified: box_id without t_in / t_out");
  PNR_CHECK_ARG(box_id == nullptr || (M >= 1 && M <= PNR_MAX_HITS), "pnr_sample_stratified: M=%d outside [1,%d]", M,
                PNR_MAX_HITS);
  if (R == 0) return PNR_OK;
  if (z == near) return set_error(PNR_ERR_ARG, "pnr_sample_stratified: in-place not allowed");
  stratified_kernel<<<blocks_for(R, 8), 256, 0, (cudaStream_t)stream>>>(
      near, far, t_vals, u, R, N, perturb, box_id, t_in, t_out, M, z, sample_box);
  PNR_LAUNCH_CHECK("stratified_kernel");
  return PNR_OK;
}

extern "C" int pnr_sample_intervals(const float* near, const float* far, const float* t_vals, const float* u,
                                    int64_t R, int32_t N, float perturb, const int32_t* box_id, const float* t_in,
                                    const float* t_out, int32_t M, float* z, int32_t* sample_box, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(near && far && t_vals && z, "pnr_sample_intervals: null pointer");
  PNR_CHECK_ARG(N >= 1 && N <= kIvMaxN, "pnr_sample_intervals: N=%d outside [1,%d]", N, kIvMaxN);
  PNR_CHECK_ARG(!(perturb > 0.f) || u, "pnr_sample_intervals: perturb > 0 needs u");
  PNR_CHECK_ARG(box_id && t_in && t_out, "pnr_sample_intervals: null interval table");
  PNR_CHECK_ARG(M >= 1 && M <= PNR_MAX_HITS, "pnr_sample_intervals: M=%d outside [1,%d]", M, PNR_MAX_HITS);
  interval_kernel<<<blocks_for(R, kIvWarps), kIvWarps * 32, 0, (cudaStream_t)stream>>>(
      near, far, t_vals, u, R, N, perturb, box_id, t_in, t_out, M, z, sample_box);
  PNR_LAUNCH_CHECK("interval_kernel");
  return PNR_OK;
}

extern "C" int pnr_tag_samples(const float* z, int64_t R, int32_t N, const int32_t* box_id,
                               const float* t_in, const float* t_out, int32_t M, int32_t* sample_box,
                               void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(z && box_id && t_in && t_out && sample_box, "pnr_tag_samples: null pointer");
  PNR_CHECK_ARG(R > 0 && N >= 1, "pnr_tag_samples: R=%lld or N=%d < 1", (long long)R, N);
  PNR_CHECK_ARG(M >= 1 && M <= PNR_MAX_HITS, "pnr_tag_samples: M=%d outside [1,%d]", M, PNR_MAX_HITS);
  if (R == 0) return PNR_OK;
  tag_kernel<<<blocks_for(R * N, 256), 256, 0, (cudaStream_t)stream>>>(z, R, N, box_id, t_in, t_out, M,
                                                                        sample_box);
  PNR_LAUNCH_CHECK("tag_kernel");
  return PNR_OK;
}

extern "C" int pnr_sample_pdf(const float* z, const float* weights, int64_t R, int32_t N, int32_t Ni,
                              const float* u, float* z_fine, int64_t* idx, float* z_all, void* stream) {
  return pnr::sample_pdf_strided(z, weights, R, N, Ni, u, Ni, z_fine, idx, z_all, stream);
}

// u row stride in floats (0: every ray reads the same row - the deterministic sampler without an [R,Ni] tensor)
int pnr::sample_pdf_strided(const float* z, const float* weights, int64_t R, int32_t N, int32_t Ni, const float* u,
                            int64_t u_stride, float* z_fine, int64_t* idx, float* z_all, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(z && weights && u, "pnr_sample_pdf: null pointer (u is required; for the deterministic\n"
                "                 sampler pass torch.linspace(0,1,Ni) broadcast over rays)");
  PNR_CHECK_ARG(N >= 3 && N <= kPdfMaxN, "pnr_sample_pdf: N=%d outside [3,%d]", N, kPdfMaxN);
  PNR_CHECK_ARG(Ni >= 1, "pnr_sample_pdf: Ni=%d < 1", Ni);
  PNR_CHECK_ARG(N + Ni <= kPdfMaxAll, "pnr_sample_pdf: N+Ni=%d > %d", N + Ni, kPdfMaxAll);
  if (R == 0) return PNR_OK;
  sample_pdf_kernel<<<blocks_for(R, kPdfWarps), kPdfWarps * 32, 0, (cudaStream_t)stream>>>(
      z, weights, R, N, Ni, u, u_stride, z_fine, idx, z_all);
  PNR_LAUNCH_CHECK("sample_pdf_kernel");
  return PNR_OK;
}
