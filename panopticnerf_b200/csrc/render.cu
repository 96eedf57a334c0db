// render.cu — pnr_render_fused: Renderer.render / batchify_rays / render_rays (SURVEY.md 8(a) a3, a4) as one
// C-ABI call.  The host side only sequences the stage kernels of this library over ray chunks; the chunk size
// follows from the caller's workspace, so the one large intermediate - raw [chunk, N+Ni, 4+C+K] - is bounded
// (~1.5 GB at the default workspace) instead of being materialised for the whole frame (46 GB at config 3).
#include <cstring>
#include "common.cuh"
#include "mlp_program.h"   // kRows
#include "ray_math.h"   // PNR_MAX_HITS

struct pnr_ctx;

namespace pnr {

int ctx_channels(const pnr_ctx* ctx);    // pnr_api.cu: 4 + C + K of the context's network
int ctx_classes(const pnr_ctx* ctx, int* C, int* K);

namespace {

constexpr size_t kAlign = 256;
inline size_t align_up(size_t x) { return (x + kAlign - 1) / kAlign * kAlign; }

// Per-ray scratch layout of one chunk.  `have_*`: the caller supplies the full-frame array, no scratch needed.
struct Layout {
  int N, Ni, Nt, CH, M;
  bool boxes, have_z, have_z0, have_w0, have_w1, have_sb, have_hits, have_nf;
  bool comp0, comp1;   // the pass runs as ONE kernel (MLP with compositing epilogue): no raw
  size_t raw, z0, zall, w0, w1, sb, near, far, hit, bid, tin, tout;   // bytes per ray
  size_t per_ray() const { return raw + z0 + zall + w0 + w1 + sb + near + far + hit + bid + tin + tout; }
};

// The compositing epilogue needs aligned groups of 32 samples per ray and composites logits, not softmax(logits).
// It is used when the network has heads: raw then is 456 B per sample (cfg3 frame: 470 -> 407 ms).  Without heads raw
// is 16 B per sample and the epilogue's extra barriers at the tile boundary cost more than the second kernel saves
// (cfg2 frame: 79.8 ms two kernels, 82.7 ms one), so the rgb + sigma configuration keeps the two-kernel path.
inline bool comp_ok(int n_samples, int CH, const pnr_render_args* a) {
  return CH > 4 && n_samples % 32 == 0 && (!a || !a->sem_softmax);
}

Layout make_layout(int N, int Ni, int CH, int M, bool boxes, const pnr_render_args* a) {
  Layout L{};
  L.N = N; L.Ni = Ni; L.Nt = N + Ni; L.CH = CH; L.M = M; L.boxes = boxes;
  const bool fine = Ni > 0;
  L.comp0 = comp_ok(N, CH, a);
  L.comp1 = fine ? comp_ok(N + Ni, CH, a) : L.comp0;
  L.have_w1 = a && a->out.weights;
  L.have_z = a && a->z_vals;
  L.have_z0 = a && a->z_vals0;
  L.have_w0 = a && a->out0.weights;
  L.have_sb = a && a->sample_box;
  L.have_hits = a && a->hit_mask && a->box_id && a->t_in && a->t_out;
  L.have_nf = a && a->near_out && a->far_out;
  L.raw = (L.comp0 && L.comp1) ? 0 : (size_t)((fine && L.comp1) ? N : L.Nt) * CH * 4;   // only for two-kernel passes
  L.zall = L.have_z ? 0 : (size_t)L.Nt * 4;
  L.z0 = (fine && !L.have_z0) ? (size_t)N * 4 : 0;
  L.w0 = (fine && !L.have_w0) ? (size_t)N * 4 : 0;
  L.w1 = L.have_w1 ? 0 : (size_t)L.Nt * 4;          // the last pass's weights (required by the one-kernel path)
  if (!fine) { L.w0 = L.w1; L.w1 = 0; }             // single pass: its weights are "w0"
  L.sb = (boxes && !L.have_sb) ? (size_t)L.Nt * 4 : 0;
  L.near = L.have_nf ? 0 : 4;
  L.far = L.have_nf ? 0 : 4;
  if (boxes && !L.have_hits) { L.hit = 1; L.bid = (size_t)M * 4; L.tin = (size_t)M * 4; L.tout = (size_t)M * 4; }
  return L;
}

// bytes of a chunk of Rc rays (each sub-buffer aligned)
size_t chunk_bytes(const Layout& L, int64_t Rc) {
  size_t b = 0;
  for (size_t per : {L.raw, L.z0, L.zall, L.w0, L.w1, L.sb, L.near, L.far, L.hit, L.bid, L.tin, L.tout})
    if (per) b += align_up(per * (size_t)Rc);
  return b;
}

struct Carver {
  uint8_t* p;
  template <class T>
  T* take(size_t per_ray, int64_t Rc) {
    if (!per_ray) return nullptr;
    T* r = reinterpret_cast<T*>(p);
    p += align_up(per_ray * (size_t)Rc);
    return r;
  }
};

inline pnr_composite_out offset_out(const pnr_composite_out& o, int64_t r0, int N, int C, int K) {
  pnr_composite_out q = o;
  if (q.rgb_map) q.rgb_map += r0 * 3;
  if (q.depth_map) q.depth_map += r0;
  if (q.acc_map) q.acc_map += r0;
  if (q.disp_map) q.disp_map += r0;
  if (q.weights) q.weights += r0 * N;
  if (q.semantic_map) q.semantic_map += r0 * C;
  if (q.instance_map) q.instance_map += r0 * K;
  if (q.fixed_semantic_map) q.fixed_semantic_map += r0 * C;
  if (q.fixed_instance_map) q.fixed_instance_map += r0 * K;
  return q;
}

}  // namespace

__global__ void __launch_bounds__(256) fill2_kernel(float* __restrict__ a, float va, float* __restrict__ b, float vb,
                                                    int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { a[i] = va; b[i] = vb; }
}

// Rays per chunk by default: raw of ~1.5 GB, never below ~64 tiles of the fused MLP per SM and pass (chunks small
// enough to keep raw L2-resident leave the persistent MLP kernel a few tiles per SM and launch, and its ramp-up / tail
// then costs more than the HBM round trip of raw saves).
int64_t default_chunk_rays(int Nt, int CH) {
  const size_t raw_per_ray = (size_t)Nt * CH * 4;
  int64_t by_bytes = (int64_t)((1536ull << 20) / raw_per_ray);
  const int64_t by_tiles = ((int64_t)num_sms() * 64 * kRows + Nt - 1) / Nt;
  return by_bytes > by_tiles ? by_bytes : by_tiles;
}

size_t workspace_bytes_for(int64_t R, int N, int Ni, int CH) {
  if (R <= 0) return 0;
  Ni = Ni > 0 ? Ni : 0;
  Layout L = make_layout(N, Ni, CH, PNR_MAX_HITS, true, nullptr);
  // sized for the worst case (a caller may ask for softmax compositing, which needs raw) when raw is small, for the
  // one-kernel path otherwise: with both heads raw is 456 B per sample against ~20 B of everything else
  if (L.raw == 0 && CH <= 8) L.raw = (size_t)L.Nt * CH * 4;
  int64_t Rc = L.raw ? default_chunk_rays(L.Nt, CH) : R;
  if (Rc > R) Rc = R;
  // A softmax call runs both passes on the two-kernel path, whose raw the one-kernel layout above leaves out: hold
  // min(R, ~64 samples per SM) rays of that layout too (cfg3: at most ~3.8 MB more, nothing more for a full frame).
  pnr_render_args softmax{};
  softmax.sem_softmax = 1;
  const Layout S = make_layout(N, Ni, CH, PNR_MAX_HITS, true, &softmax);
  int64_t Rs = ((int64_t)num_sms() * 64 + S.Nt - 1) / S.Nt;
  if (Rs > R) Rs = R;
  const size_t b = chunk_bytes(L, Rc), bs = chunk_bytes(S, Rs);
  return b > bs ? b : bs;
}

}  // namespace pnr

using namespace pnr;

#define PNR_TRY(call)              \
  do {                             \
    const int rc__ = (call);       \
    if (rc__ != PNR_OK) return rc__; \
  } while (0)

extern "C" int pnr_render_fused(pnr_ctx* ctx, pnr_ctx* ctx_fine, const pnr_render_args* a, void* stream) {
  PNR_CHECK_ARG(ctx && a, "pnr_render_fused: null pointer");
  if (a->R == 0) return PNR_OK;
  if (!ctx_fine) ctx_fine = ctx;
  const int N = a->N, Ni = a->Ni, M = a->M;
  int C = 0, K = 0, Cf = 0, Kf = 0;
  ctx_classes(ctx, &C, &K);
  ctx_classes(ctx_fine, &Cf, &Kf);
  const int CH = ctx_channels(ctx);
  // the maps are [R, C] / [R, K] of the coarse network, and both passes write them
  PNR_CHECK_ARG(Cf == C && Kf == K, "pnr_render_fused: the fine network's heads (C=%d, K=%d) differ from the coarse "
                "network's (C=%d, K=%d)", Cf, Kf, C, K);
  PNR_CHECK_ARG(a->R > 0 && a->rays, "pnr_render_fused: no rays");
  PNR_CHECK_ARG(N >= 1 && Ni >= 0 && N + Ni <= 256, "pnr_render_fused: N=%d, Ni=%d (N + Ni must be in [1,256])", N, Ni);
  PNR_CHECK_ARG(a->t_vals, "pnr_render_fused: t_vals is required (the caller's linspace(0,1,N))");
  PNR_CHECK_ARG((a->near != nullptr) == (a->far != nullptr), "pnr_render_fused: near and far come together");
  PNR_CHECK_ARG(!(a->perturb > 0.f) || a->u, "pnr_render_fused: perturb > 0 needs u");
  PNR_CHECK_ARG(Ni == 0 || (a->u_fine && N >= 3), "pnr_render_fused: Ni > 0 needs u_fine and N >= 3");
  const bool boxes = a->B > 0;
  PNR_CHECK_ARG(!boxes || (a->box_center && a->box_half && a->box_rot && M >= 1 && M <= PNR_MAX_HITS),
                "pnr_render_fused: bad primitive table (B=%d, M=%d)", a->B, M);
  PNR_CHECK_ARG((!a->mesh_tri_start && !a->mesh_tris && a->T == 0) ||
                    (a->mesh_tri_start && a->mesh_tris && a->T >= 1 && a->T < (int64_t(1) << 31)),
                "pnr_render_fused: mesh_tri_start (%s), mesh_tris (%s) and T=%lld: both null with T == 0, or both set "
                "with 1 <= T < 2^31", a->mesh_tri_start ? "set" : "null", a->mesh_tris ? "set" : "null", (long long)a->T);
  PNR_CHECK_ARG(a->sample_mode == PNR_SAMPLE_UNIFORM || (a->sample_mode == PNR_SAMPLE_INTERVALS && boxes),
                "pnr_render_fused: sample_mode %d (interval sampling needs primitives)", a->sample_mode);
  PNR_CHECK_ARG(a->workspace && a->workspace_bytes > 0, "pnr_render_fused: no workspace (see pnr_workspace_bytes)");

  const Layout L = make_layout(N, Ni, CH, boxes ? M : 0, boxes, a);
  // largest chunk the workspace holds (binary search on the aligned size)
  int64_t lo = 0, hi = a->R;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo + 1) / 2;
    if (chunk_bytes(L, mid) <= a->workspace_bytes) lo = mid; else hi = mid - 1;
  }
  const int64_t Rc = lo;
  if (Rc < 1)
    return set_error(PNR_ERR_ARG, "pnr_render_fused: workspace of %zu bytes cannot hold one ray (%zu bytes per ray)",
                     a->workspace_bytes, L.per_ray());
  cudaStream_t st = (cudaStream_t)stream;
  const bool fine = Ni > 0;
  const int Nt = N + Ni;

  for (int64_t r0 = 0; r0 < a->R; r0 += Rc) {
    const int64_t n = (a->R - r0 < Rc) ? a->R - r0 : Rc;
    Carver cv{reinterpret_cast<uint8_t*>(a->workspace)};
    float* raw = cv.take<float>(L.raw, Rc);
    float* z0_s = cv.take<float>(L.z0, Rc);
    float* zall_s = cv.take<float>(L.zall, Rc);
    float* w0_s = cv.take<float>(L.w0, Rc);
    float* w1_s = cv.take<float>(L.w1, Rc);
    int32_t* sb_s = cv.take<int32_t>(L.sb, Rc);
    float* near_s = cv.take<float>(L.near, Rc);
    float* far_s = cv.take<float>(L.far, Rc);
    uint8_t* hit_s = cv.take<uint8_t>(L.hit, Rc);
    int32_t* bid_s = cv.take<int32_t>(L.bid, Rc);
    float* tin_s = cv.take<float>(L.tin, Rc);
    float* tout_s = cv.take<float>(L.tout, Rc);

    const float* rays = a->rays + r0 * 6;
    float* near = L.have_nf ? a->near_out + r0 : near_s;
    float* far = L.have_nf ? a->far_out + r0 : far_s;
    // ---- near / far of this chunk (always a private copy: bound_by_primitives edits it in place)
    if (a->near) {
      PNR_CUDA(cudaMemcpyAsync(near, a->near + r0, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
      PNR_CUDA(cudaMemcpyAsync(far, a->far + r0, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    } else if (a->aabb_host) {
      PNR_TRY(pnr_scene_near_far(rays, n, a->aabb_host, a->near_min, a->far_default, near, far, stream));
    } else {
      fill2_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(near, a->near_min, far, a->far_default, n);
      PNR_LAUNCH_CHECK("fill2_kernel");
    }
    // ---- a5
    uint8_t* hit = nullptr; int32_t* bid = nullptr; float *tin = nullptr, *tout = nullptr;
    if (boxes) {
      hit = L.have_hits ? a->hit_mask + r0 : hit_s;
      bid = L.have_hits ? a->box_id + r0 * M : bid_s;
      tin = L.have_hits ? a->t_in + r0 * M : tin_s;
      tout = L.have_hits ? a->t_out + r0 * M : tout_s;
      if (a->T > 0)
        PNR_TRY(pnr_intersect_meshes(rays, n, a->box_center, a->box_half, a->box_rot, a->mesh_tri_start, a->mesh_tris,
                                     a->T, a->B, M, hit, bid, tin, tout, stream));
      else
        PNR_TRY(pnr_intersect(rays, n, a->box_center, a->box_half, a->box_rot, a->B, M, hit, bid, tin, tout, stream));
      if (a->bound_by_primitives) PNR_TRY(pnr_bound_by_primitives(hit, bid, tin, tout, n, M, near, far, stream));
    }
    // ---- a6: coarse depths + ids
    float* zall = L.have_z ? a->z_vals + r0 * Nt : zall_s;
    float* z0 = fine ? (L.have_z0 ? a->z_vals0 + r0 * N : z0_s) : zall;
    int32_t* sb = boxes ? (L.have_sb ? a->sample_box + r0 * Nt : sb_s) : nullptr;
    const float* u = a->u ? a->u + r0 * N : nullptr;
    if (a->sample_mode == PNR_SAMPLE_INTERVALS)
      PNR_TRY(pnr_sample_intervals(near, far, a->t_vals, u, n, N, a->perturb, bid, tin, tout, M, z0, sb, stream));
    else
      PNR_TRY(pnr_sample_stratified(near, far, a->t_vals, u, n, N, a->perturb, bid, tin, tout, boxes ? M : 0, z0, sb,
                                    stream));
    // ---- a8 + a9 (coarse pass, or the only pass): one kernel when the compositing epilogue applies
    pnr_composite_out o0 = offset_out(fine ? a->out0 : a->out, r0, N, C, K);
    if (!o0.weights) o0.weights = w0_s;
    if (L.comp0) {
      PNR_TRY(pnr_mlp_composite(ctx, rays, z0, n, N, a->white_bkgd, a->mask_outside, sb, a->box_sem, a->box_inst, a->B,
                                &o0, stream));
    } else {
      PNR_TRY(pnr_mlp_forward(ctx, nullptr, nullptr, rays, z0, n, N, raw, stream));
      PNR_TRY(pnr_composite(raw, z0, rays, n, N, C, K, a->white_bkgd, a->sem_softmax, a->mask_outside, sb, a->box_sem,
                            a->box_inst, a->B, &o0, stream));
    }
    if (!fine) continue;
    // ---- a10 + fine pass
    const float* uf = a->u_fine + (a->u_fine_stride ? r0 * a->u_fine_stride : 0);
    PNR_TRY(sample_pdf_strided(z0, o0.weights, n, N, Ni, uf, a->u_fine_stride, nullptr, nullptr, zall, stream));
    if (boxes) PNR_TRY(pnr_tag_samples(zall, n, Nt, bid, tin, tout, M, sb, stream));
    pnr_composite_out o1 = offset_out(a->out, r0, Nt, C, K);
    if (!o1.weights) o1.weights = w1_s;
    if (L.comp1) {
      PNR_TRY(pnr_mlp_composite(ctx_fine, rays, zall, n, Nt, a->white_bkgd, a->mask_outside, sb, a->box_sem, a->box_inst,
                                a->B, &o1, stream));
    } else {
      PNR_TRY(pnr_mlp_forward(ctx_fine, nullptr, nullptr, rays, zall, n, Nt, raw, stream));
      PNR_TRY(pnr_composite(raw, zall, rays, n, Nt, C, K, a->white_bkgd, a->sem_softmax, a->mask_outside, sb, a->box_sem,
                            a->box_inst, a->B, &o1, stream));
    }
  }
  return PNR_OK;
}
