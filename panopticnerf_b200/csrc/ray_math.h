// ray_math.h — per-ray arithmetic with a fully specified fp32 operation order, shared by the CUDA
// kernels (ray_kernels.cu, rays_kernel, ray_batch_kernel and the depth kernels in stream_kernels.cu, the weight kernels
// in weight_kernels.cu) and the host build
// used by the CPU tests (tests/host_emu.cpp; the weighted draws' routines in tests/host_emu_weights.cpp) to prove the
// order matches the oracle bit for bit without a GPU.  The kernels keep only layout
// here (staging, shuffles, sorts); the rules they apply per ray - the per-primitive intersection step, range clamps,
// sample depths, output slots, camera directions, batch draws - are the functions below, called by both builds.  One
// piece stays written out in stratified_kernel and again in host_emu.cpp: the interval test (pnr_tag's rule), because
// a predicate shared with pnr_tag makes pnr_tag load t_in / t_out before it tests the id, which changes the SASS of
// tag_kernel and interval_kernel.
//
// Rules (SURVEY.md 7.3 item 3): every multiply/add/subtract/divide is individually rounded (no FMA
// contraction: __f*_rn intrinsics on device, -ffp-contract=off on host), true division, and min/max
// propagate NaN like torch.minimum/torch.maximum.
#pragma once
#include <stdint.h>
#include <math.h>
#include <string.h>
#include "../../include/pnr.h"   // pnr_ray_batch_args: the ray-batch routine reads the entry point's own arguments

#if defined(__CUDACC__)
#define PNR_HD __host__ __device__ __forceinline__
#else
#define PNR_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define PNR_MUL(a, b) __fmul_rn((a), (b))
#define PNR_ADD(a, b) __fadd_rn((a), (b))
#define PNR_SUB(a, b) __fsub_rn((a), (b))
#define PNR_DIV(a, b) __fdiv_rn((a), (b))
#define PNR_DADD(a, b) __dadd_rn((a), (b))
#define PNR_DSUB(a, b) __dsub_rn((a), (b))
#define PNR_DMUL(a, b) __dmul_rn((a), (b))
#define PNR_DDIV(a, b) __ddiv_rn((a), (b))
#define PNR_SQRT(a) __fsqrt_rn((a))
#define PNR_LDG(p) __ldg((p))
#else
#define PNR_MUL(a, b) ((a) * (b))
#define PNR_ADD(a, b) ((a) + (b))
#define PNR_SUB(a, b) ((a) - (b))
#define PNR_DIV(a, b) ((a) / (b))
#define PNR_DADD(a, b) ((a) + (b))
#define PNR_DSUB(a, b) ((a) - (b))
#define PNR_DMUL(a, b) ((a) * (b))
#define PNR_DDIV(a, b) ((a) / (b))
#define PNR_SQRT(a) sqrtf((a))
#define PNR_LDG(p) (*(p))
#endif

#define PNR_MAX_HITS 8
#define PNR_FISHEYE_NEWTON 8   // fixed iteration count: the ray is a pure function of the pixel

PNR_HD float pnr_min_nan(float a, float b) { return (a != a) ? a : ((b != b) ? b : (b < a ? b : a)); }
PNR_HD float pnr_max_nan(float a, float b) { return (a != a) ? a : ((b != b) ? b : (b > a ? b : a)); }

PNR_HD float pnr_dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
  return PNR_ADD(PNR_ADD(PNR_MUL(a0, b0), PNR_MUL(a1, b1)), PNR_MUL(a2, b2));
}

// a5: slab test of one ray against one oriented box.  rot is row-major 3x3, columns = box axes.
PNR_HD bool pnr_slab(float ox, float oy, float oz, float dx, float dy, float dz, const float* c,
                     const float* h, const float* rot, float* tmin_out, float* tmax_out) {
  const float ocx = PNR_SUB(ox, c[0]), ocy = PNR_SUB(oy, c[1]), ocz = PNR_SUB(oz, c[2]);
  float tmin = 0.f, tmax = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float a0 = rot[0 + j], a1 = rot[3 + j], a2 = rot[6 + j];
    const float oj = pnr_dot3(ocx, ocy, ocz, a0, a1, a2);
    const float dj = pnr_dot3(dx, dy, dz, a0, a1, a2);
    const float t0 = PNR_DIV(PNR_SUB(-h[j], oj), dj);
    const float t1 = PNR_DIV(PNR_SUB(h[j], oj), dj);
    const float lo = pnr_min_nan(t0, t1), hi = pnr_max_nan(t0, t1);
    tmin = (j == 0) ? lo : pnr_max_nan(tmin, lo);
    tmax = (j == 0) ? hi : pnr_min_nan(tmax, hi);
  }
  *tmin_out = tmin;
  *tmax_out = tmax;
  return tmax > pnr_max_nan(tmin, 0.f);
}

// Sorted (by tmin, ties -> lower box index) list of the M nearest hits, kept in registers.
struct PnrHitList {
  float key[PNR_MAX_HITS];
  float tout[PNR_MAX_HITS];
  int32_t id[PNR_MAX_HITS];
  int n;
};
PNR_HD void pnr_hits_init(PnrHitList* L) {
  L->n = 0;
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m) { L->key[m] = 0.f; L->tout[m] = 0.f; L->id[m] = -1; }
}
PNR_HD void pnr_hits_insert(PnrHitList* L, int M, float tmin, float tmax, int32_t b) {
  // position = first p with key[p] > tmin (stable: equal keys keep box-index order)
  int p = L->n;
#pragma unroll
  for (int m = PNR_MAX_HITS - 1; m >= 0; --m)
    if (m < L->n && L->key[m] > tmin) p = m;
  if (p >= M) return;
#pragma unroll
  for (int m = PNR_MAX_HITS - 1; m >= 1; --m)
    if (m > p && m < M) { L->key[m] = L->key[m - 1]; L->tout[m] = L->tout[m - 1]; L->id[m] = L->id[m - 1]; }
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m)
    if (m == p) { L->key[m] = tmin; L->tout[m] = tmax; L->id[m] = b; }
  if (L->n < M) L->n += 1;
}

// a5, mesh primitives (DESIGN 3.2).  A primitive given as a closed triangle mesh: its box is only a cull volume, and
// its hit intervals come from the crossings of the ray's line with the triangles.
//
// Crossing: the watertight ray/triangle test of Woop, Benthin and Wald (JCGT 2013).  The vertices are translated to
// the ray origin, the axes permuted so that the largest |d| component is z (ties -> the lower axis), and sheared so
// that the ray becomes the z axis.  The 2D edge functions U, V, W are individually rounded fp32; one that is exactly 0
// is re-evaluated in double (the products of two floats are exact there, so its sign is exact).  One that is still 0
// is resolved by a half-open tie rule that depends only on the edge's two sheared endpoints P -> Q: the sign the edge
// function takes for the origin displaced to (eps, eps^2), i.e. sign(Py - Qy), else sign(Qx - Px).  The rule is
// antisymmetric in P, Q, so across an edge or vertex that triangles of a closed mesh share, a ray crosses exactly one
// of them, and a tangent touch counts an even number of times.  det = U + V + W == 0 (the ray in the triangle's
// plane) is no crossing.  t = T / det in fp32, on the whole line (either sign); a NaN t is no crossing.
struct PnrShear {
  int kx, ky, kz;
  float sx, sy, sz;
};
PNR_HD float pnr_pick3(float a, float b, float c, int k) { return k == 0 ? a : (k == 1 ? b : c); }
PNR_HD PnrShear pnr_shear(float dx, float dy, float dz) {
  const float ax = fabsf(dx), ay = fabsf(dy), az = fabsf(dz);
  int kz = ay > ax ? 1 : 0;
  if (az > (kz == 0 ? ax : ay)) kz = 2;
  int kx = kz == 2 ? 0 : kz + 1;
  int ky = kx == 2 ? 0 : kx + 1;
  const float dk = pnr_pick3(dx, dy, dz, kz);
  if (dk < 0.f) { const int s = kx; kx = ky; ky = s; }   // keeps the winding (the test is two-sided anyway)
  PnrShear S;
  S.kx = kx; S.ky = ky; S.kz = kz;
  S.sx = PNR_DIV(pnr_pick3(dx, dy, dz, kx), dk);
  S.sy = PNR_DIV(pnr_pick3(dx, dy, dz, ky), dk);
  S.sz = PNR_DIV(1.0f, dk);
  return S;
}
// sign of the edge function e = Px*Qy - Py*Qx of the sheared edge P -> Q, e its fp32 value and ed its double value
// (used when e == 0); 0 only for a degenerate edge (P == Q)
PNR_HD int pnr_edge_sign(float e, double ed, bool redo, float px, float py, float qx, float qy) {
  if (redo) {
    if (ed > 0.0) return 1;
    if (ed < 0.0) return -1;
  } else {
    if (e > 0.f) return 1;
    if (e < 0.f) return -1;
  }
  if (py != qy) return py > qy ? 1 : -1;
  if (qx != px) return qx > px ? 1 : -1;
  return 0;
}
// v = the triangle's 9 floats (v0, v1, v2).  Returns whether the line crosses it, and where (*t).
PNR_HD bool pnr_tri_cross(float ox, float oy, float oz, const PnrShear& S, const float* v, float* t) {
  float ax, ay, az, bx, by, bz, cx, cy, cz;
  {
    const float a0 = PNR_SUB(v[0], ox), a1 = PNR_SUB(v[1], oy), a2 = PNR_SUB(v[2], oz);
    const float b0 = PNR_SUB(v[3], ox), b1 = PNR_SUB(v[4], oy), b2 = PNR_SUB(v[5], oz);
    const float c0 = PNR_SUB(v[6], ox), c1 = PNR_SUB(v[7], oy), c2 = PNR_SUB(v[8], oz);
    az = pnr_pick3(a0, a1, a2, S.kz); bz = pnr_pick3(b0, b1, b2, S.kz); cz = pnr_pick3(c0, c1, c2, S.kz);
    ax = PNR_SUB(pnr_pick3(a0, a1, a2, S.kx), PNR_MUL(S.sx, az));
    ay = PNR_SUB(pnr_pick3(a0, a1, a2, S.ky), PNR_MUL(S.sy, az));
    bx = PNR_SUB(pnr_pick3(b0, b1, b2, S.kx), PNR_MUL(S.sx, bz));
    by = PNR_SUB(pnr_pick3(b0, b1, b2, S.ky), PNR_MUL(S.sy, bz));
    cx = PNR_SUB(pnr_pick3(c0, c1, c2, S.kx), PNR_MUL(S.sx, cz));
    cy = PNR_SUB(pnr_pick3(c0, c1, c2, S.ky), PNR_MUL(S.sy, cz));
  }
  float U = PNR_SUB(PNR_MUL(cx, by), PNR_MUL(cy, bx));   // edge C -> B
  float V = PNR_SUB(PNR_MUL(ax, cy), PNR_MUL(ay, cx));   // edge A -> C
  float W = PNR_SUB(PNR_MUL(bx, ay), PNR_MUL(by, ax));   // edge B -> A
  double Ud = 0.0, Vd = 0.0, Wd = 0.0;
  const bool redo = U == 0.f || V == 0.f || W == 0.f;
  if (redo) {
    Ud = PNR_DSUB(PNR_DMUL((double)cx, (double)by), PNR_DMUL((double)cy, (double)bx));
    Vd = PNR_DSUB(PNR_DMUL((double)ax, (double)cy), PNR_DMUL((double)ay, (double)cx));
    Wd = PNR_DSUB(PNR_DMUL((double)bx, (double)ay), PNR_DMUL((double)by, (double)ax));
    U = (float)Ud; V = (float)Vd; W = (float)Wd;
  }
  const int su = pnr_edge_sign(U, Ud, redo, cx, cy, bx, by);
  const int sv = pnr_edge_sign(V, Vd, redo, ax, ay, cx, cy);
  const int sw = pnr_edge_sign(W, Wd, redo, bx, by, ax, ay);
  if (!((su > 0 && sv > 0 && sw > 0) || (su < 0 && sv < 0 && sw < 0))) return false;
  const float det = PNR_ADD(PNR_ADD(U, V), W);
  if (det == 0.f) return false;
  const float T = PNR_ADD(PNR_ADD(PNR_MUL(U, PNR_MUL(S.sz, az)), PNR_MUL(V, PNR_MUL(S.sz, bz))),
                          PNR_MUL(W, PNR_MUL(S.sz, cz)));
  *t = PNR_DIV(T, det);
  return *t == *t;
}

// Crossings of one mesh -> its hit intervals.  Sorted along the line, the crossings c0 <= c1 <= ... pair up as the
// inside intervals (c0,c1), (c2,c3), ...; an odd count (an open mesh, a degenerate ray) gives the one hull interval
// [first, last].  An interval (a, b) with b > 0 is a candidate; a mesh's first M candidates are kept, and of those the
// ones with b > max(a, 0) are hits (zero-length ones are not), inserted in order with key a.  So only the parity and
// the largest of the crossings at t <= 0, the 2M smallest at t > 0, the count and the extremes are needed: exact, in
// registers.
struct PnrMeshCross {
  float pos[2 * PNR_MAX_HITS];   // the smallest crossings at t > 0, ascending
  int npos;                      // entries of pos in use (<= 2M)
  int n;                         // crossings in all
  int nneg;                      // crossings at t <= 0
  float neg_max;                 // the largest of them
  float lo, hi;                  // the smallest and largest crossing
};
PNR_HD void pnr_cross_init(PnrMeshCross* S) {
  S->npos = 0; S->n = 0; S->nneg = 0;
  S->neg_max = 0.f; S->lo = 0.f; S->hi = 0.f;
#pragma unroll
  for (int m = 0; m < 2 * PNR_MAX_HITS; ++m) S->pos[m] = 0.f;
}
PNR_HD void pnr_cross_add(PnrMeshCross* S, int M, float t) {
  S->lo = (S->n == 0 || t < S->lo) ? t : S->lo;
  S->hi = (S->n == 0 || t > S->hi) ? t : S->hi;
  S->n += 1;
  if (t <= 0.f) {
    S->neg_max = (S->nneg == 0 || t > S->neg_max) ? t : S->neg_max;
    S->nneg += 1;
    return;
  }
  const int cap = 2 * M;
  int p = S->npos;   // first p with pos[p] > t
#pragma unroll
  for (int m = 2 * PNR_MAX_HITS - 1; m >= 0; --m)
    if (m < S->npos && S->pos[m] > t) p = m;
  if (p >= cap) return;
#pragma unroll
  for (int m = 2 * PNR_MAX_HITS - 1; m >= 1; --m)
    if (m > p && m < cap) S->pos[m] = S->pos[m - 1];
#pragma unroll
  for (int m = 0; m < 2 * PNR_MAX_HITS; ++m)
    if (m == p) S->pos[m] = t;
  if (S->npos < cap) S->npos += 1;
}
PNR_HD void pnr_cross_emit(const PnrMeshCross* S, PnrHitList* L, int M, int32_t b) {
  if (S->n == 0) return;
  if (S->n & 1) {
    if (S->hi > pnr_max_nan(S->lo, 0.f)) pnr_hits_insert(L, M, S->lo, S->hi, b);
    return;
  }
  int j = 0, kept = 0;
  if (S->nneg & 1) {   // the interval around the origin: its exit is the first crossing at t > 0
    pnr_hits_insert(L, M, S->neg_max, S->pos[0], b);
    j = 1;
    kept = 1;
  }
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m) {
    const int i = j + 2 * m;
    if (kept < M && i + 1 < S->npos) {
      float a = 0.f, c = 0.f;
#pragma unroll
      for (int q = 0; q < 2 * PNR_MAX_HITS; ++q) {   // register-resident: no dynamic indexing
        if (q == i) a = S->pos[q];
        if (q == i + 1) c = S->pos[q];
      }
      if (c > a) pnr_hits_insert(L, M, a, c, b);
      kept += 1;
    }
  }
}

// intersect_kernel's per-primitive step for primitive b: the slab test of its box q (center, half, rot: 15 floats),
// then on a hit either the box's own interval (an empty triangle range: a cuboid) or the intervals of the mesh made of
// triangles [k0, k1) of tris.
PNR_HD void pnr_prim_step(float ox, float oy, float oz, float dx, float dy, float dz, const float* q, int k0, int k1,
                          const float* tris, int M, int32_t b, PnrHitList* L) {
  float tmin, tmax;
  const bool hit = pnr_slab(ox, oy, oz, dx, dy, dz, q, q + 3, q + 6, &tmin, &tmax);
  if (k0 == k1) {
    if (hit) pnr_hits_insert(L, M, tmin, tmax, b);
  } else if (hit) {
    const PnrShear S = pnr_shear(dx, dy, dz);
    PnrMeshCross X;
    pnr_cross_init(&X);
    for (int k = k0; k < k1; ++k) {
      float v[9];
#pragma unroll
      for (int e = 0; e < 9; ++e) v[e] = PNR_LDG(tris + (int64_t)k * 9 + e);
      float t;
      if (pnr_tri_cross(ox, oy, oz, S, v, &t)) pnr_cross_add(&X, M, t);
    }
    pnr_cross_emit(&X, L, M, b);
  }
}

// Triangle range [*k0, *k1) of primitive b, clamped into [0, T], so a malformed start table cannot read outside the
// triangle table.  T < 2^31 (pnr_intersect_meshes checks it), so the range fits in int.
PNR_HD void pnr_tri_range(const int32_t* tri_start, int b, int64_t T, int* k0, int* k1) {
  const int64_t s0 = tri_start[b], s1 = tri_start[b + 1];
  int64_t lo = s0 > 0 ? s0 : 0;
  lo = lo < T ? lo : T;
  int64_t hi = s1 > lo ? s1 : lo;
  hi = hi < T ? hi : T;
  *k0 = (int)lo;
  *k1 = (int)hi;
}
// Dynamic block [*b0, *b1) of frame f in a sequence table of S static and Bt primitives (DESIGN 3.2): the entry
// frame_boxes[f] = (begin, end) clamped into [S, Bt], empty when end < begin; a frame outside [0, F) has no block, so
// its rays meet the static primitives only.
PNR_HD void pnr_frame_range(int f, const int32_t* frame_boxes, int F, int S, int Bt, int* b0, int* b1) {
  int lo = S, hi = S;
  if (f >= 0 && f < F) {
    const int a = frame_boxes[2 * f], e = frame_boxes[2 * f + 1];
    lo = a < S ? S : (a > Bt ? Bt : a);
    hi = e < lo ? lo : (e > Bt ? Bt : e);
  }
  *b0 = lo;
  *b1 = hi;
}
// Output slots of ray r: the M nearest hits, then padding (id -1, depths 0); t_in starts at the origin.
PNR_HD void pnr_hits_store(const PnrHitList* L, int M, int64_t r, uint8_t* hit, int32_t* box_id, float* t_in,
                           float* t_out) {
  hit[r] = L->n > 0 ? 1 : 0;
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m)
    if (m < M) {
      const bool v = m < L->n;
      box_id[r * M + m] = v ? L->id[m] : -1;
      t_in[r * M + m] = v ? pnr_max_nan(L->key[m], 0.f) : 0.f;
      t_out[r * M + m] = v ? L->tout[m] : 0.f;
    }
}

// a6
PNR_HD float pnr_strat_z(float near, float far, float t) {
  return PNR_ADD(PNR_MUL(near, PNR_SUB(1.0f, t)), PNR_MUL(far, t));
}
PNR_HD float pnr_strat_z_jitter(float near, float far, const float* t_vals, int i, int N, float u) {
  const float zi = pnr_strat_z(near, far, t_vals[i]);
  float lower = zi, upper = zi;
  if (i > 0) lower = PNR_MUL(0.5f, PNR_ADD(zi, pnr_strat_z(near, far, t_vals[i - 1])));
  if (i < N - 1) upper = PNR_MUL(0.5f, PNR_ADD(pnr_strat_z(near, far, t_vals[i + 1]), zi));
  return PNR_ADD(lower, PNR_MUL(PNR_SUB(upper, lower), u));
}
// depth of sample i of a ray (u_row: the ray's jitter row, read only when perturb > 0)
PNR_HD float pnr_sample_z(float near, float far, const float* t_vals, const float* u_row, int i, int N,
                          float perturb) {
  return (perturb > 0.f) ? pnr_strat_z_jitter(near, far, t_vals, i, N, u_row[i]) : pnr_strat_z(near, far, t_vals[i]);
}
PNR_HD int32_t pnr_tag(float z, const int32_t* box_id, const float* t_in, const float* t_out, int M) {
  for (int m = 0; m < M; ++m)
    if (box_id[m] >= 0 && z >= t_in[m] && z <= t_out[m]) return box_id[m];
  return -1;
}

// a6, interval mode: the N samples of a ray are placed INSIDE its hit intervals (the reference samples inside
// ray/primitive intersections; how it divides the samples is not in the mount - SURVEY 8(c) question 4 - so the
// rule below is chosen here and stated in DESIGN.md as "chosen, unverified"):
//   1. every valid interval m (box_id >= 0) is clipped to [near, far]: a = max(t_in, near), b = min(t_out, far),
//      len = b - a, kept when len > 0;
//   2. L = sum of the kept lengths in interval order (nearest first); interval m gets
//      n_m = min(floor(N * len_m / L), samples still unassigned) samples, in interval order; what is left after
//      that goes one sample at a time to the kept intervals, nearest first (cyclically);
//   3. sample j of interval m sits at a + (b - a) * ((j + c) / n_m), c = 0.5 (or the jitter u of that sample slot
//      when perturb > 0);
//   4. the N depths are sorted ascending (pnr_tag then names the first interval containing each).
// A ray with no kept interval falls back to the uniform near..far rule.  All arithmetic is individually rounded fp32.
struct PnrIntervalPlan {
  float a[PNR_MAX_HITS], b[PNR_MAX_HITS];
  int n[PNR_MAX_HITS];      // samples per interval (0 for dropped ones)
  int first[PNR_MAX_HITS];  // slot of its first sample in allocation order
  int kept;                 // number of kept intervals (0 -> uniform fallback)
};
PNR_HD void pnr_interval_plan(float near, float far, const int32_t* box_id, const float* t_in, const float* t_out,
                              int M, int N, PnrIntervalPlan* P) {
  float len[PNR_MAX_HITS];
  float L = 0.f;
  P->kept = 0;
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m) {
    P->a[m] = 0.f; P->b[m] = 0.f; P->n[m] = 0; P->first[m] = 0; len[m] = 0.f;
    if (m < M && box_id[m] >= 0) {
      const float a = pnr_max_nan(t_in[m], near), b = pnr_min_nan(t_out[m], far);
      const float l = PNR_SUB(b, a);
      if (l > 0.f) {
        P->a[m] = a; P->b[m] = b; len[m] = l;
        L = (P->kept == 0) ? l : PNR_ADD(L, l);
        P->kept += 1;
      }
    }
  }
  if (P->kept == 0) return;
  int left = N;
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m) {
    if (len[m] > 0.f) {
      int q = (int)floorf(PNR_DIV(PNR_MUL((float)N, len[m]), L));
      if (q > left) q = left;
      if (q < 0) q = 0;
      P->n[m] = q;
      left -= q;
    }
  }
  while (left > 0) {   // at most `kept` passes are ever needed in exact arithmetic; cyclic for safety
#pragma unroll
    for (int m = 0; m < PNR_MAX_HITS; ++m)
      if (len[m] > 0.f && left > 0) { P->n[m] += 1; left -= 1; }
  }
  int off = 0;
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m) { P->first[m] = off; off += P->n[m]; }
}
// depth of allocation slot k (before the sort); c = 0.5 or the slot's jitter
PNR_HD float pnr_interval_z(const PnrIntervalPlan* P, int k, float c) {
  float z = 0.f;
#pragma unroll
  for (int m = 0; m < PNR_MAX_HITS; ++m) {
    const int j = k - P->first[m];
    if (j >= 0 && j < P->n[m]) {
      const float t = PNR_DIV(PNR_ADD((float)j, c), (float)P->n[m]);
      z = PNR_ADD(P->a[m], PNR_MUL(PNR_SUB(P->b[m], P->a[m]), t));
    }
  }
  return z;
}
// the same with the slot's c chosen (u_row: the ray's jitter row, read only when perturb > 0)
PNR_HD float pnr_interval_slot_z(const PnrIntervalPlan* P, const float* u_row, int k, float perturb) {
  return pnr_interval_z(P, k, (perturb > 0.f) ? u_row[k] : 0.5f);
}

// a10: cdf over the Nb = N-1 bin edges from coarse weights[0..N-1] (uses weights[1..N-2]).
// Sequential running sums with a double accumulator rounded to fp32 per element (= torch.cumsum CPU).
PNR_HD void pnr_pdf_cdf(const float* weights, int N, float* cdf /* [N-1] */) {
  const int nw = N - 2;
  double acc = 0.0;
  for (int k = 0; k < nw; ++k) acc = PNR_DADD(acc, (double)PNR_ADD(weights[k + 1], 1e-5f));
  const float total = (float)acc;
  acc = 0.0;
  cdf[0] = 0.f;
  for (int k = 0; k < nw; ++k) {
    const float pdf = PNR_DIV(PNR_ADD(weights[k + 1], 1e-5f), total);
    acc = PNR_DADD(acc, (double)pdf);
    cdf[k + 1] = (float)acc;
  }
}
// searchsorted(cdf, u, right=True): number of entries <= u.
PNR_HD int pnr_searchsorted_right(const float* cdf, int n, float u) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
  }
  return lo;
}
PNR_HD float pnr_bin_mid(const float* z, int k) { return PNR_MUL(0.5f, PNR_ADD(z[k + 1], z[k])); }
PNR_HD float pnr_pdf_sample(const float* z, const float* cdf, int Nb, float u, int* idx_out) {
  const int idx = pnr_searchsorted_right(cdf, Nb, u);
  const int below = idx - 1 > 0 ? idx - 1 : 0;
  const int above = idx < Nb - 1 ? idx : Nb - 1;
  const float cb = cdf[below], ca = cdf[above];
  const float bb = pnr_bin_mid(z, below), ba = pnr_bin_mid(z, above);
  float denom = PNR_SUB(ca, cb);
  if (denom < 1e-5f) denom = 1.0f;
  const float t = PNR_DIV(PNR_SUB(u, cb), denom);
  *idx_out = idx;
  return PNR_ADD(bb, PNR_MUL(t, PNR_SUB(ba, bb)));
}

// 8(f) rank 3: KITTI-360 fisheye (unified / MEI model; intr = gamma1, gamma2, u0, v0, xi, k1, k2).  Pixel (u, v) ->
// direction on the unit sphere in the camera frame.  m = distorted normalised point; radial undistortion
// rd = ro (1 + k1 ro^2 + k2 ro^4) solved for ro by PNR_FISHEYE_NEWTON Newton steps from ro = rd; lift:
// X = (f x, f y, f - xi), f = (xi + sqrt(max(1 + (1 - xi^2) r^2, 0))) / (1 + r^2)  (xi > 1: beyond the mirror's
// field of view the radicand is negative; it is clamped and the caller masks those pixels).
PNR_HD void pnr_fisheye_dir(float u, float v, float g1, float g2, float u0, float v0, float xi, float k1, float k2,
                            float* x, float* y, float* z) {
  const float mx = PNR_DIV(PNR_SUB(u, u0), g1);
  const float my = PNR_DIV(PNR_SUB(v, v0), g2);
  const float rd = PNR_SQRT(PNR_ADD(PNR_MUL(mx, mx), PNR_MUL(my, my)));
  const float k1x3 = PNR_MUL(3.0f, k1), k2x5 = PNR_MUL(5.0f, k2);
  float ro = rd;
  for (int it = 0; it < PNR_FISHEYE_NEWTON; ++it) {
    const float ro2 = PNR_MUL(ro, ro);
    const float f = PNR_SUB(PNR_MUL(ro, PNR_ADD(1.0f, PNR_MUL(ro2, PNR_ADD(k1, PNR_MUL(k2, ro2))))), rd);
    const float fp = PNR_ADD(1.0f, PNR_MUL(ro2, PNR_ADD(k1x3, PNR_MUL(k2x5, ro2))));
    ro = PNR_SUB(ro, PNR_DIV(f, fp));
  }
  const float scale = rd > 0.f ? PNR_DIV(ro, rd) : 1.0f;
  const float px = PNR_MUL(mx, scale), py = PNR_MUL(my, scale);
  const float r2 = PNR_ADD(PNR_MUL(px, px), PNR_MUL(py, py));
  float rad = PNR_ADD(1.0f, PNR_MUL(PNR_SUB(1.0f, PNR_MUL(xi, xi)), r2));
  if (rad < 0.f) rad = 0.f;
  const float fac = PNR_DIV(PNR_ADD(xi, PNR_SQRT(rad)), PNR_ADD(1.0f, r2));
  *x = PNR_MUL(fac, px);
  *y = PNR_MUL(fac, py);
  *z = PNR_SUB(fac, xi);
}
// Pinhole camera: pixel (u, v) -> unnormalised direction (x, y, 1) in the camera frame.
PNR_HD void pnr_pinhole_dir(float u, float v, float fx, float fy, float cx, float cy, float* x, float* y, float* z) {
  *x = PNR_DIV(PNR_SUB(u, cx), fx);
  *y = PNR_DIV(PNR_SUB(v, cy), fy);
  *z = 1.0f;
}
// Camera-frame direction -> world frame by the rotation of c2w (row-major 3x4 [R|t]).
PNR_HD void pnr_cam_to_world(const float* c2w, float x, float y, float z, float* d0, float* d1, float* d2) {
  *d0 = PNR_ADD(PNR_ADD(PNR_MUL(c2w[0], x), PNR_MUL(c2w[1], y)), PNR_MUL(c2w[2], z));
  *d1 = PNR_ADD(PNR_ADD(PNR_MUL(c2w[4], x), PNR_MUL(c2w[5], y)), PNR_MUL(c2w[6], z));
  *d2 = PNR_ADD(PNR_ADD(PNR_MUL(c2w[8], x), PNR_MUL(c2w[9], y)), PNR_MUL(c2w[10], z));
}

// ---------------------------------------------------------------------------------------------- training ray batches
// pnr_sample_ray_batch (include/pnr.h; DESIGN 3.4): a random pixel of a frame set per ray, its camera ray, targets and
// jitter, all a function of (seed, step, global ray index).  Integer work (Philox, the 64-bit multiply, the search) is
// exact on both builds; the float work is the camera routines above and one true division per colour channel.

// Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC 2011): 10 rounds of two 32x32 -> 64-bit multiplies, the key bumped by
// the Weyl constants between rounds.
PNR_HD void pnr_mulhilo32(uint32_t a, uint32_t b, uint32_t* hi, uint32_t* lo) {
#if defined(__CUDA_ARCH__)
  *hi = __umulhi(a, b);
  *lo = a * b;
#else
  const uint64_t p = (uint64_t)a * b;
  *hi = (uint32_t)(p >> 32);
  *lo = (uint32_t)p;
#endif
}
PNR_HD void pnr_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                              uint32_t out[4]) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    uint32_t hi0, lo0, hi1, lo1;
    pnr_mulhilo32(0xD2511F53u, c0, &hi0, &lo0);
    pnr_mulhilo32(0xCD9E8D57u, c2, &hi1, &lo1);
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
// block `block` of ray r: counter (block, r, step low word, step high word), key = the seed (low word first)
PNR_HD void pnr_ray_draw(uint64_t seed, uint64_t step, int64_t r, uint32_t block, uint32_t out[4]) {
  pnr_philox4x32_10(block, (uint32_t)r, (uint32_t)step, (uint32_t)(step >> 32), (uint32_t)seed, (uint32_t)(seed >> 32),
                    out);
}
// high 64 bits of the 128-bit product a * b: a uniform 64-bit a gives an index in [0, b), biased by at most b / 2^64
PNR_HD uint64_t pnr_mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
// a 32-bit word -> [0, 1) on the 2^-24 grid (exact in fp32)
PNR_HD float pnr_u01(uint32_t w) { return (float)(w >> 8) * 5.9604644775390625e-08f; }
// frame of flat pixel p: the last f with off[f] <= p (upper bound over off[0..F]), clamped into [0, F)
PNR_HD int pnr_frame_of(const int64_t* off, int F, int64_t p) {
  int lo = 0, hi = F + 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= p) lo = mid + 1; else hi = mid;
  }
  const int f = lo - 1;
  return f < 0 ? 0 : (f >= F ? F - 1 : f);
}
// an 8-bit colour channel -> [0, 1], as torch's u8.float() / 255 on the CPU (true division)
PNR_HD float pnr_u8_unit(uint8_t b) { return PNR_DIV((float)b, 255.0f); }

// ---------------------------------------------------------------------------------------------- weighted draws
// pnr_pixel_weights / pnr_pixel_cdf / pnr_sample_ray_batch_weighted (include/pnr.h; DESIGN 3.4).

#define PNR_WEIGHT_GROUP 32         // pixels per entry of the weight table's prefix sum
#define PNR_WEIGHT_MAX 65535.0f

// the class-factor slot of a label: 1 + label for a label in [0, C), else 0 (-1 and every other value)
PNR_HD int pnr_weight_slot(int16_t label, int C) { return (label >= 0 && label < C) ? 1 + label : 0; }
// one pixel's weight: x = (scale * frame_factor) * class_factor in fp32, each product rounded; 0 when masked, NaN or
// x <= 0; 65535 when x >= 65535 (+Inf too); otherwise x rounded to the nearest integer, ties to even (adding and
// subtracting 2^23 rounds a float in [0, 2^23) to an integer in the current mode, round-to-nearest-even)
PNR_HD uint16_t pnr_pixel_weight(bool keep, float scale, float frame_factor, float class_factor) {
  if (!keep) return 0;
  const float x = PNR_MUL(PNR_MUL(scale, frame_factor), class_factor);
  if (!(x > 0.f)) return 0;
  if (x >= PNR_WEIGHT_MAX) return 65535;
  return (uint16_t)PNR_SUB(PNR_ADD(x, 8388608.0f), 8388608.0f);
}
// pixel q of frame f (camera cam, of n clamped pixels starting at lo) under the rule above.  A camera mask covers the
// camera's H W pixels; a pixel past them (a malformed table) is not kept.
PNR_HD uint16_t pnr_weight_of_pixel(const pnr_pixel_weights_args& a, int f, int cam, int64_t lo, int64_t q) {
  const uint8_t* mask = a.mask[0];
#pragma unroll
  for (int k = 1; k < PNR_RAY_BATCH_MAX_CAMERAS; ++k)
    if (k == cam) mask = a.mask[k];
  int64_t HW = 0;
#pragma unroll
  for (int k = 0; k < PNR_RAY_BATCH_MAX_CAMERAS; ++k)
    if (k == cam) HW = (int64_t)a.cams[k].H * a.cams[k].W;
  const bool keep = q < HW && (mask == nullptr || mask[q] != 0);
  const float ff = a.frame_factor ? a.frame_factor[f] : 1.0f;
  const int slot = a.label ? pnr_weight_slot(a.label[lo + q], a.C) : 0;
  const float cf = a.class_factor ? a.class_factor[slot] : 1.0f;
  return pnr_pixel_weight(keep, a.scale, ff, cf);
}
// the weighted pick: the smallest p with S(p) > x, S the inclusive prefix sum of weight [P], through its group sums
// cum [ceil(P / 32)] (cum[g] = S(min(P, 32 (g + 1)) - 1)): an upper-bound search of cum for the group, then a scan of
// its (at most 32) weights.  Tables that disagree with x are clamped: the result always lies in [0, P).
PNR_HD int64_t pnr_weighted_pixel(const uint16_t* weight, const uint64_t* cum, int64_t P, uint64_t x) {
  const int64_t G = (P + PNR_WEIGHT_GROUP - 1) / PNR_WEIGHT_GROUP;
  int64_t lo = 0, hi = G;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (PNR_LDG(cum + mid) <= x) lo = mid + 1; else hi = mid;
  }
  const int64_t g = lo < G ? lo : G - 1;
  uint64_t s = g > 0 ? PNR_LDG(cum + g - 1) : 0;
  const int64_t q0 = g * PNR_WEIGHT_GROUP, q1 = q0 + PNR_WEIGHT_GROUP < P ? q0 + PNR_WEIGHT_GROUP : P;
  for (int64_t q = q0; q < q1; ++q) {
    s += PNR_LDG(weight + q);
    if (s > x) return q;
  }
  return q1 - 1;
}
// the reweighting factor of a drawn pixel of weight w: T / (nonzero w), one double division, rounded to fp32 once
PNR_HD float pnr_importance(uint64_t T, int64_t nonzero, uint16_t w) {
  return (float)PNR_DDIV((double)T, PNR_DMUL((double)nonzero, (double)w));
}

// Row r - a.r0 of every output of pnr_sample_ray_batch for the global ray r (off: a.pix_offset or a copy of it).
// kWeighted: the pixel drawn through the weight table *wt (pnr_sample_ray_batch_weighted; the caller has checked it).
template <bool kWeighted = false>
PNR_HD void pnr_ray_batch_row(const pnr_ray_batch_args& a, const int64_t* off, int64_t r,
                              const pnr_ray_batch_weights* wt = nullptr) {
  const int64_t row = r - a.r0;
  uint32_t w[4];
  pnr_ray_draw(a.seed, a.step, r, 0u, w);
  int64_t p;
  if (kWeighted) {
    p = pnr_weighted_pixel(wt->weight, wt->weight_cum, a.P,
                           pnr_mulhi64(((uint64_t)w[0] << 32) | w[1], wt->weight_total));
    if (wt->importance)
      wt->importance[row] = pnr_importance(wt->weight_total, wt->weight_nonzero, PNR_LDG(wt->weight + p));
  } else {
    p = (int64_t)pnr_mulhi64(((uint64_t)w[0] << 32) | w[1], (uint64_t)a.P);
  }
  const int f = pnr_frame_of(off, a.F, p);
  int cam = a.frame_cam[f];
  cam = cam < 0 ? 0 : (cam >= a.num_cameras ? a.num_cameras - 1 : cam);
  pnr_ray_camera c = a.cams[0];   // selected with constant indices: the table stays in the kernel's parameters
#pragma unroll
  for (int k = 1; k < PNR_RAY_BATCH_MAX_CAMERAS; ++k)
    if (k == cam) c = a.cams[k];
  const int64_t q = p - off[f];
  const int v = (int)(q / c.W), u = (int)(q % c.W);
  float x, y, z;
  if (c.model == 0)
    pnr_pinhole_dir((float)u, (float)v, c.intr[0], c.intr[1], c.intr[2], c.intr[3], &x, &y, &z);
  else
    pnr_fisheye_dir((float)u, (float)v, c.intr[0], c.intr[1], c.intr[2], c.intr[3], c.intr[4], c.intr[5], c.intr[6],
                    &x, &y, &z);
  float m[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) m[i] = a.c2w[(int64_t)f * 12 + i];
  float* o = a.rays + row * 6;
  o[0] = m[3]; o[1] = m[7]; o[2] = m[11];
  pnr_cam_to_world(m, x, y, z, o + 3, o + 4, o + 5);
#pragma unroll
  for (int k = 0; k < 3; ++k) a.rgb[row * 3 + k] = pnr_u8_unit(a.rgb8[p * 3 + k]);
  if (a.depth_out) a.depth_out[row] = a.depth ? a.depth[p] : 0.f;
  if (a.pseudo_label) a.pseudo_label[row] = a.label ? (int32_t)a.label[p] : -1;
  if (a.pixel) a.pixel[row] = p;
  if (a.frame) a.frame[row] = f;
  const int nw = a.N + a.Ni;
  for (int k = 0; k < nw; k += 4) {
    pnr_ray_draw(a.seed, a.step, r, 1u + (uint32_t)(k >> 2), w);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = k + j;
      if (i < a.N) a.u[row * a.N + i] = pnr_u01(w[j]);
      else if (i < nw) a.u_fine[row * a.Ni + (i - a.N)] = pnr_u01(w[j]);
    }
  }
}

// ---------------------------------------------------------------------------------------------- LiDAR depth targets
// pnr_project_depth (include/pnr.h; DESIGN 3.4): a scan's points projected into a frame, the nearest per pixel.  The
// projections are the inverses of pnr_pinhole_dir / pnr_fisheye_dir; depth_kernels in stream_kernels.cu and the host
// build (tests/host_emu.cpp) call the routines below.

PNR_HD uint32_t pnr_float_bits(float x) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(x);
#else
  uint32_t b;
  memcpy(&b, &x, 4);
  return b;
#endif
}
PNR_HD float pnr_bits_float(uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(b);
#else
  float x;
  memcpy(&x, &b, 4);
  return x;
#endif
}
#define PNR_DEPTH_NONE 0x7f800000u   // +Inf: a z-buffer entry no point reached

// Pinhole: camera point (x, y, z) -> (uf, vf), u = (fx x) / z + cx.
PNR_HD void pnr_pinhole_project(float x, float y, float z, float fx, float fy, float cx, float cy, float* u, float* v) {
  *u = PNR_ADD(PNR_DIV(PNR_MUL(fx, x), z), cx);
  *v = PNR_ADD(PNR_DIV(PNR_MUL(fy, y), z), cy);
}
// Fisheye (MEI): camera point -> (uf, vf) and its distance n = |p|; false when x_s.z + xi <= 0 (or NaN).
PNR_HD bool pnr_fisheye_project(float x, float y, float z, float g1, float g2, float u0, float v0, float xi, float k1,
                                float k2, float* u, float* v, float* n_out) {
  const float n = PNR_SQRT(PNR_ADD(PNR_ADD(PNR_MUL(x, x), PNR_MUL(y, y)), PNR_MUL(z, z)));
  *n_out = n;
  const float xs = PNR_DIV(x, n), ys = PNR_DIV(y, n), zs = PNR_DIV(z, n);
  const float den = PNR_ADD(zs, xi);
  if (!(den > 0.f)) return false;
  const float mx = PNR_DIV(xs, den), my = PNR_DIV(ys, den);
  const float r2 = PNR_ADD(PNR_MUL(mx, mx), PNR_MUL(my, my));
  const float d = PNR_ADD(PNR_ADD(1.0f, PNR_MUL(k1, r2)), PNR_MUL(k2, PNR_MUL(r2, r2)));
  *u = PNR_ADD(PNR_MUL(PNR_MUL(g1, mx), d), u0);
  *v = PNR_ADD(PNR_MUL(PNR_MUL(g2, my), d), v0);
  return true;
}
// One point (x, y, z) of a scan through M (row-major 3x4 [R|t], scan -> camera) into camera c: whether it lands, the
// pixel v * W + u within the frame (*pix) and its depth (*t).
PNR_HD bool pnr_project_point(const pnr_ray_camera& c, const float* M, float x, float y, float z, float min_depth,
                              float max_depth, int64_t* pix, float* t_out) {
  float xc, yc, zc;
  pnr_cam_to_world(M, x, y, z, &xc, &yc, &zc);
  xc = PNR_ADD(xc, M[3]);
  yc = PNR_ADD(yc, M[7]);
  zc = PNR_ADD(zc, M[11]);
  float uf, vf, t;
  if (c.model == 0) {
    t = zc;
    if (!(t > min_depth && t <= max_depth)) return false;
    pnr_pinhole_project(xc, yc, zc, c.intr[0], c.intr[1], c.intr[2], c.intr[3], &uf, &vf);
  } else {
    if (!pnr_fisheye_project(xc, yc, zc, c.intr[0], c.intr[1], c.intr[2], c.intr[3], c.intr[4], c.intr[5], c.intr[6],
                             &uf, &vf, &t))
      return false;
    if (!(t > min_depth && t <= max_depth)) return false;
  }
  const float fu = floorf(PNR_ADD(uf, 0.5f)), fv = floorf(PNR_ADD(vf, 0.5f));
  if (!(fu >= 0.f && fu < (float)c.W && fv >= 0.f && fv < (float)c.H)) return false;   // NaN fails too
  *pix = (int64_t)fv * c.W + (int64_t)fu;
  *t_out = t;
  return true;
}
// Frame f of a depth call: its camera (frame_cam clamped into the table) and pixel range [*lo, *hi) (pix_offset
// clamped into [0, P]), so a malformed device table is never read or written outside.
PNR_HD int pnr_depth_frame(const int32_t* frame_cam, const int64_t* off, int num_cameras, int64_t P, int f,
                           int64_t* lo, int64_t* hi) {
  int cam = frame_cam[f];
  cam = cam < 0 ? 0 : (cam >= num_cameras ? num_cameras - 1 : cam);
  int64_t a = off[f], b = off[f + 1];
  a = a < 0 ? 0 : (a > P ? P : a);
  b = b < a ? a : (b > P ? P : b);
  *lo = a;
  *hi = b;
  return cam;
}
// The final depth of pixel q (= v * W + u, q < n) of a frame whose z-buffer (bits, PNR_DEPTH_NONE = none) holds its n
// pixels at z: r = 0 -> the nearest depth or 0; r > 0 -> the occlusion filter: 0 unless d <= fp32(m * fp32(1 + margin))
// with m the smallest depth in the (2r+1)^2 window around (u, v) inside the frame.
PNR_HD float pnr_depth_pixel(const uint32_t* z, int64_t n, int W, int H, int64_t q, int r, float margin) {
  const uint32_t bd = z[q];
  if (bd == PNR_DEPTH_NONE) return 0.f;
  const float d = pnr_bits_float(bd);
  if (r == 0) return d;
  const int v = (int)(q / W), u = (int)(q % W);
  float m = d;
  for (int dv = -r; dv <= r; ++dv) {
    const int vv = v + dv;
    if (vv < 0 || vv >= H) continue;
    for (int du = -r; du <= r; ++du) {
      const int uu = u + du;
      if (uu < 0 || uu >= W) continue;
      const int64_t k = (int64_t)vv * W + uu;
      if (k >= n) continue;
      const float x = pnr_bits_float(z[k]);   // +Inf (none) never wins
      m = x < m ? x : m;
    }
  }
  return d <= PNR_MUL(m, PNR_ADD(1.0f, margin)) ? d : 0.f;
}
