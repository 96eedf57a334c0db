// ray_math.h — per-ray arithmetic with a fully specified fp32 operation order, shared by the CUDA
// kernels (ray_kernels.cu) and a host build used by the CPU tests (tests/host_emu.cpp) to prove the
// order matches the oracle bit for bit without a GPU.
//
// Rules (SURVEY.md 7.3 item 3): every multiply/add/subtract/divide is individually rounded (no FMA
// contraction: __f*_rn intrinsics on device, -ffp-contract=off on host), true division, and min/max
// propagate NaN like torch.minimum/torch.maximum.
#pragma once
#include <stdint.h>
#include <math.h>

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
#define PNR_SQRT(a) __fsqrt_rn((a))
#else
#define PNR_MUL(a, b) ((a) * (b))
#define PNR_ADD(a, b) ((a) + (b))
#define PNR_SUB(a, b) ((a) - (b))
#define PNR_DIV(a, b) ((a) / (b))
#define PNR_DADD(a, b) ((a) + (b))
#define PNR_DSUB(a, b) ((a) - (b))
#define PNR_DMUL(a, b) ((a) * (b))
#define PNR_SQRT(a) sqrtf((a))
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
