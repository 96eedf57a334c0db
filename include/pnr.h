/* pnr.h — C ABI of libpnr (PanopticNeRF render hot path, sm_90a).
 *
 * The reference exposes this path only as a Python plugin surface in lib/networks
 * (make_network, Renderer.render, batchify_rays, raw2outputs, sample_pdf; SURVEY.md 8(b)); it has
 * no native/FFI boundary of its own, and its source is not in the mount (/root/reference holds the
 * landing branch only: README.md:7, README.md:13), so no reference file:line can be cited per entry
 * point.  Each entry point below names the SURVEY.md 8(a) row (a1..a10) it implements; the
 * reference-side binding a maintainer would add is shown in INTEGRATION.md.
 *
 * Conventions
 *  - every function returns 0 on success, <0 on error; pnr_last_error() gives a thread-local text.
 *  - all array arguments are DEVICE pointers unless the name ends in _host.
 *  - buffers are caller-owned; nothing is allocated on the stage entry points; all work is
 *    enqueued asynchronously on `stream` (a cudaStream_t passed as void*).
 *  - a context belongs to one device (cfg.device); every entry point that takes a context makes that
 *    device current for the call and restores the caller's current device before it returns; the
 *    context-free stage entry points run on the caller's current device (the one their pointers and
 *    stream belong to).  Several contexts, devices and streams may be used from one process; a single
 *    context is not thread-safe.  Outputs are deterministic (no atomics on outputs), so any ray
 *    sharding reproduces the single-GPU result bit for bit.
 */
#ifndef PNR_H_
#define PNR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PNR_VERSION 100

enum { PNR_OK = 0, PNR_ERR_ARG = -1, PNR_ERR_CUDA = -2, PNR_ERR_STATE = -3, PNR_ERR_UNSUPPORTED = -4 };

/* MLP arithmetic mode: element format of the tensor-core operands (accumulation is always fp32).
 * The x3 modes split every operand x = hi + lo in that format and issue A_hi*B_hi + A_lo*B_hi + A_hi*B_lo. */
enum { PNR_PREC_BF16X3 = 0, /* operand split to 2^-17 |x|, fp32 exponent range; ~1e-4 end to end (marginal) */
       PNR_PREC_BF16 = 1,   /* 1 pass, 2^-8 |x|; ~1e-2 end to end: fast mode, outside the tolerance         */
       PNR_PREC_FP16X3 = 2, /* operand split to max(2^-23 |x|, 2^-25), needs |activation| < 65504; meets
                               1e-4 with margin at O(1) operands.  The 2^-25 floor (fp16 subnormals) leaves an
                               operand of 1e-4 only ~2^-12 relative, like one fp16 part                    */
       PNR_PREC_FP16 = 3    /* 1 pass, max(2^-11 |x|, 2^-25); ~1e-3 end to end: fast mode, outside the tolerance */ };

typedef struct pnr_ctx pnr_ctx;

typedef struct pnr_config {
  int32_t D;             /* trunk depth (8)                           a8 */
  int32_t W;             /* trunk width (256); 64, 128 or 256         a8 */
  int32_t xyz_res;       /* Lx, positional-encoding octaves for xyz   a7 */
  int32_t view_res;      /* Ld, octaves for the view direction        a7 */
  int32_t num_classes;   /* C semantic logits, 0 = no head            a8 */
  int32_t num_instances; /* K instance logits, 0 = no head            a8 */
  int32_t precision;     /* PNR_PREC_*                                   */
  int32_t device;        /* CUDA ordinal                                 */
  /* Trunk input (8(f) rank 4).  An all-zero tail is the frequency network above.  PNR_XYZ_HASHGRID: the trunk input
   * is h(x), the hash-grid features of the sample point (pnr_hashgrid_encode with these arguments and the table bound
   * by pnr_bind_hashgrid_table), E = hash_levels * hash_features <= 64 columns in place of gamma(x) in layer 0 and in
   * the skip concatenation; xyz_res is ignored.  The view branch keeps gamma(d).  hash_aabb = {lo.xyz, hi.xyz}. */
  int32_t xyz_encoding;  /* PNR_XYZ_*                                    */
  int32_t hash_levels, hash_features, hash_log2_size;
  float hash_base_resolution, hash_per_level_scale;
  float hash_aabb[6];
} pnr_config;
enum { PNR_XYZ_FREQUENCY = 0, PNR_XYZ_HASHGRID = 1 };

int pnr_version(void);
const char* pnr_last_error(void);

/* a1/a2: context = packed weights + kernel attributes for one Network on one device. */
int pnr_create(const pnr_config* cfg, pnr_ctx** out);
int pnr_destroy(pnr_ctx* ctx);

/* a8 range check: sticky status of the fused-MLP launches enqueued so far on `stream` (synchronises it).
 * bit 0 (PNR_STATUS_RANGE): a value written into a 16-bit operand - an embedding (gamma(x), gamma(d), hash-grid
 * features), a trunk activation, a head's hidden activation, a scaled gradient of the backward program - had a hi
 * part that rounds to inf (fp16 modes: |x| >= 65520; 65519 is carried exactly as 65504 + 15) or was NaN, or a
 * hash-grid sample point was not finite.  Outputs of that launch are not trustworthy: a finite overflow, re-run with
 * PNR_PREC_BF16X3.  The ReLU keeps NaN (as torch.relu does), so a NaN input or parameter also reaches the outputs.
 * bit 1: pnr_update_weights packed a weight outside the fp16 range (fp16 modes; see there).
 * reset != 0 clears the word after reading it. */
#define PNR_STATUS_RANGE 1u
int pnr_status(pnr_ctx* ctx, uint32_t* status_host, int32_t reset, void* stream);

/* Hash-grid contexts (cfg.xyz_encoding = PNR_XYZ_HASHGRID): the table [hash_levels, 2^hash_log2_size, hash_features]
 * fp32, a caller-owned DEVICE pointer.  It is not copied: every fused-MLP launch of the context (pnr_mlp_forward,
 * pnr_mlp_composite, pnr_mlp_trunk_forward, pnr_mlp_backward_trunk, pnr_render_fused) reads it when it executes, so an
 * in-place update on the same stream is seen by the next launch.  Those entry points return PNR_ERR_STATE on a
 * hash-grid context without a table; NULL unbinds.  PNR_ERR_STATE on a frequency context.  A table that is not
 * aligned to one corner's features when they are read as a vector (8 bytes at F = 2, 16 at F = 4) is refused
 * (PNR_ERR_ARG), here and by pnr_hashgrid_encode. */
int pnr_bind_hashgrid_table(pnr_ctx* ctx, const float* table);

/* Tile of the fused MLP kernel for this context's raw-row launches (pnr_mlp_forward, and pnr_render_fused on a network
 * without heads): 0 (default) = 128 samples on two consumer warpgroups when the network's program allows it (a
 * 256-wide network without heads, pnr_program_tile_rows), else 64; 64 = always the 64-sample kernel; 128 = the
 * 128-sample kernel, and a launch whose program does not allow it returns PNR_ERR_UNSUPPORTED.  Both kernels give the
 * same bits.  The compositing and backward launches run 64-sample tiles whatever the setting.  PNR_ERR_ARG for any
 * other value. */
int pnr_set_mlp_rows(pnr_ctx* ctx, int32_t rows);

/* Host only: the tile (64 or 128 samples) a raw-row launch of `program` (the MlpProgram struct pnr_program_host
 * returns, program_bytes = its size) runs on when pnr_set_mlp_rows is 0. */
int pnr_program_tile_rows(const void* program, size_t program_bytes, int32_t* rows);

/* a2: load a Network state_dict.  `tensors_host[i]` are HOST fp32 pointers in this fixed order:
 *   pts_linears.{0..D-1}.weight/.bias (interleaved w,b), alpha_linear.w/.b, feature_linear.w/.b,
 *   views_linears.0.w/.b, rgb_linear.w/.b, [semantic_linears.0.w/.b, semantic_linears.1.w/.b],
 *   [instance_linears.0.w/.b, instance_linears.1.w/.b]
 * `shapes[2*i], shapes[2*i+1]` = (out, in) for weights, (out, 1) for biases.  The trunk input width (layer 0's `in`,
 * the skip layer's first columns) is 3 + 6*xyz_res, or E = hash_levels * hash_features for a hash-grid context (whose
 * table is not in this list: pnr_bind_hashgrid_table).  The forward program's packing plan (built from cfg and the
 * shapes) is applied to the weights on the host: they are split into 16-bit hi/lo parts of the context's operand
 * format (fp16 or bf16, cfg.precision), laid out as the no-swizzle K-major wgmma stage images of the packed weight
 * stream (csrc/mlp_program.h) and uploaded, together with the weights themselves, from which the programs built later
 * and pnr_update_weights pack on the device.  In the fp16 modes a packed weight with |w| > 65504 (after the
 * feature_linear fold) or not finite is rejected (PNR_ERR_UNSUPPORTED): use a bf16 mode.  The bf16 modes accept a
 * NaN weight, and no mode checks the fp32 biases: a NaN there propagates to the outputs and sets bit 0 of pnr_status
 * where it enters an operand. */
int pnr_load_weights(pnr_ctx* ctx, const float* const* tensors_host, const int64_t* shapes, int32_t n);

/* a5: ray / oriented-box slab test.  rays [R,6] (o||d); box_center, box_half [B,3]; box_rot [B,3,3]
 * row-major, columns = box axes.  Out: hit_mask [R] u8, box_id [R,M] i32 (-1 pad), t_in/t_out [R,M]. */
int pnr_intersect(const float* rays, int64_t R, const float* box_center, const float* box_half,
                  const float* box_rot, int32_t B, int32_t M, uint8_t* hit_mask, int32_t* box_id,
                  float* t_in, float* t_out, void* stream);

/* a5 with mesh primitives (DESIGN 3.2).  mesh_tri_start [B+1] i32, non-decreasing, [0] = 0, [B] = T; mesh_tris
 * [T,3,3] world-space vertices; primitive b owns the triangles [start[b], start[b+1]).  A primitive with an empty
 * range is a cuboid (the slab test of pnr_intersect).  One with triangles is a closed mesh whose box is a cull volume
 * containing all its vertices: a ray that misses the box misses the mesh, and the box's own interval is never
 * reported; the mesh's inside intervals (watertight crossings, paired along the line) enter the M-nearest list, so
 * one primitive may take several slots.  Ranges are clamped into [0, T].  Both mesh pointers NULL with T = 0 is
 * pnr_intersect; otherwise both are set and 1 <= T < 2^31 (PNR_ERR_ARG before any launch). */
int pnr_intersect_meshes(const float* rays, int64_t R, const float* box_center, const float* box_half,
                         const float* box_rot, const int32_t* mesh_tri_start, const float* mesh_tris, int64_t T,
                         int32_t B, int32_t M, uint8_t* hit_mask, int32_t* box_id, float* t_in, float* t_out,
                         void* stream);

/* a5 with a sequence table (DESIGN 3.2): one primitive table for the rays of many frames.  Primitives [0, S) are
 * static; frame f owns the dynamic block frame_boxes [F,2] i32 row f = (begin, end), S <= begin <= end <= B (blocks may
 * be shared, e.g. by the cameras of one timestamp).  Ray r is intersected with [0, S) and then with the block of its
 * frame ray_frame [R] i32, in that order, so its outputs equal, bit for bit, those of pnr_intersect_meshes on the table
 * cat(static, block) with the block's ids shifted by begin - S.  Box ids index the whole table (box_sem, box_inst and
 * mesh_tri_start index it unchanged).  A block entry is clamped into [S, B] (end < begin: empty); a ray_frame outside
 * [0, F) meets the static primitives only.  F = 0 is no frame table: ray_frame and frame_boxes NULL and S = 0, every
 * primitive static (the bytes of pnr_intersect_meshes).  Refused before any launch (PNR_ERR_ARG, by name): F < 0, a
 * null ray_frame or frame_boxes with F >= 1, either set or S != 0 with F = 0, S outside [0, B]; and whatever
 * pnr_intersect_meshes refuses. */
typedef struct pnr_frame_table {
  const int32_t* ray_frame;     /* [R] frame of each ray                                                          */
  const int32_t* frame_boxes;   /* [F,2] (begin, end) of each frame's dynamic block                               */
  int32_t F, S;                 /* frames, static primitives                                                      */
} pnr_frame_table;
typedef struct pnr_intersect_frames_args {
  const float* rays;            /* [R,6]                                                                          */
  int64_t R;
  const float* box_center;      /* [B,3] the sequence table                                                       */
  const float* box_half;        /* [B,3]                                                                          */
  const float* box_rot;         /* [B,3,3]                                                                        */
  int32_t B, M;
  const int32_t* mesh_tri_start;  /* [B+1] or NULL with T = 0, as pnr_intersect_meshes                            */
  const float* mesh_tris;       /* [T,3,3]                                                                        */
  int64_t T;
  pnr_frame_table frames;
  uint8_t* hit_mask;            /* [R]                                                                            */
  int32_t* box_id;              /* [R,M]                                                                          */
  float* t_in;                  /* [R,M]                                                                          */
  float* t_out;                 /* [R,M]                                                                          */
} pnr_intersect_frames_args;
int pnr_intersect_frames(const pnr_intersect_frames_args* args, void* stream);

/* a5 (AABB special case): per-ray near = max(tmin, near_min), far = tmax, or
 * (near_min, far_default) when the scene box is missed.  aabb_host = {lo.xyz, hi.xyz}. */
int pnr_scene_near_far(const float* rays, int64_t R, const float* aabb_host, float near_min,
                       float far_default, float* near, float* far, void* stream);

/* a5 helper (cfg.bound_by_primitives): clamp near/far to the hull of the hit intervals, in place. */
int pnr_bound_by_primitives(const uint8_t* hit_mask, const int32_t* box_id, const float* t_in,
                            const float* t_out, int64_t R, int32_t M, float* near, float* far,
                            void* stream);

/* a6: z[R,N] = near*(1-t)+far*t (t_vals [N]); if perturb>0, jittered with u [R,N].
 * sample_box (nullable) [R,N] i32 = id of the first hit interval containing the sample, else -1. */
int pnr_sample_stratified(const float* near, const float* far, const float* t_vals, const float* u,
                          int64_t R, int32_t N, float perturb, const int32_t* box_id,
                          const float* t_in, const float* t_out, int32_t M, float* z,
                          int32_t* sample_box, void* stream);

/* a6, interval mode: the N samples are placed inside the ray's hit intervals (clipped to [near, far]):
 * n_m = floor(N * len_m / sum len) samples for interval m, the remainder one by one to the nearest intervals,
 * sample j of an interval at a + (b-a)*(j+0.5)/n_m (or (j+u)/n_m when perturb > 0, u [R,N] per allocation slot),
 * the depths sorted ascending; rays without a hit interval fall back to the uniform rule of pnr_sample_stratified.
 * Same arguments as pnr_sample_stratified (box_id/t_in/t_out required).  The reference's own allocation rule is
 * not in the mount (SURVEY 8(c) question 4): this one is chosen here and documented in DESIGN.md. */
int pnr_sample_intervals(const float* near, const float* far, const float* t_vals, const float* u,
                         int64_t R, int32_t N, float perturb, const int32_t* box_id,
                         const float* t_in, const float* t_out, int32_t M, float* z,
                         int32_t* sample_box, void* stream);

/* a6: re-tag an existing depth array (after the coarse+fine merge). */
int pnr_tag_samples(const float* z, int64_t R, int32_t N, const int32_t* box_id, const float* t_in,
                    const float* t_out, int32_t M, int32_t* sample_box, void* stream);

/* 8(f) rank 3 (the step before the path): camera rays for image rows [row0, row0+rows) of an H x W image,
 * rays [rows*W, 6] = origin || unnormalised direction, row-major over (v, u).
 * camera 0 = pinhole: d_cam = ((u-cx)/fx, (v-cy)/fy, 1); camera 1 = equirectangular:
 * lon = (u/W-0.5)*2pi, lat = (0.5-v/H)*pi, d_cam = (cos lat sin lon, -sin lat, cos lat cos lon).
 * camera 2 = KITTI-360 fisheye (unified / MEI model), intr_host = {gamma1, gamma2, u0, v0, xi, k1, k2}: the pixel's
 * distorted normalised point is undistorted radially (rd = ro (1 + k1 ro^2 + k2 ro^4), 8 Newton steps from ro = rd)
 * and lifted to the unit sphere, d_cam = (f x, f y, f - xi), f = (xi + sqrt(1 + (1 - xi^2) r^2)) / (1 + r^2).
 * intr_host = {fx, fy, cx, cy} otherwise; c2w_host = row-major 3x4 [R|t]: d = R d_cam, o = t. */
int pnr_generate_rays(int32_t H, int32_t W, int32_t row0, int32_t rows, int32_t camera, const float* intr_host,
                      const float* c2w_host, float* rays, void* stream);

/* A training batch of random pixels from a set of frames kept on the device (DESIGN 3.4): per ray the camera ray,
 * its targets and its sampling jitter.
 * Frame set (caller-owned, device): c2w [F, 12] (row-major 3x4 [R|t] as pnr_generate_rays), frame_cam [F] i32 (an
 * entry of cams), pix_offset [F+1] i64: frame f owns the flat pixels [off[f], off[f+1]), row-major over (v, u) of its
 * camera's W, off[0] = 0, off[F] = P (a malformed table is clamped, never read outside); per pixel rgb8 [P, 3] u8 and
 * optionally label [P] i16 (-1 = ignore) and depth [P] f32 (<= 0 = none).  cams[0 .. num_cameras): model 0 pinhole
 * (intr = fx, fy, cx, cy) or 2 fisheye (gamma1, gamma2, u0, v0, xi, k1, k2); the equirect model (1) is refused, its
 * rays are device-only.
 * Draws: Philox4x32-10 with key = seed (low word first) and counter (block, r, step low word, step high word) for the
 * global ray index r.  Block 0: the pixel p = mulhi64(w0 << 32 | w1, P) (the high 64 bits of the 128-bit product), the
 * frame f by an upper-bound search of pix_offset, (v, u) = divmod(p - off[f], W).  Blocks 1, 2, ...: jitter word k
 * (k = 0 .. N+Ni) is word k % 4 of block 1 + k / 4, as (w >> 8) * 2^-24; u[r, j] = word j, u_fine[r, j] = word N + j.
 * Every output row is a function of (seed, step, r) alone: the launch writes the rays r0 .. r1-1 into rows
 * 0 .. r1-r0-1, equal bit for bit to the matching rows of [0, R).
 * Outputs [r1 - r0, ...]: rays [., 6] (row v*W + u of pnr_generate_rays for that frame, bit for bit), rgb [., 3] =
 * byte / 255 (true division), u [., N], u_fine [., Ni] (needed when Ni > 0); nullable: depth_out [.] (0 without a depth
 * table), pseudo_label [.] i32 (-1 without a label table), pixel [.] i64 (the flat index p), frame [.] i32 (f).
 * Refused before any launch (PNR_ERR_ARG, by name): F < 1 or >= 2^31 - 1, P < 1, r0 < 0, r1 < r0, r1 > 2^32, N outside
 * [1, 256], Ni < 0 or N + Ni > 256, num_cameras outside [1, PNR_RAY_BATCH_MAX_CAMERAS], a camera model other than 0 / 2
 * or H, W < 1, a null frame-set or required output pointer. */
#define PNR_RAY_BATCH_MAX_CAMERAS 4
typedef struct pnr_ray_camera {
  int32_t model, H, W;
  float intr[7];
} pnr_ray_camera;
typedef struct pnr_ray_batch_args {
  const float* c2w;
  const int32_t* frame_cam;
  const int64_t* pix_offset;
  int32_t F;
  int64_t P;
  const uint8_t* rgb8;
  const int16_t* label;
  const float* depth;
  pnr_ray_camera cams[PNR_RAY_BATCH_MAX_CAMERAS];
  int32_t num_cameras;
  uint64_t seed, step;
  int64_t r0, r1;
  int32_t N, Ni;
  float* rays;
  float* rgb;
  float* depth_out;
  int32_t* pseudo_label;
  float* u;
  float* u_fine;
  int64_t* pixel;
  int32_t* frame;               /* [.] i32 the frame f of the pixel, nullable (the index pnr_frame_table's
                                   ray_frame takes when the frames map one to one onto frame_boxes)          */
} pnr_ray_batch_args;
int pnr_sample_ray_batch(const pnr_ray_batch_args* args, void* stream);

/* Weighted draws (DESIGN 3.4): pnr_sample_ray_batch with the pixel drawn through a per-pixel weight table weight [P]
 * u16 (pnr_pixel_weights) and its group sums weight_cum [ceil(P/32)] u64 (pnr_pixel_cdf), with T = weight_total and
 * weight_nonzero (the count of non-zero weights) passed by value.  Block 0 gives x = mulhi64(w0 << 32 | w1, T) and the
 * pixel is the smallest p with S(p) > x, S(p) = sum_{q <= p} weight[q]: an upper-bound search of weight_cum for the
 * group of 32 pixels, then a scan of its weights.  A pixel of weight 0 is never drawn, and a table of all ones draws
 * p = x, the unweighted pixel, so every output equals pnr_sample_ray_batch's bit for bit.  The frame, ray, targets and
 * jitter follow from p as there.  importance [r1 - r0] f32 (nullable) = fp32(T / (weight_nonzero weight[p])) in
 * double, one division rounded once: its mean under the draw is 1.
 * Refused before any launch (PNR_ERR_ARG, by name): everything pnr_sample_ray_batch refuses; a null w, weight or
 * weight_cum, weight_total = 0, weight_nonzero outside [1, P], weight_total outside [weight_nonzero,
 * 65535 weight_nonzero]. */
typedef struct pnr_ray_batch_weights {
  const uint16_t* weight;       /* [P] u16 device                                                                */
  const uint64_t* weight_cum;   /* [ceil(P/32)] u64 device (pnr_pixel_cdf's cum)                                 */
  uint64_t weight_total;        /* T = the sum of the weights (pnr_pixel_cdf's totals[0])                        */
  int64_t weight_nonzero;       /* the count of non-zero weights (totals[1])                                     */
  float* importance;            /* [r1 - r0] f32 device, nullable: T / (weight_nonzero weight[p])                */
} pnr_ray_batch_weights;
int pnr_sample_ray_batch_weighted(const pnr_ray_batch_args* args, const pnr_ray_batch_weights* w, void* stream);

/* Per-pixel weights of a frame set for weighted draws (DESIGN 3.4).  Rule (chosen here), per pixel q of frame f,
 * slot = 1 + label for a label in [0, C), else 0 (-1 and any other value; every pixel without a label table):
 *   x = (scale * frame_factor[f]) * class_factor[slot] in fp32, each product rounded, no FMA (a NULL table reads 1);
 *   weight = 0 when the camera's mask is 0 at q, when x is NaN or x <= 0; 65535 when x >= 65535 (+Inf included);
 *   otherwise x rounded to the nearest integer, ties to even (0.5 -> 0, 1.5 -> 2, 65534.5 -> 65534).
 * Inputs: the frame table as pnr_ray_batch_args (frame_cam [F], pix_offset [F+1], P, cams; a malformed device table is
 * clamped, never read or written outside, and a frame's pixels past its camera's H W are given weight 0), label [P]
 * i16 (nullable), frame_factor [F] f32 and class_factor [C+1] f32 (nullable), mask[k] [H_k W_k] u8 of camera k
 * (nullable; non-zero = keep), all on the device.  Output weight [P] u16: the pixels of the frames of the table are
 * written, every other byte is left as it is.  No host copy or synchronisation: the call can be captured.
 * Refused before any launch (PNR_ERR_ARG, by name): F < 1 or >= 2^31 - 1, P < 1, C outside [0, 32767], num_cameras
 * outside [1, PNR_RAY_BATCH_MAX_CAMERAS], a camera model other than 0 / 2 or H, W outside [1, 2^31), a null
 * frame_cam, pix_offset or weight, scale not finite and > 0. */
typedef struct pnr_pixel_weights_args {
  const int32_t* frame_cam;     /* [F] device                                                                    */
  const int64_t* pix_offset;    /* [F+1] device                                                                  */
  int32_t F;
  int64_t P;
  pnr_ray_camera cams[PNR_RAY_BATCH_MAX_CAMERAS];
  int32_t num_cameras;
  const int16_t* label;         /* [P] device, nullable                                                          */
  int32_t C;                    /* classes: class_factor has C + 1 entries (slot 0 = outside [0, C))             */
  const float* frame_factor;    /* [F] device, nullable = 1                                                      */
  const float* class_factor;    /* [C+1] device, nullable = 1                                                    */
  const uint8_t* mask[PNR_RAY_BATCH_MAX_CAMERAS];   /* [H*W] device per camera, nullable = keep every pixel     */
  float scale;
  uint16_t* weight;             /* [P] device                                                                    */
} pnr_pixel_weights_args;
int pnr_pixel_weights(const pnr_pixel_weights_args* args, void* stream);

/* Class histogram of a label table: counts [C+1] u64 (device), slot 0 = labels outside [0, C) (-1 included), slot
 * 1 + c = class c.  Integer sums: exact and independent of the order of the pixels.  counts is overwritten (zeroed
 * on the stream first).  Refused (PNR_ERR_ARG, by name): P < 1, C outside [0, 8191], a null label or counts. */
int pnr_label_counts(const int16_t* label, int64_t P, int32_t C, uint64_t* counts, void* stream);

/* Exact prefix sum of a weight table in groups of 32 pixels: cum[g] = sum_{q < min(P, 32 (g+1))} weight[q] u64, for
 * g < ceil(P/32), and totals[2] u64 = {T = the sum of all weights, the count of non-zero weights}, all on the device.
 * Integer addition: every schedule gives the same bits.  Reduce-then-scan: per tile of 2^15 pixels its sum, one
 * block's scan of the tile sums, then per tile the group sums scanned on top of its prefix (the weights are read
 * twice).  No host copy or synchronisation: the call can be captured.  workspace: pnr_pixel_cdf_workspace_bytes(P)
 * bytes of device scratch, 16-byte aligned (two u64 per tile); 0 for P outside [1, 2^47).
 * Refused (PNR_ERR_ARG, by name): P outside [1, 2^47), a null or misaligned (16 bytes) weight, a null cum or totals,
 * a short or misaligned workspace. */
size_t pnr_pixel_cdf_workspace_bytes(int64_t P);
int pnr_pixel_cdf(const uint16_t* weight, int64_t P, uint64_t* cum, uint64_t* totals, void* workspace,
                  size_t workspace_bytes, void* stream);

/* Depth targets from LiDAR scans (DESIGN 3.4): the points of scan s, projected into frame f of a frame set, leave per
 * pixel the nearest depth, written into that set's depth table.  Rules (chosen here: the reference's preprocessing
 * is not public):
 *   1. Transform.  pair_M[k] is the row-major 3x4 [R|t] from the scan's Velodyne frame to the camera of frame
 *      pair_frame[k], composed by the caller in float64 and rounded once (kitti360/lidar.py:
 *      inv(cam_to_world_f) @ poses[s] @ cam_to_pose[image_00] @ inv(cam_to_velo)).  p_c = R p + t in fp32 without
 *      FMA: ((R0 x + R1 y) + R2 z) + t0, each operation rounded, as the rotation of pnr_generate_rays.
 *   2. Projection, the inverse of the rays of pnr_generate_rays.  Pinhole (model 0): u = (fx x) / z + cx,
 *      v = (fy y) / z + cy.  Fisheye (model 2, MEI): n = sqrt((x x + y y) + z z), x_s = p_c / n (three divisions),
 *      m = (x_s.x, x_s.y) / (x_s.z + xi), r2 = m.x m.x + m.y m.y, d = (1 + k1 r2) + k2 (r2 r2),
 *      u = ((gamma1 m.x) d) + u0, v likewise; no p1 / p2 terms (the rays have none); a point with
 *      x_s.z + xi <= 0 (or NaN) is not projected.  The equirect model (1) is refused.
 *   3. Pixel: u = floor(fp32(uf + 0.5)), v likewise, kept when 0 <= u < W and 0 <= v < H (a pixel's ray goes through
 *      its integer coordinates).
 *   4. Depth: the ray parameter t of the camera's ray direction, t = z for the pinhole (direction (x, y, 1)) and t = n
 *      for the fisheye (unit directions); a point counts when min_depth < t <= max_depth (NaN never counts).
 *   5. Nearest wins: per pixel the smallest t, by an integer atomicMin on the bits of the positive floats over a buffer
 *      set to +Inf, then +Inf -> 0 (no depth).  The result does not depend on the order of the points, the pairs or
 *      the launches.
 *   6. Occlusion filter (occlusion_radius r > 0): a pixel's depth d is kept iff d <= fp32(m * fp32(1 + margin)), m the
 *      smallest non-zero depth in the (2r+1)^2 window around it inside the same frame (clipped at its borders), else
 *      0.  It reads the whole z-buffer of the frame and writes depth, so it does not depend on thread order.
 * Inputs: points [Npts, 4] f32 device (x, y, z, reflectance; reflectance unread; 16-byte aligned); scan_offset [S+1]
 * i64 HOST: scan s is points [scan_offset[s], scan_offset[s+1]).  Pairs, HOST: pair_frame [Q] i32, pair_scan [Q] i32,
 * pair_M [Q, 12] f32.  Frame set (device, as pnr_ray_batch_args: frame_cam [F], pix_offset [F+1], P pixels; a malformed
 * device table is clamped, never read or written outside) and cams[0 .. num_cameras) by value.  Output depth [P] f32
 * device: only the pixels of the frames named by some pair are rewritten (every pixel of such a frame: 0 where no point
 * lands), every other byte is left as it is.  The host tables are read during the call; the device work is a fixed
 * sequence of launches on `stream`, with the tables in the kernels' parameters, so the call can be captured in a CUDA
 * graph.
 * workspace: pnr_project_depth_workspace_bytes(P, occlusion_radius) bytes of device scratch, 16-byte aligned (the
 * filter's z-buffer, P u32; 0 bytes and NULL without the filter).
 * Refused before any launch (PNR_ERR_ARG, by name): F < 1 or >= 2^31 - 1, P < 1, Q < 0, S < 0, Npts < 0, a pair_frame
 * outside [0, F) or pair_scan outside [0, S), a scan_offset that is negative, decreasing or past Npts, num_cameras
 * outside [1, PNR_RAY_BATCH_MAX_CAMERAS], a camera model other than 0 / 2 or H, W outside [1, 2^24), min_depth not
 * finite and > 0, max_depth not finite or <= min_depth, occlusion_radius outside [0, 8], occlusion_margin outside
 * (0, 1) when the filter is on, a null required pointer, a misaligned points pointer, a short or misaligned
 * workspace. */
typedef struct pnr_project_depth_args {
  const float* points;          /* [Npts, 4] device                                                             */
  int64_t Npts;
  const int64_t* scan_offset;   /* [S+1] host                                                                   */
  int32_t S;
  const int32_t* pair_frame;    /* [Q] host                                                                     */
  const int32_t* pair_scan;     /* [Q] host                                                                     */
  const float* pair_M;          /* [Q, 12] host                                                                 */
  int32_t Q;
  const int32_t* frame_cam;     /* [F] device                                                                   */
  const int64_t* pix_offset;    /* [F+1] device                                                                 */
  int32_t F;
  int64_t P;
  pnr_ray_camera cams[PNR_RAY_BATCH_MAX_CAMERAS];
  int32_t num_cameras;
  float min_depth, max_depth;
  int32_t occlusion_radius;     /* 0 = no filter                                                                */
  float occlusion_margin;
  float* depth;                 /* [P] device                                                                   */
  void* workspace;
  size_t workspace_bytes;
} pnr_project_depth_args;
size_t pnr_project_depth_workspace_bytes(int64_t P, int32_t occlusion_radius);
int pnr_project_depth(const pnr_project_depth_args* args, void* stream);

/* Depth targets from a rectified stereo pair by semi-global matching (DESIGN 3.4).  Rules (chosen here: the
 * reference's stereo preprocessing is not public), per pair of H x W RGB8 images (left = the frame's pixels in the
 * frame store, right = right[i]), D disparities; all integer until step 7:
 *   1. Grey: g = (4899 R + 9617 G + 1868 B + 8192) >> 14.
 *   2. Census: a 9 x 7 window (9 wide, 7 high) in raster order, centre excluded, 62 bits; bit k = g(q_k) < g(p);
 *      coordinates outside the image clamped to the nearest edge pixel.
 *   3. Cost: C(x, y, d) = popcount(census_L(x, y) ^ census_R(x - d, y)) for x - d >= 0, else 63; d in [0, D).
 *   4. Aggregation over the 8 directions r in {(+-1, 0), (0, +-1), (+-1, +-1)}:
 *      L_r(p, d) = C(p, d) + min(L_r(p-r, d), L_r(p-r, d-1) + P1, L_r(p-r, d+1) + P1, m_r(p-r) + P2) - m_r(p-r),
 *      m_r = min_k L_r(., k), out-of-range d +- 1 terms absent, L_r = C where p - r is outside the image.
 *      L_r <= 63 + P2, so S(p, d) = sum_r L_r(p, d) <= 8 (63 + 2048) fits in u16.
 *   5. Winner d* = argmin_d S, lowest d on ties.  Invalid if some d with |d - d*| > 1 has S(d) (100 - U) <
 *      S(d*) 100 (uniqueness), or unless x - d* >= 0 and |d* - d_R(x - d*)| <= 1 (left-right check), with
 *      d_R(x') = argmin_d S(x' + d, y, d) over x' + d < W, lowest d on ties.
 *   6. Subpixel, in sixteenths: for 0 < d* < D - 1, den = max(S(d*-1) + S(d*+1) - 2 S(d*), 1),
 *      d16 = 16 d* + ((S(d*-1) - S(d*+1)) 16 + den) / (2 den) with C's division (toward zero); else d16 = 16 d*;
 *      an invalid pixel has d16 = -1.
 *   7. Depth t = B16 / fp32(d16), one IEEE fp32 division (B16 = fp32(16 (P_rect_00[0,3] - P_rect_01[0,3])) = 16 fx b,
 *      composed in float64 by the caller), kept when d16 > 0 and min_depth < t <= max_depth, else 0 (no target).
 *      t is z in rectified camera 0, the units of the pinhole's rays.
 * Inputs: the frame store rgb8 [P, 3] u8 and pix_offset [F+1] i64 (device), the host table frames [n] of the call's
 * frames (each of H x W pixels), right [n, H, W, 3] u8 (device).  Outputs (at least one): depth [P] f32 (the store's;
 * only the pixels of the named frames are rewritten) and disparity [n, H, W] i16 (d16).  A frame whose device
 * pix_offset range is not H W pixels inside [0, P] is not read and not written (its disparity is -1).  The call is a
 * fixed sequence of launches on `stream` with the frame table in the kernels' parameters: no host copy, allocation
 * or synchronisation, so it can be captured in a CUDA graph.
 * workspace: pnr_stereo_workspace_bytes(n, H, W, D) bytes of device scratch, 16-byte aligned, laid out as four
 * sections, each starting on a 16-byte boundary (N = n H W): census_L [N] u64, census_R [N] u64, S [N, D] u16,
 * d_R [N] i16.  0 for arguments outside the accepted ranges.
 * Refused before any launch (PNR_ERR_ARG, by name): n < 1, H or W outside [1, 65535], D not in {32, 64, .., 256},
 * P1 / P2 outside 0 <= P1 <= P2 <= 2048, U outside [0, 99], F < 1, P < 1, a frames[i] outside [0, F), a null rgb8,
 * pix_offset, right or frames, both outputs null, with depth: B16 not finite and > 0, min_depth not finite and > 0,
 * max_depth not finite and > min_depth; a short or misaligned workspace. */
typedef struct pnr_stereo_args {
  const uint8_t* rgb8;          /* [P, 3] device: the frame store's colours                                    */
  const int64_t* pix_offset;    /* [F+1] device                                                                */
  int64_t P;
  int32_t F;
  const int32_t* frames;        /* [n] host: the store's frame of each pair                                    */
  int32_t n, H, W;
  const uint8_t* right;         /* [n, H, W, 3] device                                                         */
  int32_t D, P1, P2, U;
  float B16, min_depth, max_depth;
  float* depth;                 /* [P] device, nullable                                                        */
  int16_t* disparity;           /* [n, H, W] device, nullable                                                  */
  void* workspace;
  size_t workspace_bytes;
} pnr_stereo_args;
size_t pnr_stereo_workspace_bytes(int32_t n, int32_t H, int32_t W, int32_t D);
int pnr_stereo_depth(const pnr_stereo_args* args, void* stream);

/* a7: standalone positional encoding, out [n, 3+6L]. */
int pnr_encode(const float* x, int64_t n, int32_t L, float* out, void* stream);

/* a8: Network.forward.  Either (pts, viewdirs) [n,3] each, or (rays [R,6], z [R,N]) with pts and the
 * normalised view direction formed in-kernel (pass pts = NULL).  raw [n or R*N, 4+C+K]. */
int pnr_mlp_forward(pnr_ctx* ctx, const float* pts, const float* viewdirs, const float* rays,
                    const float* z, int64_t R, int32_t N, float* raw, void* stream);

/* a9: raw2outputs.  raw [R,N,4+C+K], z [R,N], rays [R,6].  Any output pointer may be NULL.
 * sem_softmax: composite softmax(logits) instead of logits.  sample_box/box_sem/box_inst nullable. */
typedef struct pnr_composite_out {
  float* rgb_map;    /* [R,3] */
  float* depth_map;  /* [R]   */
  float* acc_map;    /* [R]   */
  float* disp_map;   /* [R]   */
  float* weights;    /* [R,N] */
  float* semantic_map;        /* [R,C] */
  float* instance_map;        /* [R,K] */
  float* fixed_semantic_map;  /* [R,C] */
  float* fixed_instance_map;  /* [R,K] */
} pnr_composite_out;
int pnr_composite(const float* raw, const float* z, const float* rays, int64_t R, int32_t N,
                  int32_t C, int32_t K, int32_t white_bkgd, int32_t sem_softmax, int32_t mask_outside,
                  const int32_t* sample_box, const int32_t* box_sem, const int32_t* box_inst,
                  int32_t B, const pnr_composite_out* out, void* stream);

/* 8(e) label tiles / 8(f) rank 4 (panoptic label fusion): what a rank contributes to the all-gather when labels,
 * not logits, are wanted - rgb8 [R,3] u8 = round(255*clamp(rgb)), depth_out [R] f32, sem_label / inst_label [R] i16 =
 * argmax of the composited semantic / instance maps (ties -> lowest index, NaN counts as -inf).
 * 13 bytes per ray instead of 4*(5+C+K).  Any output pointer may be NULL. */
int pnr_label_tiles(const float* rgb_map, const float* depth_map, const float* semantic_map,
                    const float* instance_map, int64_t R, int32_t C, int32_t K, uint8_t* rgb8,
                    float* depth_out, int16_t* sem_label, int16_t* inst_label, void* stream);

/* 8(f) rank 2, the loss side: the per-ray terms of the training objective on the rendered maps and their gradients
 * w.r.t. those maps, in one pass (inputs any subset; NULL skips a term / an output):
 *   photometric  sum_c (rgb_map - rgb_gt)^2  (+ the same for the coarse map rgb_map0)
 *   depth        |depth_map - depth_gt| where depth_gt > 0
 *   semantic     label >= 0: cross-entropy of semantic_map [R,C] against label - softmax CE when the map holds rendered
 *                logits (sem_is_prob = 0), -log(max(p_label, eps)) when it holds rendered probabilities - times
 *                label_weight[r] (optional confidence)
 *   fixed        -log(max(fixed_semantic_map[label], eps)) * label_weight
 *                (the gradient of max(p, eps) passes at p == eps, as torch.clamp_min's does)
 * per_ray [R,4] receives the four unweighted values; the caller sums them.  Every gradient is already multiplied by
 * the term's weight w_* and normaliser inv_n_* (1 / number of elements or valid rays, which the caller knows), i.e.
 * it is dL/dmap of L = w_rgb*mean_rgb + w_depth*mean_depth + w_sem*mean_sem + w_fix*mean_fix, ready for
 * pnr_composite_backward.  (Terms as in the paper; the reference's NetworkWrapper is not in the mount.)
 *
 * Instance term (on when instance_map != NULL; the fields after d_fixed_semantic_map, zero = off): the target of ray r
 * is the lowest slot k whose fixed_instance_map[r,k] [R,K] equals the row maximum; the ray counts when that maximum is
 * >= inst_min_weight (in (0,1]; a NaN maximum or a ray without primitives does not count).  inst_label [R] receives k
 * or -1 and n_inst (one device int) the number of counted rays, both written by a label pass before the loss pass, so
 * no host synchronisation is needed.  per_ray_inst [R] (nullable) = lse(instance_map[r]) - instance_map[r,k] (0 when
 * not counted); d_instance_map [R,K] (nullable) = (softmax - onehot(k)) * w_inst / n_inst, i.e. the gradient of
 * w_inst * (mean over counted rays).  No gradient flows into fixed_instance_map (the target is piecewise constant). */
typedef struct pnr_loss_args {
  int64_t R; int32_t C; int32_t sem_is_prob;
  const float* rgb_map; const float* rgb_map0; const float* rgb_gt;
  const float* depth_map; const float* depth_gt;
  const float* semantic_map; const float* fixed_semantic_map; const int32_t* label; const float* label_weight;
  float w_rgb, w_depth, w_sem, w_fix;
  float inv_n_rgb, inv_n_depth, inv_n_sem;
  float eps;
  float* per_ray;
  float* d_rgb_map; float* d_rgb_map0; float* d_depth_map; float* d_semantic_map; float* d_fixed_semantic_map;
  int32_t K;
  const float* instance_map; const float* fixed_instance_map;
  float w_inst;
  float inst_min_weight;
  float* per_ray_inst;
  int32_t* inst_label;
  int32_t* n_inst;
  float* d_instance_map;
} pnr_loss_args;
int pnr_losses(const pnr_loss_args* args, void* stream);

/* 8(f) rank 4: panoptic label fusion + colour mapping of the composited maps (the step after the path).
 * s = argmax semantic_map [R,C] (ties -> lowest index, NaN = -inf).  A stuff class (is_thing[s] == 0, or no instance
 * map) gives id(s)*1000 with id(s) = class_id[s] (or s when class_id is NULL).  A thing class takes the best instance
 * slot among the slots k with inst_class[k] == s: panoptic = inst_id[k] (or id(s)*1000 + k + 1 when inst_id is NULL);
 * without such a slot it falls back to id(s)*1000.  color [R,3] u8: palette[s], for instances averaged with a colour
 * hashed from the panoptic id.  Outputs are optional.  (Rule chosen here; the reference's is not in the mount.) */
int pnr_panoptic_fuse(const float* semantic_map, const float* instance_map, int64_t R, int32_t C, int32_t K,
                      const uint8_t* is_thing, const int32_t* inst_class, const int32_t* inst_id,
                      const int32_t* class_id, const uint8_t* palette, int32_t* panoptic, int16_t* sem_label,
                      int16_t* inst_slot, uint8_t* color, void* stream);

/* 8(f) rank 4: multi-resolution hash-grid features (the 360 model's extra encoder; published algorithm of
 * Mueller et al. 2022): level l has resolution floor(base_resolution * per_level_scale^l) (double, on the host);
 * x [n,3] is mapped to [0,1]^3 by aabb (DEVICE {lo.xyz, hi.xyz}; NULL: already normalised) and clamped; the 8 corners
 * of its cell are read from table [L, 2^T_log2, F] fp32 - dense index x + y*(res+1) + z*(res+1)^2 while the level fits,
 * else (x*1) ^ (y*2654435761) ^ (z*805459861) mod 2^T_log2 - and blended trilinearly (corner order x fastest).
 * out [n, L*F], level-major.  F in {1,2,4,8}. */
int pnr_hashgrid_encode(const float* x, int64_t n, const float* aabb, const float* table, int32_t L, int32_t F,
                        int32_t T_log2, float base_resolution, float per_level_scale, float* out, void* stream);

/* Gradient of pnr_hashgrid_encode w.r.t. its table: grad_table [L, 2^T_log2, F] += scatter of grad_out [n, L*F] with the
 * forward's corner weights (fp32 atomic adds: ACCUMULATES - zero grad_table first; the summation order, hence the last
 * bits, vary between runs).  Same arguments as the forward. */
int pnr_hashgrid_backward(const float* x, int64_t n, const float* aabb, const float* grad_out, int32_t L, int32_t F,
                          int32_t T_log2, float base_resolution, float per_level_scale, float* grad_table, void* stream);

/* The same gradient, reproducible bit for bit: a fixed-point sum that does not depend on the order of the points, the
 * launch or the GPU.  Same arguments as pnr_hashgrid_backward, plus a workspace; ACCUMULATES into grad_table.  For a
 * call over n > 0 points, level l, entry e of that level and feature f:
 *   1. Scale.  m_l = the largest finite |grad_out[p, l*F + f]| over all p and f; m_l = frac * 2^e_l with frac in
 *      [0.5, 1) (frexp); s_l = 61 - ceil(log2 n) - e_l.  A level with m_l = 0 adds nothing.
 *   2. Contribution of corner k of point p (w_k and the row idx from the forward's corner arithmetic):
 *      c = fp32(w_k * g), g = grad_out[p, l*F + f] (the product the atomic path makes);
 *      q = round-to-nearest-even((double)c * 2^s_l) as an int64 (the product is exact in double).
 *   3. Sum.  acc[l, e, f] = sum of q over the contributions to (l, e, f), in int64: exact, in any order.
 *   4. Result.  grad_table[l, e, f] += fp32((double)acc * 2^-s_l): int64 -> double (round to nearest), the exact
 *      product with the power of two, double -> float (round to nearest), then one fp32 add.
 *   5. Non-finite gradients.  A non-finite g at (p, l, f) is left out of m_l and of the sums; it sets the (l, idx_k, f)
 *      entries of all 8 of p's corners to NaN.  Every other entry is the rule applied to the finite contributions.
 * Overflow cannot happen: a point's 8 corner weights sum to at most 1 + 2^-20, |c| * 2^s_l <= |w_k| m_l (1 + 2^-24)
 * 2^s_l and m_l 2^s_l < 2^(61 - ceil(log2 n)) <= 2^61 / n, so the absolute sum of every quantized contribution of a
 * level - a fortiori of one entry - stays below 2^61 (1 + 2^-20) + 4n < 2^63 (each rounding adds at most 1/2).
 * Error against float64: 2^-24 |w_k g| + 2^-(s_l + 1) per contribution (at n = 2^19 the quantum 2^-s_l is at most
 * 2^-42 m_l), then the final two roundings of each entry.
 * workspace: pnr_hashgrid_fixed_workspace_bytes(L, F, T_log2) bytes of device scratch, 16-byte aligned, zeroed by the
 * call: int64 acc [L, 2^T_log2, F], one poison bit per entry (in 16-byte units), u32 max_bits [L], i32 scale [L],
 * u32 flags [2], rounded up to 16 bytes.  A short or misaligned workspace is refused before any launch.  The host
 * reads nothing back: the call can be captured in a CUDA graph.  pnr_hashgrid_fixed_workspace_bytes returns 0 for an
 * L, F or T_log2 the call refuses. */
size_t pnr_hashgrid_fixed_workspace_bytes(int32_t L, int32_t F, int32_t T_log2);
int pnr_hashgrid_backward_fixed(const float* x, int64_t n, const float* aabb, const float* grad_out, int32_t L,
                                int32_t F, int32_t T_log2, float base_resolution, float per_level_scale,
                                float* grad_table, void* workspace, size_t workspace_bytes, void* stream);

/* a8 + a9 in ONE kernel: Network.forward with the compositing done in the MLP's epilogue - per-sample alpha /
 * transmittance / weight right after the sigma-producing layer, colours and logits reduced on chip per ray - so the
 * network outputs `raw` [R,N,4+C+K] (456 B per sample with both heads) are never written to memory; only
 * out->weights [R,N] (REQUIRED) and the per-ray maps leave the SM.  Same maps as pnr_mlp_forward + pnr_composite
 * (weights bit-identical, sums in a different but fixed order); fixed_* maps come from the weights and the id
 * tables (a small second kernel).  Needs N % 32 == 0 and rays mode; sem_softmax is not available here
 * (PNR_ERR_UNSUPPORTED: use the two-call path). */
int pnr_mlp_composite(pnr_ctx* ctx, const float* rays, const float* z, int64_t R, int32_t N,
                      int32_t white_bkgd, int32_t mask_outside, const int32_t* sample_box,
                      const int32_t* box_sem, const int32_t* box_inst, int32_t B,
                      const pnr_composite_out* out, void* stream);

/* a9 backward (SURVEY 8(f) rank 2, first stage of the backward chain): d(loss)/d(raw) [R,N,4+C+K] from the
 * gradients of the composited maps (any pointer may be NULL = zero gradient; disp_map is not differentiated).
 * Same arguments as pnr_composite.  sem_softmax != 0 returns PNR_ERR_UNSUPPORTED. */
typedef struct pnr_composite_grads {
  const float* rgb_map;    /* [R,3] */
  const float* depth_map;  /* [R]   */
  const float* acc_map;    /* [R]   */
  const float* weights;    /* [R,N] */
  const float* semantic_map;        /* [R,C] */
  const float* instance_map;        /* [R,K] */
  const float* fixed_semantic_map;  /* [R,C] */
  const float* fixed_instance_map;  /* [R,K] */
} pnr_composite_grads;
int pnr_composite_backward(const float* raw, const float* z, const float* rays, int64_t R, int32_t N,
                           int32_t C, int32_t K, int32_t white_bkgd, int32_t sem_softmax, int32_t mask_outside,
                           const int32_t* sample_box, const int32_t* box_sem, const int32_t* box_inst,
                           int32_t B, const pnr_composite_grads* g, float* d_raw, void* stream);

/* a8 backward, first slice (SURVEY 8(f) rank 2; replaces autograd through Network.forward's trunk - the D
 * `pts_linears` with their ReLUs and the skip concatenation): dL/d(trunk input) (the first 3 + 6*xyz_res columns
 * of grad_emb [R*N, ld_emb], or E = hash_levels * hash_features columns = dL/dh(x) for a hash-grid context; ld_emb =
 * that width rounded up to 16 on a 16-byte aligned base lets the kernel use 16-byte stores) from
 * grad_h = dL/dh of the trunk output [R*N, W].  One kernel on the same 128-sample tiles as pnr_mlp_forward: the
 * forward trunk is recomputed (ReLU sign patterns stay in shared memory), then the layers run in reverse with the
 * transposed weight stream on the tensor cores, gradients split hi/lo like activations.  Samples are given as pts
 * [R*N,3] or as (rays [R,6], z [R,N]).  x3 precisions only; D <= 9.  grad_scale: a power of two applied to grad_h on
 * load and removed from everything the kernel writes (exact): pick it so that max |grad_h| * grad_scale is a few
 * hundred, or the fp16 operand parts of small gradients go subnormal (absolute floor 2^-25 / grad_scale; 1.0 when
 * grad_h is already O(1)).  The same scale carries every intermediate dZ_j, which can grow well past max |grad_h|
 * (a layer with small weights feeding one with large ones): one whose scaled value reaches 65520 in fp16x3 sets
 * PNR_STATUS_RANGE; rerun with a smaller grad_scale. */
int pnr_mlp_backward_trunk(pnr_ctx* ctx, const float* pts, const float* rays, const float* z, int64_t R, int32_t N,
                           const float* grad_h, float grad_scale, float* grad_emb, int32_t ld_emb, float* stash,
                           uint32_t* stash_absmax, void* stream);
/* The weight gradients of the trunk come from `stash` [2D-1, R*N, W] fp32 (NULL: not kept): every A operand the
 * kernel produces on the way - slot i < D-1: H_i, the activations of forward layer i; slot 2D-2-j: dZ_j, the gradient
 * w.r.t. layer j's pre-activation - so that dW_j = dZ_j^T [H_{j-1} (, gamma(x))], db_j = sum_s dZ_j are GEMMs over
 * the samples: pnr_wgrad.  pnr_mlp_trunk_forward returns the trunk's output h [R*N, W] (16-byte
 * aligned), the input of the layers after the trunk (alpha / feature / view / rgb / heads), which the caller
 * differentiates itself to obtain grad_h.
 * stash_absmax (nullable; needs stash) [2D-1] u32, zeroed by the call: slot k receives the largest magnitude written
 * to stash slot k, as the bit pattern of its 16-bit hi part in the context's operand format (fp16 / bf16) and for
 * the gradient slots BEFORE the division by grad_scale - enough to pick pnr_wgrad's power-of-two dz_scale without
 * another pass over the stash. */
int pnr_mlp_trunk_forward(pnr_ctx* ctx, const float* pts, const float* rays, const float* z, int64_t R, int32_t N,
                          float* h_out, void* stream);

/* a8 backward, weight gradients (SURVEY 8(f) rank 2): dW [No, Ni] (row stride ld_w) (+)= dZ^T X and db [No] (+)= column
 * sums of dZ (NULL: skipped), for dZ [S, No] (row stride ld_dz) and X [S, Ni] (row stride ld_x), fp32, No, Ni <= 256
 * (wider layers - the skip layer's [gamma(x), h], the view layer's [feature, gamma(d)] - are split by columns into
 * two calls on the same dZ).  A split-K GEMM over the samples on the tensor cores: every CTA accumulates its share of
 * the samples in registers (operands split into 16-bit hi / lo parts on the fly, hi.hi + lo.hi + hi.lo, fp32
 * accumulation), the partial products are added in a fixed order by a second kernel (deterministic).
 * precision = PNR_PREC_BF16X3 (~2^-17 per product, fp32 exponent range: gradients need no scaling) or PNR_PREC_FP16X3
 * (~2^-21 per product; dz_scale - DEVICE scalar or NULL - is a power of two dZ is multiplied by on load and dW divided
 * by, exact, so that the fp16 parts of ~1e-6 gradients stay normal; |X| and |dZ * scale| must stay below 65504).
 * accumulate != 0 adds to dW / db instead of overwriting them.
 * workspace: pnr_wgrad_workspace_bytes(No, Ni) bytes of device scratch (16-byte aligned) on the current device.
 * S = 0 needs no workspace (NULL is accepted): dW and db (when given) are set to 0, or left as they are under
 * accumulate.  A NaN or Inf in dZ[s, o] reaches only row o of dW and db[o]; one in X[s, i] only column i of dW.
 * Replaces the trunk's dW_j = dZ_j^T [H_{j-1}] on pnr_mlp_backward_trunk's stash and the weight gradients of the
 * layers after the trunk; the reference gets them from torch.autograd through nn.Linear. */
size_t pnr_wgrad_workspace_bytes(int32_t No, int32_t Ni);
int pnr_wgrad(const float* dz, int64_t ld_dz, int32_t No, const float* x, int64_t ld_x, int32_t Ni, int64_t S,
              int32_t precision, const float* dz_scale, float* dW, int64_t ld_w, float* db, int32_t accumulate,
              void* workspace, size_t workspace_bytes, void* stream);

/* a8 on the training path, the layers AFTER the trunk (alpha / feature / view / rgb / heads; SURVEY 8(f) rank 2):
 * y [S, N] (row stride ld_y) = act(x W^T + bias) for x [S, K] (row stride ld_x), fp32, N <= 256, K <= 512, on the
 * tensor cores with the 3-product 16-bit operand split of the fused MLP kernel (precision = PNR_PREC_FP16X3 or
 * PNR_PREC_BF16X3), fp32 accumulation in registers.  W is [N, K] (row stride ld_w), or with transposed != 0 a
 * [K, N] matrix read transposed: dL/dx = g W of a layer y = x W^T is pnr_linear(g, W, transposed = 1).  bias [N] or
 * NULL; relu != 0 applies max(., 0) and keeps NaN as NaN (as torch.relu does).  S = 0 writes nothing.
 * in_scale: DEVICE scalar or NULL - a power of two the rows of x are multiplied
 * by on load, the result divided by it (exact): gradients of a mean-reduced loss are ~1e-6 and their fp16 parts would
 * go subnormal unscaled.  workspace: pnr_linear_workspace_bytes(N, K) bytes, 16-byte aligned (the packed weights).
 * The render path does not use this (there these layers are steps of the fused kernel); the reference runs
 * nn.Linear / autograd here. */
size_t pnr_linear_workspace_bytes(int32_t N, int32_t K);
int pnr_linear(const float* x, int64_t ld_x, int32_t K, const float* W, int64_t ld_w, int32_t transposed,
               const float* bias, int32_t N, int64_t S, int32_t relu, int32_t precision, const float* in_scale,
               float* y, int64_t ld_y, void* workspace, size_t workspace_bytes, void* stream);

/* a10: sample_pdf + merge.  z [R,N] coarse depths, weights [R,N] coarse weights; bins are the mid
 * points, the pdf is weights[1:-1]+1e-5.  u [R,Ni] is required (deterministic sampler: the host's
 * linspace(0,1,Ni) broadcast over rays, so the values are the caller's, bit for bit).
 * Out (nullable each): z_fine [R,Ni], idx [R,Ni] i64 (searchsorted right), z_all [R,N+Ni] sorted. */
int pnr_sample_pdf(const float* z, const float* weights, int64_t R, int32_t N, int32_t Ni,
                   const float* u, float* z_fine, int64_t* idx, float* z_all, void* stream);

/* Refresh the weights of a loaded context from DEVICE tensors (same list, order and shapes as pnr_load_weights; fp32,
 * contiguous), stream-ordered on `stream`: what a training loop calls after every optimiser step.  The per-tile
 * programs and their packing plans do not depend on the values, so nothing is rebuilt or copied through the host: the
 * tensors are copied into the context's weight vector, the feature_linear fold is recomputed there, and kernels apply
 * the plans of the forward program (and of the trunk-forward / backward programs once they exist) to it; a plan goes
 * to the device on its program's first update.  Bit-identical to a fresh pnr_load_weights of the same values.  A
 * packed weight outside the fp16 range sets bit 1 of the status word (pnr_status) in the fp16 modes. */
int pnr_update_weights(pnr_ctx* ctx, const float* const* device_tensors, int32_t n, void* stream);

/* Host-only twin of pnr_load_weights (no CUDA call, no context): builds the per-tile program of the fused MLP
 * kernel and its packing plan for `cfg`, applies the plan to the tensors as pnr_load_weights does (same checks), and
 * returns the program, the packed 16-bit weight stream and the constant table in caller buffers (each may be NULL to
 * query sizes only).  `program` receives the MlpProgram struct of csrc/mlp_program.h.
 * For the CPU test tier: tests/test_cpu_program.py replays the program on the host and compares it with
 * the oracle's Network.forward. */
#define PNR_PROGRAM_SPLIT_E1 4  /* flags: E1 signalled in two blocks */
#define PNR_PROGRAM_NO_SPLIT 8  /* flags: start from one-block epilogues instead of the precision's default */
#define PNR_PROGRAM_BACKWARD 16 /* flags: the backward program of the trunk (pnr_mlp_backward_trunk) instead */
#define PNR_PROGRAM_VIEW_PRODUCERS 32 /* flags: the variant whose view epilogue runs on the producer warps (no heads) */
int pnr_program_host(const pnr_config* cfg, const float* const* tensors_host, const int64_t* shapes, int32_t n,
                     int32_t flags, void* program, size_t program_cap, size_t* program_bytes,
                     void* wpacked, size_t wpacked_cap, size_t* wpacked_bytes,
                     float* consts, size_t consts_cap, size_t* n_consts);

/* a3/a4: Renderer.render / batchify_rays as ONE call.  Everything render_rays does for R rays - scene near/far,
 * ray/primitive intersection, stratified sampling + per-sample ids, Network.forward, raw2outputs and, when
 * Ni > 0, sample_pdf + merge + the fine pass - is enqueued on `stream` in ray chunks sized by the caller's
 * workspace, so the big intermediate (raw [chunk, N+Ni, 4+C+K]) never exceeds it (size it with
 * pnr_workspace_bytes).
 * Results do not depend on the chunking (every kernel is per-ray and deterministic).
 * All pointers are DEVICE pointers except aabb_host; outputs and most inputs are optional (NULL). */
enum { PNR_SAMPLE_UNIFORM = 0,    /* z = near*(1-t) + far*t over [near, far], samples tagged with the interval they fall in */
       PNR_SAMPLE_INTERVALS = 1   /* a6: the N samples are placed inside the ray's M hit intervals (pnr_sample_intervals) */ };
typedef struct pnr_render_args {
  const float* rays;            /* [R,6] origin || direction                                                      */
  int64_t R;
  const float* near;            /* [R] and                                                                        */
  const float* far;             /* [R]; or both NULL: from aabb_host (pnr_scene_near_far) or near_min/far_default  */
  const float* aabb_host;       /* {lo.xyz, hi.xyz} HOST floats, or NULL                                          */
  float near_min, far_default;
  const float* box_center;      /* [B,3]   bounding primitives (B = 0: none)                                      */
  const float* box_half;        /* [B,3]                                                                          */
  const float* box_rot;         /* [B,3,3]                                                                        */
  const int32_t* box_sem;       /* [B] class id per primitive (fixed_semantic_map), nullable                      */
  const int32_t* box_inst;      /* [B] instance id per primitive (fixed_instance_map), nullable                   */
  int32_t B, M;                 /* M = hits kept per ray (<= 8)                                                   */
  int32_t N, Ni;                /* coarse samples, importance samples (0: single pass)                            */
  const float* t_vals;          /* [N] linspace(0,1,N) computed by the caller (host linspace, bit for bit)        */
  const float* u;               /* [R,N] jitter, required when perturb > 0                                        */
  float perturb;
  const float* u_fine;          /* [R,Ni] (row stride u_fine_stride floats; 0 = one row shared by all rays)       */
  int64_t u_fine_stride;
  int32_t sample_mode;          /* PNR_SAMPLE_*                                                                   */
  int32_t white_bkgd, sem_softmax, mask_outside, bound_by_primitives;
  pnr_composite_out out;        /* maps of the final pass                                                         */
  pnr_composite_out out0;       /* maps of the coarse pass (only used when Ni > 0)                                */
  float* z_vals;                /* [R,N+Ni] depths of the final pass                                              */
  float* z_vals0;               /* [R,N] coarse depths (Ni > 0)                                                   */
  uint8_t* hit_mask;            /* [R]                                                                            */
  int32_t* box_id;              /* [R,M]                                                                          */
  float* t_in;                  /* [R,M]                                                                          */
  float* t_out;                 /* [R,M]                                                                          */
  int32_t* sample_box;          /* [R,N+Ni] primitive id per sample of the final pass (-1 = none)                 */
  float* near_out;              /* [R] near / far actually used                                                   */
  float* far_out;               /* [R]                                                                            */
  void* workspace;              /* device scratch, caller-owned                                                   */
  size_t workspace_bytes;
  const int32_t* mesh_tri_start;  /* [B+1] mesh primitives (pnr_intersect_meshes), or NULL with T = 0: cuboids only */
  const float* mesh_tris;       /* [T,3,3]                                                                        */
  int64_t T;
} pnr_render_args;
/* ctx_fine: the network of the fine pass (NULL = ctx), with the same num_classes and num_instances as ctx
 * (PNR_ERR_ARG otherwise: the maps are [R,C] / [R,K] of ctx). */
int pnr_render_fused(pnr_ctx* ctx, pnr_ctx* ctx_fine, const pnr_render_args* args, void* stream);
/* pnr_render_fused on a sequence table: `frames` (nullable; NULL or F = 0 is pnr_render_fused) gives each ray's frame
 * (ray_frame [R], offset with the ray chunks) and the table's frame blocks, and the intersection is
 * pnr_intersect_frames'.  Refused as there, and F >= 1 without primitives (B = 0).  pnr_render_args keeps its layout,
 * so callers built against it are unchanged. */
int pnr_render_fused_frames(pnr_ctx* ctx, pnr_ctx* ctx_fine, const pnr_render_args* args, const pnr_frame_table* frames,
                            void* stream);

/* Bytes of device scratch pnr_render_fused wants for R rays: enough for one chunk of min(R, rays_per_chunk) rays
 * with every optional output absent, where rays_per_chunk puts `raw` near 1.5 GB and never below ~64 tiles of the
 * fused MLP per SM (smaller chunks cost more in kernel ramp-up than they save), and at least enough for
 * min(R, ~64 samples per SM) rays of a sem_softmax call, whose passes keep `raw`.  So every call of R rays with
 * M <= 8 renders in it.  Any workspace that holds at least one ray of the call works (more chunks); a smaller one is
 * refused before any launch (PNR_ERR_ARG, "cannot hold one ray"). */
size_t pnr_workspace_bytes(const pnr_ctx* ctx, int64_t R, int32_t N, int32_t Ni);

/* 8(e) multi-GPU entry: one NCCL communicator per rank (NCCL is bound at run time: pnr_comm_available() == 0
 * when libnccl.so.2 cannot be loaded) and ONE all-gather of the rendered per-ray tiles.  Rays shard across ranks
 * with no data-path collective; this gather of image / label tiles is the only exchange step of the path.
 * Rank 0 creates the id with pnr_comm_unique_id and hands its PNR_COMM_ID_BYTES bytes to the other ranks over any
 * out-of-band channel (the host application's launcher; torch.distributed.broadcast in the Python layer).
 * pnr_allgather_outputs: recv [world * bytes_per_rank] <- each rank's send [bytes_per_rank], in rank order,
 * asynchronously on `stream` (in place when send == recv + rank * bytes_per_rank). */
#define PNR_COMM_ID_BYTES 128
typedef struct pnr_comm pnr_comm;
int pnr_comm_available(void);
int pnr_comm_unique_id(uint8_t* id_out);
int pnr_comm_init(pnr_comm** out, const uint8_t* id, int32_t rank, int32_t world, int32_t device);
int pnr_comm_destroy(pnr_comm* comm);
int pnr_allgather_outputs(pnr_comm* comm, const void* send, void* recv, size_t bytes_per_rank, void* stream);
/* buf [bytes] on every rank <- root's buf, asynchronously on `stream` (data-parallel training starts every replica from
 * rank 0's parameters and optimiser state with it). */
int pnr_broadcast(pnr_comm* comm, void* buf, size_t bytes, int32_t root, void* stream);

/* Adam over one flat fp32 parameter vector param [P] with moments exp_avg, exp_avg_sq [P], whose gradient is the sum of
 * G slices grads[g * ld_grad + i] (the all-gathered gradients of G data-parallel ranks), added in rank order
 * g = 0, 1, ..., G-1 in fp32 starting from slice 0 (G = 1 uses the slice as it is).  The update is torch.optim.Adam's
 * single-tensor path (foreach=False), operation for operation, every operation rounded to fp32 (no FMA contraction):
 *   g += weight_decay * p                                      (only when weight_decay != 0)
 *   m  = lerp(m, g, w1), w1 = (float)(1 - beta1):  m + w1 * (g - m) when w1 < 0.5, else g - (g - m) * (1 - w1)
 *   v  = v * (float)beta2 + ((float)(1 - beta2) * g) * g
 *   denom = sqrt(v) / bc2_sqrt + eps
 *   p  = p + (-step_size) * (m / denom)
 * beta1, beta2: as the user set them (double; rounded as torch's kernels receive them); step_size = lr / (1 - beta1^t)
 * and bc2_sqrt = sqrt(1 - beta2^t), computed by the caller in double for step t and rounded to float.
 * grad_sum [P] (nullable) receives the summed gradient (before weight decay).  NaN and Inf propagate, unsuppressed.
 * HBM-bound: (G + 3) reads and 3 writes of 4P bytes (+ one write with grad_sum); 16-byte accesses when ld_grad % 4 == 0
 * and every buffer is 16-byte aligned.  Refused before any launch (PNR_ERR_ARG): G < 1, P < 0, ld_grad < P, a null
 * buffer when P > 0, a hyper-parameter that is not finite, betas outside [0, 1), eps, weight_decay or step_size < 0,
 * bc2_sqrt <= 0. */
typedef struct pnr_adam_args {
  int64_t P, ld_grad;
  int32_t G;
  double beta1, beta2;
  float eps, weight_decay, step_size, bc2_sqrt;
} pnr_adam_args;
int pnr_adam_step(const float* grads, float* param, float* exp_avg, float* exp_avg_sq, const pnr_adam_args* args,
                  float* grad_sum, void* stream);

/* Evaluation of rendered frames against their ground truth (the step after pnr_panoptic_fuse; the reference's
 * evaluator is not in the mount, so these rules are chosen here - DESIGN.md 3.4, oracle/reference_eval.py).
 * Ids are panoptic ids id*1000 + n, as pnr_panoptic_fuse writes them and KITTI-360's 2D instance images store them.
 * An id's class channel: a negative id is void; otherwise the dataset id d = id / 1000 maps to
 * id_to_channel[d] (DEVICE [n_ids] i32) when the table is given - void when d >= n_ids or the entry is outside
 * [0, C) - and to d itself when d < C without a table (void otherwise).  C in [1, 64]; n < 2^31.
 * Every accumulator ACCUMULATES (zero it first); counts are exact integers and every floating-point result is
 * deterministic (no float atomics), so the same inputs give bit-identical accumulators. */
/* conf [C, C+1] u64 += pixels by (gt channel, prediction channel) over the pixels whose gt channel is not void;
 * column C counts predictions that map to no channel.  IoU_c = conf[c,c] / (row_c + col_c - conf[c,c]). */
int pnr_eval_semantic(const int32_t* pred_pan, const int32_t* gt_pan, int64_t n, int32_t C,
                      const int32_t* id_to_channel, int32_t n_ids, uint64_t* conf, void* stream);
/* Panoptic quality of one frame (Kirillov et al. 2019, with the void / crowd handling of the COCO / Cityscapes
 * panoptic tools): segments are the distinct non-void ids; a gt pixel of channel -1 is void; a gt segment of a thing
 * class (is_thing [C] u8) with n == 0 is a crowd region.  A prediction and a gt of the same channel match when
 * IoU > 0.5 (exactly 0.5 does not), union = area_p + area_g - inter - |p ∩ void|.  Per channel c:
 * tp[c], fp[c], fn[c] u64 += the frame's matches, unmatched predictions (except those with
 * (|p ∩ void| + |p ∩ crowd of c|) / area_p > 0.5) and unmatched non-crowd gt segments; iou_sum[c] (double) += the
 * frame's matched IoUs, summed exactly and rounded once (so equal to math.fsum of them).
 * workspace: pnr_eval_workspace_bytes(n) bytes of device scratch, 16-byte aligned (hash tables of >= 2n slots, so
 * they cannot fill; a smaller workspace is rejected before any launch). */
size_t pnr_eval_workspace_bytes(int64_t n);
int pnr_eval_panoptic(const int32_t* pred_pan, const int32_t* gt_pan, int64_t n, int32_t C,
                      const int32_t* id_to_channel, int32_t n_ids, const uint8_t* is_thing, void* workspace,
                      size_t workspace_bytes, uint64_t* tp, uint64_t* fp, uint64_t* fn, double* iou_sum, void* stream);
/* Image and depth error sums of one frame, in double from the fp32 maps: frame_sums [6] +=
 * {sum over pixels and channels of (rgb_map - rgb_gt)^2 [n,3], pixels, then over the pixels with depth_gt > 0:
 * sum |d|, sum d^2, sum |d| / depth_gt, pixels} with d = depth_map - depth_gt.  Either pair may be NULL (its sums are
 * left alone).  Fixed-shape reductions: block trees over a grid that depends on n only, then one fixed tree.
 * workspace: any buffer of pnr_eval_workspace_bytes(n) bytes (any n) works. */
int pnr_eval_image(const float* rgb_map, const float* rgb_gt, const float* depth_map, const float* depth_gt,
                   int64_t n, double* frame_sums, void* workspace, size_t workspace_bytes, void* stream);

/* Number of kernels this library has launched on this thread since the last reset (bench evidence). */
int64_t pnr_launch_count(int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* PNR_H_ */
