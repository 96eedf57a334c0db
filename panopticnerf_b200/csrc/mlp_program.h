// mlp_program.h — the per-tile "program" the fused MLP kernel interprets (built once on the host when
// weights are loaded, see pnr_api.cu) and the shared-memory map of the sm_90 kernel (mlp_wgmma.cu).
//
// A tile runs a fixed sequence of STEPS (one GEMM + epilogue each: trunk layers, heads, view branch with the feature
// layer folded in).  Every step is issued as two N-HALVES (h0, h1) with separate accumulator column ranges; each half
// is a list of weight STAGES (<= 32 KB: up to 128 rows x 64 K, hi image then lo image), streamed by TMA.  A operands
// are addressed as packed operand columns (see the column map below).  The sm_90 kernel runs the steps in order and
// reads the stage list (st) and the epilogue table (ep).
//
// UNUSED ON SM_90.  The program also carries a finer-grained schedule, written for a kernel in which a step's
// epilogue overlaps the next step's MMAs: per stage the epilogue hand-offs it waits for and the commits it makes
// (flags other than F_FIRST / F_COMMIT_ACC1 / F_COMMIT_VIEW, IssueDesc, acc_flip, view_step), placed on the host from the
// operand-column footprints of every stage and epilogue part (Builder::finalize; its consistency is checked by
// tests/test_cpu_hazards.py).  The sm_90 kernel executes none of it: it runs each step's epilogue after all of that
// step's MMAs have retired, and reads F_FIRST (first MMA of a half overwrites) and F_COMMIT_ACC1 / F_COMMIT_VIEW (last
// stage of a step) only.  The parts of that schedule:
//
// E1 works in two PARTS (column blocks a, b; part b may be empty) that are SIGNALLED separately, so the next step's
// first K-chunks can start when half of E1 is done.  Epilogue -> MMA hand-offs are three monotonic counters (E0 done,
// E1 part a done, E1 done): every stage carries the counts it needs.
//
// ACCUMULATOR FLIP.  With acc_flip set, odd tiles address every accumulator column XOR 128 (no accumulator range
// straddles column 128), so that the first half of a tile's layer 0 does not wait for the previous tile's last
// epilogue.
//
// VIEW ON PRODUCERS (networks without heads, forward; built by pnr_program_host with PNR_PROGRAM_VIEW_PRODUCERS only, a
// context does not launch it).  view_step >= 0: the view step is the tile's last and may run its epilogue apart from
// the other steps; its last stage is flagged F_COMMIT_VIEW and the first stage of the next tile that reuses its
// accumulator columns waits for it.
//
// BACKWARD (dL/d(embedded input) through the trunk, on the same tiles).  A backward program is the trunk's forward
// steps - whose EPI_RELU_TO_A epilogues also save the 16-column sign patterns of their activations - followed by one
// step per layer in reverse order with the TRANSPOSED weights streamed the same way: the A operand is the gradient
// w.r.t. the layer's pre-activation (hi/lo split like any activation), the accumulator receives the gradient w.r.t.
// the layer's input, and the epilogue gates it with the saved pattern of the layer below.  The last forward layer's
// epilogue does not keep its activation: it loads the incoming gradient from global memory and gates it with its own
// sign pattern.  The embedded-input columns (layer 0, and the skip layer's first columns) are written / accumulated
// to the output rows by EPI_GRAD_OUT steps.
//
// The program travels as a __grid_constant__ kernel parameter (constant bank; nothing shared between contexts,
// streams, devices or graph replays).
#pragma once
#include <stdint.h>
#include <string.h>
#if defined(__CUDACC__)
#include <cuda_fp16.h>
#endif

namespace pnr {

constexpr int kTileM = 128;               // M of the program's instruction descriptors (IssueDesc::idesc)
constexpr int kRows = 64;                 // samples per tile of the sm_90 kernel = wgmma M of one warpgroup
constexpr int kRing = 2;                  // weight stages in flight
constexpr int kStageBytes = 32768;        // max stage: N=128 rows x 64 K x 2 bytes x (hi + lo images)
constexpr int kConsumerThreads = 128;     // one warpgroup: MMAs, positional encoding and epilogues
constexpr int kMlpThreads = kConsumerThreads + 32;   // + the weight-stream warp
constexpr int kMaxStages = 256;
constexpr int kMaxSteps = 24;
// floats: biases + sigma / rgb weights.  They live in global memory (MlpParams::consts); the bound is what the uint16_t
// offsets of EpiDesc can address: a table of at most 65536 floats starts every block at an offset <= 65535.
constexpr int kMaxConsts = 65536;
static_assert(kMaxConsts - 1 <= 0xFFFF, "EpiDesc::bias_off / aux_off are uint16_t");

// Operand column map.  The program addresses its A operands as "packed columns" of 32 bits (two 16-bit values of
// consecutive K) - 512 of them per row, the first 256 being accumulator space.
constexpr int kColAcc = 0;                // fp32 accumulators, up to 256 columns
constexpr int kColAHi = 256;              // activations, 16-bit hi parts, 2 per column (K <= 256)
constexpr int kColALo = 384;              // activations, 16-bit lo parts
constexpr int kColHeadHi = 128;           // head hidden activations (K <= 128) live in the upper
constexpr int kColHeadLo = 192;           //   half of the accumulator region while it is free
// The sm_90 kernel keeps accumulators in registers and the operand columns [kColOpBase, 512) in shared memory, in
// the no-swizzle K-major layout of wgmma: packed column c of row r is K-core (c - kColOpBase) / 4, i.e. the bytes
// ((c - kColOpBase) / 4 * kRows + r) * 16 + (c % 4) * 4.
constexpr int kColOpBase = 128;

// Shared-memory map of the sm_90 kernel (bytes from the 1024-aligned dynamic base).
constexpr int kSmemRing = 0;
constexpr int kSmemOp = kRing * kStageBytes;           // operand columns [128, 512): 96 K-cores x kRows x 16 B
constexpr int kOpKCoreBytes = kRows * 16;
constexpr int kSmemEmb = kSmemOp + (512 - kColOpBase) / 4 * kOpKCoreBytes;   // xyz embedding: hi 8K, lo 8K
constexpr int kEmbPartBytes = kRows * 64 * 2;
constexpr int kSmemDir = kSmemEmb + 2 * kEmbPartBytes; // view-dir embedding: hi 4K, lo 4K
constexpr int kDirPartBytes = kRows * 32 * 2;
constexpr int kSmemStage = kSmemDir + 2 * kDirPartBytes;   // fp32 accumulators of one 128-column window
constexpr int kStageLd = 128 + 4;                      // floats per staged row (padding: conflict-free 16-byte reads)

enum : uint8_t { A_TMEM = 0, A_EMB = 1, A_DIR = 2 };
enum : uint16_t {
  F_FIRST = 1,          // first MMA of this half overwrites the accumulator
  F_WAIT_E0 = 2,        // first stage of a step: needs E0 of the previous step
  F_WAIT_E1 = 4,        // first stage that touches anything E1 part b of the previous step reads or writes
  F_COMMIT_ACC0 = 8,    // last stage of h0: signal E0 when the MMAs so far retire
  F_COMMIT_ACC1 = 16,   // last stage of the step: signal E1
  F_COMMIT_WAR = 32,    // last stage reading the activation columns E0 of THIS step overwrites
  F_WAIT_EMB = 64, F_RELEASE_EMB = 128, F_WAIT_DIR = 256, F_RELEASE_DIR = 512,
  F_WAIT_E1A = 1024,    // first stage that touches anything E1 part a of the previous step reads or writes
  F_COMMIT_VIEW = 2048  // VIEW-ON-PRODUCERS programs: last stage of the view step (instead of F_COMMIT_ACC0/1)
};
enum : uint8_t { EPI_RELU_TO_A = 0, EPI_VIEW_RGB = 2, EPI_LOGITS = 3,   // (1 was a linear hand-over: feature_linear is folded now)
                 // backward programs (BWD kernels, see "BACKWARD" below):
                 EPI_MASK_TO_A = 4,     // v = acc where the saved ReLU sign pattern (slot n_valid-1) is set, else 0 -> A operand
                 EPI_LOADG_TO_A = 5,    // last forward layer: v = grad_in where acc + bias > 0, else 0 -> A operand
                 EPI_GRAD_OUT = 6,      // acc columns [0, n_valid) -> grad row + out_off (added to it when n_valid1 != 0)
                 EPI_ACT_OUT = 7 };     // relu(acc + bias) -> output row (the trunk's output h, for the layers torch differentiates)
#if defined(__CUDACC__)
__host__ __device__
#endif
constexpr bool epi_writes_a(uint8_t kind) { return kind == EPI_RELU_TO_A || kind == EPI_MASK_TO_A || kind == EPI_LOADG_TO_A; }

#if defined(__CUDACC__)
__host__ __device__ inline uint16_t bf16_rne(float x) {   // round to nearest even on the bit pattern (= cvt.rn.bf16.f32)
  uint32_t u;
  memcpy(&u, &x, 4);
  return (uint16_t)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}

// Element of the packed weight stream: part 0 (hi) or 1 (lo) of weight w in the operand format (fmt 0 = fp16, 1 = bf16),
// hi = w rounded to nearest even, lo = (w - hi) rounded to nearest even.  A stage's hi image holds part 0 of its
// weights, the lo image (x3 modes) part 1.  Packing plans are applied with this function on the host and on the device
// (pnr_update_weights, programs built after the load), so a stream packed on either is bit-identical to the other.
__host__ __device__ inline uint16_t weight_part16(float w, int part, int fmt) {
  if (fmt == 1) {
    const uint16_t hi = bf16_rne(w);
    if (part == 0) return hi;
    const uint32_t hb = (uint32_t)hi << 16;
    float h;
    memcpy(&h, &hb, 4);
    return bf16_rne(w - h);
  }
  const __half h = __float2half_rn(w);
  return __half_as_ushort(part == 0 ? h : __float2half_rn(w - __half2float(h)));
}
#endif

struct StageDesc {     // one weight stage = one bulk copy + its MMAs
  uint32_t gofs;       // byte offset into the packed weight stream
  uint32_t bytes;
  uint16_t n;          // MMA N (rows of the weight tile = width of this half)
  uint16_t acc_col;    // accumulator column of this half
  uint16_t a_off;      // A_TMEM: packed column of the first K16 step (hi part)
  uint16_t a_lo_off;   //         and of the lo part
  uint16_t flags;
  uint16_t lo_off16;   // offset of the lo image inside the stage, in 16-byte units (x3 modes)
  uint8_t ksteps;      // K16 steps covered by this stage
  uint8_t a_kind;
};

struct IssueDesc {     // the same stage, pre-digested for the MMA-issuing warp: every word is used as it is
  uint32_t idesc;      // instruction-descriptor word (M=128, N=n, operand format); not read on sm_90
  uint32_t b_lo_base;  // low word of the weight-tile descriptor without its address: (n*16 >> 4) << 16
  uint32_t b_inc;      // address-field step per K16: 2 * n*16 >> 4
  uint32_t lo_off16;
  uint32_t acc_col;
  uint32_t a_off, a_lo_off;
  uint32_t flags_k;    // flags | ksteps << 16 | a_kind << 24
  uint32_t needs;      // epilogue hand-offs this stage needs, as step counts + 1 relative to the tile's first step:
                       // E0 | E1 part a << 8 | E1 << 16  (v: the first v-1 steps of this tile - and every earlier
                       // tile - have finished that epilogue part; v = 0: the previous tile's last step may lack it)
};

struct EpiDesc {
  uint8_t kind;
  uint8_t sigma;       // also accumulate the sigma head (dot with consts[aux_off..]) on the activated values
  uint16_t n;          // accumulator columns of the step (multiple of 16)
  uint16_t n0;         // columns handled by E0 (h0); E1 handles [n0, n)
  uint16_t n_valid;    // EPI_LOGITS: real channel count
  uint16_t acc_col;
  uint16_t dst_col;    // packed destination column (hi) ; lo at dst_lo_col
  uint16_t dst_lo_col;
  uint16_t bias_off;   // float offset into consts (16-byte aligned)
  uint16_t aux_off;    // sigma weights (EPI_*_TO_A with sigma) or rgb weights [3][n] (EPI_VIEW_RGB)
  uint16_t out_off;    // EPI_LOGITS: channel offset in the raw row of column 0 (columns [0, n0), n_valid real ones)
  uint16_t out_off1;   //             and of column n0 (columns [n0, n), n_valid1 real ones) when the second half is a
                       // (backward programs: stash slot + 1 of the A operand this epilogue produces, 0 = not kept)
  uint16_t n_valid1;   //             layer of its own (two logit layers issued as the two halves of one step)
  uint16_t n1a;        // E1 part a = columns [n0, n1a), part b = [n1a, n)   (multiple of 16; n1a = n: one block)
};

struct MlpProgram {
  int32_t n_stages, n_steps, n_consts;
  int32_t sigma_bias_off, rgb_bias_off;   // float offsets into consts
  int32_t Lx, Ld;                          // octaves of gamma(x) (0 for a hash-grid trunk input) and gamma(d)
  int32_t passes;                          // 1 or 3
  int32_t acc_flip;                        // 1: odd tiles use the accumulator columns XOR 128 (see below)
  int32_t view_step;                       // >= 0: this (last) step's epilogue runs on the producer warps (see below)
  StageDesc st[kMaxStages];
  IssueDesc is[kMaxStages];
  EpiDesc ep[kMaxSteps];
};

enum { kMlpForward = 0, kMlpComposite = 1, kMlpBackward = 2 };   // launch_mlp's `mode`

// Launch arguments of the fused kernel (device pointers).
struct MlpParams {
  const uint8_t* wpacked;
  const float* consts;
  const float* pts;       // [S,3] or null
  const float* viewdirs;  // [S,3] or null
  const float* rays;      // [R,6] (used when pts == null)
  const float* z;         // [R,N]
  int64_t S;              // samples
  int32_t N;              // samples per ray (rays mode)
  int32_t CH;             // raw row width 4 + C + K
  float* raw;
  int32_t num_tiles;
  uint32_t* status;       // sticky device word: bit 0 = a non-finite / out-of-range activation was seen (may be null)
  int32_t head_blocks;    // 1: the sigma / rgb heads are summed in 8-column blocks (head_dot_*, mlp_wgmma.cu), the order
                          // of the 128-row kernel, for every launch of a program mlp_rows128_ok accepts; 0: one running
                          // sum per column share (the order of every other program); set by launch_mlp
  // ---- compositing epilogue (COMPOSITE kernels only: rays mode, N % 32 == 0; `raw` is not written)
  int64_t rays_per_cta;   // every CTA owns a contiguous range of whole rays (carries stay on chip)
  const int32_t* sample_box;   // [S] primitive id per sample, or null (only read when mask_outside)
  int32_t mask_outside, white_bkgd;
  int32_t C, K;           // semantic / instance channels of the network
  float* weights;         // [S]   per-sample compositing weights (always written)
  float* rgb_map;         // [R,3] nullable, like the rest
  float* depth_map;       // [R]
  float* acc_map;         // [R]
  float* disp_map;        // [R]
  float* sem_map;         // [R,C]
  float* inst_map;        // [R,K]
  // ---- backward kernels only: dL/dh of the trunk output, [S, W]; `raw` receives dL/d(embedded input), row stride CH
  const float* grad_in;
  // optional fp32 copies of every A operand the epilogues produce (hidden activations on the way up, pre-activation
  // gradients on the way down): slot k = stash + k * S * W, rows of W floats.  What the weight-gradient GEMMs read.
  float* stash;
  // the incoming gradient is multiplied by grad_scale as it is loaded and every gradient that leaves the kernel
  // (output rows, stashed dZ) by grad_unscale = 1 / grad_scale: a power of two chosen by the caller so that the
  // 16-bit operand parts of small gradients stay in the normal range (the backward pass is linear in grad_in)
  float grad_scale, grad_unscale;
  // optional [2D-1] words, zeroed by the launcher: slot k receives (atomic max) the largest |value| the kernel put into
  // stash slot k, as the bit pattern of its 16-bit hi part in the operand format and BEFORE grad_unscale is applied -
  // what the caller needs to pick the power-of-two scale of the weight-gradient GEMM without another pass over the stash
  uint32_t* stash_absmax;
  // ---- hash-grid trunk input (pnr_config.xyz_encoding = PNR_XYZ_HASHGRID): hash_table != null makes the prologue write
  // h(x) (hashgrid_math.cuh) instead of gamma(x) into the embedding operand; its E = hash_L * hash_F columns are padded
  // with zeros to the program's K (a multiple of 16)
  const float* hash_table;     // [hash_L, 2^hash_T_log2, hash_F] fp32, read as the launch executes
  int32_t hash_L, hash_F, hash_T_log2;
  float hash_aabb[6];          // {lo.xyz, hi.xyz}
  uint32_t hash_res[32];       // per-level resolutions (hash_level_resolutions)
};

// What a launch carries: arguments + the context's program, as ONE __grid_constant__ kernel parameter.
struct MlpLaunch {
  MlpParams p;
  MlpProgram prog;
};
static_assert(sizeof(MlpLaunch) <= 32764, "kernel parameter space is 32764 bytes");

// backward kernels: ReLU sign patterns, uint16 [slot][16-column group][row], in the head operand columns (unused by
// backward programs)
constexpr int kSmemMask = kSmemOp;
constexpr int kMaskSlotU16 = 16 * kRows;                      // one layer of up to 256 columns
constexpr int kMaxMaskSlots = 8;
static_assert(kMaxMaskSlots * kMaskSlotU16 * 2 <= (kColAHi - kColOpBase) / 4 * kOpKCoreBytes, "sign patterns overflow");
constexpr int kSmemPart = kSmemStage + kRows * kStageLd * 4;   // [2 column shares][kRows][4] floats
constexpr int kSmemBars = kSmemPart + 2 * kRows * 4 * 4;
constexpr int kSmemTotal = kSmemBars + 256;
// compositing epilogue: weights of the tile's rows, per-quarter transmittance products and the carried transmittance
// (double-buffered by tile parity), per-quarter partial sums of every composited channel (double-buffered); a
// "quarter" is an aligned group of 32 samples, kRows / 32 of them per tile
constexpr int kQuarters = kRows / 32;
constexpr int kCompMaxCh = 5 + 128 + 128;                       // rgb(3) depth acc + C + K
constexpr int kCompChPad = (kCompMaxCh + 31) / 32 * 32;         // 288
constexpr int kSmemCompW = kSmemTotal;                          // float w_row[kRows]
constexpr int kSmemCompQ = kSmemCompW + kRows * 4;              // float qprod[2][kQuarters]; float carry[2]; (64 bytes)
constexpr int kSmemCompS = kSmemCompQ + 64;                     // float qsum[2][kQuarters][kCompChPad]
constexpr int kSmemCompR = kSmemCompS + 2 * kQuarters * kCompChPad * 4; // float racc[kCompChPad]: running sums of the open ray
constexpr int kSmemTotalComp = kSmemCompR + kCompChPad * 4;
static_assert(kSmemTotalComp <= 232448, "shared-memory map exceeds the 227 KB per-CTA limit");

// Shared-memory map of the 128-row kernel (mlp_rows128_kernel: forward programs without heads, see
// mlp_rows128_ok).  Two consumer warpgroups, rows [64g, 64g + 64) of a 128-sample tile each; warpgroup g owns block g:
// its trunk activations (operand columns [256, 512), hi and lo), its xyz embedding and its view-dir embedding, in the
// layouts of the 64-row kernel.  Both read every slot of one 3-slot weight ring.  No staging tile: every epilogue runs
// from the accumulator registers.
constexpr int kRows128 = 2 * kRows;
constexpr int kMlp128Threads = 3 * kConsumerThreads;     // two consumer warpgroups + the weight-stream warpgroup
constexpr int kSlots128 = 3;
constexpr int kSlot128Bytes = kStageBytes / 2;            // half a stage, as in the 64-row kernel's ring
constexpr int kSmem128Ring = 0;
constexpr int kSmem128Blk = kSmem128Ring + kSlots128 * kSlot128Bytes;           // block of warpgroup 0
constexpr int kBlk128Op = 0;                                                     // columns [256, 512): 64 K-cores
constexpr int kBlk128Emb = kBlk128Op + (512 - kColAHi) / 4 * kOpKCoreBytes;      // xyz embedding: hi 8K, lo 8K
constexpr int kBlk128Dir = kBlk128Emb + 2 * kEmbPartBytes;                       // view-dir embedding: hi 4K, lo 4K
constexpr int kBlk128Bytes = kBlk128Dir + 2 * kDirPartBytes;
constexpr int kSmem128Sig = kSmem128Blk + 2 * kBlk128Bytes;   // float [kRows128]: each row's sigma dot, bias not added
constexpr int kSmem128Bars = kSmem128Sig + kRows128 * 4;      // full [kSlots128], empty [kSlots128]
constexpr int kSmem128Total = kSmem128Bars + 2 * kSlots128 * 8;
static_assert(kBlk128Bytes == 65536 + 16384 + 8192, "block: activations, embedding, view-dir embedding");
static_assert(kSmem128Blk % 1024 == 0 && kBlk128Bytes % 1024 == 0, "operand blocks 1024-aligned");
static_assert(kSmem128Total <= 232448, "128-row shared-memory map exceeds the 227 KB per-CTA limit");
static_assert(kConsumerThreads / 32 * 24 + 2 * kConsumerThreads / 32 * 240 <= 65536 / 32,
              "register split: 24 per weight-stream thread and 240 per consumer thread fit the register file");

// Can the 128-row kernel run forward program `pg`?  Its epilogues are the register ones (mlp_wgmma.cu): every step
// but the last is a ReLU hand-over of N = 256 as two N = 128 halves into the trunk activation columns, the one before
// the last also forming the sigma head; the last is the view step, N = 128 as one half.  Every A operand is the xyz
// embedding (K <= 64), the view-dir embedding (K <= 32) or the trunk activations, so no step reads or writes the head
// columns [128, 256), which the 128-row map does not have.  A 256-wide network without heads: cfg2, in every precision
// and with either trunk input.
inline bool mlp_rows128_ok(const MlpProgram& pg) {
  const int S = pg.n_steps;
  if (S < 2 || S > kMaxSteps || pg.n_stages < 1 || pg.n_stages > kMaxStages) return false;
  for (int s = 0; s < S; ++s) {
    const EpiDesc& e = pg.ep[s];
    if (e.acc_col != kColAcc || e.sigma != (s == S - 2 ? 1 : 0)) return false;
    if (s < S - 1 && !(e.kind == EPI_RELU_TO_A && e.n == 256 && e.n0 == 128 && e.dst_col == kColAHi &&
                       e.dst_lo_col == kColALo))
      return false;
    if (s == S - 1 && !(e.kind == EPI_VIEW_RGB && e.n == 128 && e.n0 == 128)) return false;
  }
  for (int i = 0; i < pg.n_stages; ++i) {
    const StageDesc& sd = pg.st[i];
    const int k = sd.ksteps * 16;   // K of the stage
    if (sd.a_kind == A_EMB) {
      if (k > 64) return false;
    } else if (sd.a_kind == A_DIR) {
      if (k > 32) return false;
    } else if (sd.a_kind != A_TMEM || sd.a_off < kColAHi || sd.a_lo_off < kColAHi || sd.a_off + k / 2 > 512 ||
               sd.a_lo_off + k / 2 > 512) {
      return false;
    }
  }
  return true;
}

}  // namespace pnr
