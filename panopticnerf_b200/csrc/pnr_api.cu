// pnr_api.cu — context management, weight packing / MLP program construction and the
// pnr_mlp_forward entry point of the C ABI (include/pnr.h).
#include <cstring>
#include <string>
#include <vector>
#include "common.cuh"
#include "hashgrid_math.cuh"
#include "mlp_program.h"
#include "sm90.cuh"

namespace pnr {

// ---------------------------------------------------------------- error / accounting plumbing
static thread_local char g_err[512] = "";
static thread_local int64_t g_launches = 0;

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
void count_launch(int n) { g_launches += n; }

int launch_mlp(MlpLaunch& L, int passes, int fmt, int mode, cudaStream_t stream);  // mlp_wgmma.cu

}  // namespace pnr

using namespace pnr;

// The MLP programs of a context, all over the same weights: forward (pnr_mlp_forward, pnr_mlp_composite,
// pnr_render_fused), backward (pnr_mlp_backward_trunk) and trunk-forward (pnr_mlp_trunk_forward).  pnr_load_weights
// builds the forward program; the other two are built on first use.
enum ProgramKind { kProgForward = 0, kProgBackward = 1, kProgTrunkForward = 2, kNumPrograms = 3 };

// A program's packing plan, which depends on the configuration and the shapes only.  V is the weight vector: the
// tensors of pnr_load_weights' list concatenated in order, then the derived block (Fold).  Packed element p is part
// wpart[p] (weight_part16) of V[wpos[p]], constant c is V[cpos[c]]; position -1 is zero padding.
struct Plan {
  std::vector<int32_t> wpos, cpos;
  std::vector<uint8_t> wpart;
};

struct PackedProgram {
  bool ready = false;             // built and packed since the last pnr_load_weights
  MlpLaunch launch;               // launch.prog = the program; launch.p is filled per call.  The whole struct travels as
                                  // the kernel's __grid_constant__ parameter: nothing is shared between contexts,
                                  // streams, devices or CUDA-graph replays.
  uint8_t* d_wpacked = nullptr;
  float* d_consts = nullptr;
  size_t n_w = 0, n_c = 0;        // packed 16-bit elements / constants
  Plan plan;                      // on the host until the program is first packed on the device (refresh)
  int32_t* d_widx = nullptr;
  uint8_t* d_wpart = nullptr;
  int32_t* d_cidx = nullptr;
};

struct pnr_ctx {
  pnr_config cfg;
  int passes = 3;
  int fmt = 0;   // 0 = fp16, 1 = bf16 (instruction-descriptor encoding)
  bool loaded = false;
  PackedProgram prog[kNumPrograms];
  uint32_t* d_status = nullptr; // sticky range-check word of the fused MLP (bit 0: activation out of operand range)
  const float* hash_table = nullptr;   // hash-grid contexts: the caller's table (pnr_bind_hashgrid_table), not owned
  uint32_t hash_res[kHashMaxLevels] = {};
  float* d_V = nullptr;   // V of the load or of the last pnr_update_weights: what programs are packed from on the device
  std::vector<int64_t> v_off, shapes;   // V's layout (Builder::v_off); the shapes given to pnr_load_weights
};

namespace {

// Instruction-descriptor word of the program's issue table (IssueDesc::idesc): M, N and operand-format fields of a
// 16-bit-operand MMA with fp32 accumulators.  Part of the overlapped schedule the sm_90 kernel does not execute
// (mlp_program.h, "UNUSED ON SM_90").
constexpr uint32_t make_idesc_f32acc(int M, int N, int fmt) {
  return (1u << 4) | (uint32_t(fmt) << 7) | (uint32_t(fmt) << 10) | (uint32_t(N >> 3) << 17) | (uint32_t(M >> 4) << 24);
}

// A row-major [out, in] matrix by the positions of its elements in V: element (r, c) is V[first + r * in + c] for a
// tensor of the list, V[pos[r * in + c]] for a matrix the build derives (a transposed or stacked copy of positions).
struct Mat {
  int32_t first;
  int out, in;
  const int32_t* pos = nullptr;
  int32_t at(int r, int c) const { return pos ? pos[(size_t)r * in + c] : first + r * in + c; }
};

struct Seg {
  uint8_t kind;        // A_TMEM / A_EMB / A_DIR
  Mat m;
  int col0, kvalid;    // columns of m feeding this segment
  int kpad;            // K rounded up (multiple of 16)
  int a_hi, a_lo;      // TMEM packed columns (A_TMEM)
  bool release;        // A_EMB/A_DIR: last reader in the tile
};

// Builds a program and its plan from the configuration and the tensors' shapes: it never reads a weight value, and
// looks at the tensor pointers only to check that they are given.
struct Builder {
  MlpProgram prog;
  Plan plan;
  int passes, fmt;
  // E1 in two blocks signalled separately (mlp_program.h).  Pays off when a half spans several weight stages
  // (the x3 modes, K = 64 per stage: 75.4 k -> 71.5 k cycles per tile); the 1-pass modes keep one block.
  bool split_e1;
  bool acc_flip = true;             // odd tiles use the accumulator columns XOR 128 when the program allows it
  bool view_on_producers = false;   // the (last, one-half) view step's epilogue runs on the producer warps (mlp_program.h)
  // V's layout, laid down as the build takes the tensors of the list, in list order: tensor i at v_off[i], and
  // v_off.back() the end of the last one taken - where the derived block starts once every tensor is taken
  std::vector<int64_t> v_off{0};
  const char* what = "";            // names the program in error texts (finish, pack_host)
  std::string err;

  Builder(int passes_, int fmt_) : passes(passes_), fmt(fmt_) {
    memset(&prog, 0, sizeof(prog));
    split_e1 = passes == 3;
  }

  // Position in V of tensor i, the next one of the list, whose shape has been checked
  int32_t take_tensor(const int64_t* shapes, int i) {
    v_off.push_back(v_off.back() + shapes[2 * i] * shapes[2 * i + 1]);
    return (int32_t)v_off[i];
  }

  int add_consts(int32_t first, int n_valid, int n_pad) {   // V[first .. first + n_valid), zero padded to n_pad
    const int off = (int)plan.cpos.size();
    for (int i = 0; i < n_pad; ++i) plan.cpos.push_back(i < n_valid ? first + i : -1);
    return off;
  }

  // Stage image of rows [row0, row0 + n_rows) x K [k0, k0 + 8*kcores): no-swizzle K-major core matrices,
  // byte offset of element (n, k) = ((k/8) * n_rows + n) * 16 + (k%8) * 2  (LBO = n_rows*16, SBO = 128).
  void pack_stage(const Mat& m, int row0, int n_rows, int col0, int kvalid, int k0, int kcores, int part) {
    const size_t base = plan.wpos.size();
    const int n_pad = n_rows;
    plan.wpos.resize(base + (size_t)n_pad * kcores * 8);
    plan.wpart.resize(plan.wpos.size(), (uint8_t)part);
    for (int kc = 0; kc < kcores; ++kc)
      for (int nn = 0; nn < n_pad; ++nn)
        for (int e = 0; e < 8; ++e) {
          const int n = row0 + nn;
          const int k = k0 + kc * 8 + e;
          plan.wpos[base + ((size_t)kc * n_pad + nn) * 8 + e] = (n < m.out && k < kvalid) ? m.at(n, col0 + k) : -1;
        }
  }

  struct StepInfo { int first_stage, n_stages, n0_stage; };  // n0_stage = first stage of h1 (or end)
  std::vector<StepInfo> steps;

  // One GEMM step: acc[:, acc_col:acc_col+n_pad) = sum_seg A_seg * W_seg^T, then epilogue `ed`.
  // Issued as two N-halves (rows [0,n0) then [n0,n_pad)) when n_pad >= 64, each its own stage list.
  // `segs_h1` + `n0_split`: the second half is a GEMM of its own (own matrices, rows counted from 0, own K range) -
  // two small layers that share nothing but the step, e.g. the two logit layers (block-diagonal, zero blocks skipped).
  bool add_step(std::vector<Seg> segs, int n_pad, int acc_col, EpiDesc ed, bool first_of_tile,
                const std::vector<Seg>* segs_h1 = nullptr, int n0_split = 0) {
    if (prog.n_steps >= kMaxSteps) { err = "too many steps"; return false; }
    const int n0 = n0_split > 0 ? n0_split : (n_pad >= 64 ? n_pad / 2 : n_pad);
    const int halves = n0 < n_pad ? 2 : 1;
    StepInfo info{prog.n_stages, 0, 0};
    bool emb_waited = false;
    for (int h = 0; h < halves; ++h) {
      const int r0 = h == 0 ? 0 : n0, r1 = h == 0 ? n0 : n_pad;
      const std::vector<Seg>& hsegs = (h == 1 && segs_h1) ? *segs_h1 : segs;
      const int mrow0 = (h == 1 && segs_h1) ? 0 : r0;     // first row of the half in its weight matrix
      const int half_first = prog.n_stages;
      if (h == 1) info.n0_stage = prog.n_stages;
      // the kernel issues one wgmma m64nNk16 per K step of a half: N a multiple of 8, at most 128
      if ((r1 - r0) % 8 != 0 || r1 - r0 > 128 || r1 <= r0) { err = "half of a step is not an MMA width (multiple of 8, <= 128)"; return false; }
      for (size_t si = 0; si < hsegs.size(); ++si) {
        const Seg& sg = hsegs[si];
        // K per stage: 64 with hi+lo images (x3), 128 with the hi image only (1-pass): <= 32 KB either way
        const int chunk = passes == 3 ? 64 : 128;
        for (int k0 = 0; k0 < sg.kpad; k0 += chunk) {
          const int kcores = ((sg.kpad - k0) < chunk ? (sg.kpad - k0) : chunk) / 8;
          {
            if (prog.n_stages >= kMaxStages) { err = "too many stages"; return false; }
            const int parts = passes == 3 ? 2 : 1;
            StageDesc& sd = prog.st[prog.n_stages++];
            memset(&sd, 0, sizeof(sd));
            sd.gofs = (uint32_t)(plan.wpos.size() * 2);
            sd.bytes = (uint32_t)((r1 - r0) * kcores * 16 * parts);
            sd.n = (uint16_t)(r1 - r0);
            sd.acc_col = (uint16_t)(acc_col + r0);
            sd.a_off = (uint16_t)(sg.a_hi + k0 / 2);
            sd.a_lo_off = (uint16_t)(sg.a_lo + k0 / 2);
            sd.lo_off16 = (uint16_t)((r1 - r0) * kcores);
            sd.ksteps = (uint8_t)(kcores / 2);
            sd.a_kind = sg.kind;
            const bool seg_first = (k0 == 0);
            const bool seg_last = (k0 + chunk >= sg.kpad);
            const bool last_half = h == halves - 1;
            if (sg.kind == A_EMB && seg_first && first_of_tile && !emb_waited) { sd.flags |= F_WAIT_EMB; emb_waited = true; }
            if (sg.kind == A_EMB && seg_last && sg.release && last_half) sd.flags |= F_RELEASE_EMB;
            if (sg.kind == A_DIR && seg_first && h == 0) sd.flags |= F_WAIT_DIR;
            if (sg.kind == A_DIR && seg_last && sg.release && last_half) sd.flags |= F_RELEASE_DIR;
            for (int part = 0; part < parts; ++part) pack_stage(sg.m, mrow0, r1 - r0, sg.col0, sg.kvalid, k0, kcores, part);
          }
        }
      }
      prog.st[half_first].flags |= F_FIRST;
      prog.st[prog.n_stages - 1].flags |= (h == 0 ? F_COMMIT_ACC0 : F_COMMIT_ACC1);
    }
    if (halves == 1) {
      prog.st[prog.n_stages - 1].flags |= F_COMMIT_ACC1;
      info.n0_stage = prog.n_stages;
    }
    prog.st[info.first_stage].flags |= F_WAIT_E0;
    info.n_stages = prog.n_stages - info.first_stage;
    steps.push_back(info);
    ed.n = (uint16_t)n_pad;
    ed.n0 = (uint16_t)n0;
    ed.acc_col = (uint16_t)acc_col;
    const int g1 = (n_pad - n0) / 16;
    ed.n1a = (uint16_t)(n0 + ((split_e1 && g1 >= 2) ? (g1 / 2) * 16 : (n_pad - n0)));
    prog.ep[prog.n_steps++] = ed;
    return true;
  }

  static bool overlap(int a0, int a1, int b0, int b1) { return a0 < a1 && b0 < b1 && a0 < b1 && b0 < a1; }

  // Tensor-memory footprints (column intervals) used to place the cross-step hazard flags.
  struct Foot { int acc0, acc1, hi0, hi1, lo0, lo1; };
  // what the columns [c0, c1) of step s's epilogue read (accumulator) and write (activation columns)
  Foot epi_foot(int s, int c0, int c1) const {
    const EpiDesc& e = prog.ep[s];
    Foot f{e.acc_col + c0, e.acc_col + c1, 0, 0, 0, 0};
    if (epi_writes_a(e.kind) && c0 < c1) {
      f.hi0 = e.dst_col + c0 / 2; f.hi1 = e.dst_col + c1 / 2;
      if (passes == 3) { f.lo0 = e.dst_lo_col + c0 / 2; f.lo1 = e.dst_lo_col + c1 / 2; }
    }
    return f;
  }
  bool stage_touches(const StageDesc& sd, const Foot& f) const {
    const int a0 = sd.acc_col, a1 = sd.acc_col + sd.n;   // accumulator columns this stage writes
    if (overlap(a0, a1, f.acc0, f.acc1) || overlap(a0, a1, f.hi0, f.hi1) || overlap(a0, a1, f.lo0, f.lo1)) return true;
    if (sd.a_kind == A_TMEM) {
      const int h0 = sd.a_off, h1 = sd.a_off + sd.ksteps * 8;
      if (overlap(h0, h1, f.hi0, f.hi1) || overlap(h0, h1, f.acc0, f.acc1)) return true;
      if (passes == 3) {
        const int l0 = sd.a_lo_off, l1 = sd.a_lo_off + sd.ksteps * 8;
        if (overlap(l0, l1, f.lo0, f.lo1) || overlap(l0, l1, f.acc0, f.acc1)) return true;
      }
    }
    return false;
  }

  // Place the waits on the previous step's E1 parts (cyclically: the first step of a tile follows the last step
  // of the previous tile), the write-after-read commit for this step's own E0, and the per-stage hand-off counts
  // of the issue table.
  void finalize() {
    const int S = prog.n_steps;
    // accumulator flip (mlp_program.h): allowed when no activation lives inside the accumulator region (the head
    // columns of single-head programs do) and no accumulator range straddles column 128
    bool flip = acc_flip;
    for (int s = 0; s < S; ++s) flip = flip && !(epi_writes_a(prog.ep[s].kind) && prog.ep[s].dst_col < kColAHi);
    for (int i = 0; i < prog.n_stages; ++i)
      flip = flip && prog.st[i].acc_col / 128 == (prog.st[i].acc_col + prog.st[i].n - 1) / 128;
    prog.acc_flip = flip ? 1 : 0;
    // view on producers: the view step must be the tile's last, issued as one half, with at least one step before it
    const bool vp = view_on_producers && S >= 2 && prog.ep[S - 1].kind == EPI_VIEW_RGB && prog.ep[S - 1].n0 == prog.ep[S - 1].n;
    prog.view_step = vp ? S - 1 : -1;
    if (vp) {
      StageDesc& last = prog.st[steps[S - 1].first_stage + steps[S - 1].n_stages - 1];
      last.flags = (uint16_t)((last.flags & ~(F_COMMIT_ACC0 | F_COMMIT_ACC1)) | F_COMMIT_VIEW);
    }
    std::vector<int> at_a(S), at_b(S);
    for (int s = 0; s < S; ++s) {
      const StepInfo& in = steps[s];
      const int end = in.first_stage + in.n_stages;
      // the step whose E0 / E1 counts precede this one's: cyclically the tile's last step - the last one the
      // epilogue warps run, i.e. not the view step of a view-on-producers program
      const int prev_step = (s == 0) ? (vp ? S - 2 : S - 1) : s - 1;
      const EpiDesc& pe = prog.ep[prev_step];
      const bool split = in.n0_stage < end;
      auto first_touch = [&](Foot f) {
        if (s == 0 && prog.acc_flip) {   // the previous step ran in the other tile parity: its accumulator columns
          const int w = f.acc1 - f.acc0; //   are the XOR-128 image of what the program says
          f.acc0 ^= 128;
          f.acc1 = f.acc0 + w;
        }
        int at = -1;
        for (int i = in.first_stage; i < end && at < 0; ++i)
          if (stage_touches(prog.st[i], f)) at = i;
        if (at < 0) at = split ? in.n0_stage : in.first_stage;
        else if (split && at > in.n0_stage) at = in.n0_stage;   // never later than the first stage of h1
        return at;
      };
      const int prev = prev_step;
      at_b[s] = first_touch(pe.n1a < pe.n ? epi_foot(prev, pe.n1a, pe.n) : epi_foot(prev, pe.n0, pe.n));
      at_a[s] = pe.n1a < pe.n ? first_touch(epi_foot(prev, pe.n0, pe.n1a)) : at_b[s];
      if (at_a[s] > at_b[s]) at_a[s] = at_b[s];                 // "E1 done" implies "E1 part a done"
      prog.st[at_a[s]].flags |= F_WAIT_E1A;
      prog.st[at_b[s]].flags |= F_WAIT_E1;
      // E0 of this step overwrites dst columns [dst, dst + n0/2) (hi and lo): last stage reading them
      const EpiDesc& e = prog.ep[s];
      int war = in.first_stage;
      if (epi_writes_a(e.kind)) {
        Foot f = epi_foot(s, 0, e.n0);
        f.acc0 = f.acc1 = 0;   // stores only: the loads of E0 are ordered by acc_full
        for (int i = in.first_stage; i < end; ++i)
          if (stage_touches(prog.st[i], f)) war = i;
      }
      // (the epilogue warps count one write-after-read phase per step THEY run: none for a producer-run view step)
      if (!(vp && s == S - 1)) prog.st[war].flags |= F_COMMIT_WAR;
    }
    // view on producers: the first stage of the tile that touches the accumulator columns the previous tile's view
    // epilogue reads (the other tile parity's image when the program flips) and every stage after it wait for it
    int v_from = prog.n_stages;
    if (vp) {
      const EpiDesc& ve = prog.ep[S - 1];
      Foot f{ve.acc_col, ve.acc_col + ve.n, 0, 0, 0, 0};
      if (prog.acc_flip) { f.acc0 ^= 128; f.acc1 = f.acc0 + ve.n; }
      for (int i = 0; i < prog.n_stages && v_from == prog.n_stages; ++i)
        if (stage_touches(prog.st[i], f)) v_from = i;
      // no stage of the next tile touches them (narrow networks in a flipping program: the columns come up again one
      // tile later): gate the whole next tile - the count is per tile, and a done epilogue stays done
      if (v_from == prog.n_stages) v_from = 0;
    }
    for (int s = 0; s < S; ++s) {
      const StepInfo& in = steps[s];
      for (int i = in.first_stage; i < in.first_stage + in.n_stages; ++i)
        prog.is[i].needs = (uint32_t)(s + 1) | ((uint32_t)(i >= at_a[s] ? s + 1 : s) << 8) |
                           ((uint32_t)(i >= at_b[s] ? s + 1 : s) << 16) | ((uint32_t)(i >= v_from ? 1 : 0) << 24);
    }
    for (int i = 0; i < prog.n_stages; ++i) {   // issue table (flags are final now)
      const StageDesc& sd = prog.st[i];
      IssueDesc& d = prog.is[i];
      const uint32_t rows = sd.n;                         // rows of the weight tile
      d.idesc = make_idesc_f32acc(kTileM, sd.n, fmt);     // fmt: 0 = fp16, 1 = bf16
      d.b_lo_base = (uint32_t)(((rows * 16u) >> 4) & 0x3FFFu) << 16;
      d.b_inc = (2u * rows * 16u) >> 4;
      d.lo_off16 = sd.lo_off16;
      d.acc_col = sd.acc_col;
      d.a_off = sd.a_off;
      d.a_lo_off = sd.a_lo_off;
      d.flags_k = (uint32_t)sd.flags | ((uint32_t)sd.ksteps << 16) | ((uint32_t)sd.a_kind << 24);
    }
  }

  // The end of every build: `ok` = every step was added; `name` names the program in the error texts.
  int finish(bool ok, const char* name) {
    what = name;
    if (!ok) return set_error(PNR_ERR_UNSUPPORTED, "%s: program build failed: %s", what, err.c_str());
    if ((int)plan.cpos.size() > kMaxConsts)
      return set_error(PNR_ERR_UNSUPPORTED, "%s: %d constants > %d", what, (int)plan.cpos.size(), kMaxConsts);
    prog.n_consts = (int)plan.cpos.size();
    finalize();
    return PNR_OK;
  }
};

// The feature_linear fold, V's derived block: the folded view matrix [W/2, W+Ed], then the folded bias [W/2].
// feature_linear has no activation, so it is folded into the view layer (exact algebra, done in double):
//   W_view [feat ; gamma(d)] + b_view  with  feat = W_feat h + b_feat
//   = (W_view[:, :W] W_feat) h + W_view[:, W:] gamma(d) + (W_view[:, :W] b_feat + b_view).
// One 256x256 GEMM per sample (11 % of the MLP) and its epilogue disappear; the view step reads the trunk output h
// directly.  Positions in V of the tensors it reads and of the block it writes:
struct Fold {
  int64_t view_w, view_b, feat_w, feat_b, out;
  int W, Ed;
};

// Element (n, k) of [W/2, W + Ed + 1]: k < W the folded matrix, k < W + Ed a gamma(d) column of W_view, k = W + Ed the
// folded bias.  Double sums, j ascending: host (host_v) and device (fold_kernel) fold bit-identically with it.
__host__ __device__ inline void fold_element(float* V, const Fold& f, int n, int k) {
  const float* vrow = V + f.view_w + (int64_t)n * (f.W + f.Ed);
  if (k < f.W) {
    double acc = 0.0;
    for (int j = 0; j < f.W; ++j) acc += (double)vrow[j] * (double)V[f.feat_w + (int64_t)j * f.W + k];
    V[f.out + (int64_t)n * (f.W + f.Ed) + k] = (float)acc;
  } else if (k < f.W + f.Ed) {
    V[f.out + (int64_t)n * (f.W + f.Ed) + k] = vrow[k];
  } else {
    double acc = (double)V[f.view_b + n];
    for (int j = 0; j < f.W; ++j) acc += (double)vrow[j] * (double)V[f.feat_b + j];
    V[f.out + (int64_t)(f.W / 2) * (f.W + f.Ed) + n] = (float)acc;
  }
}

// The fold of tensors laid out by `v_off` (all taken; list order: trunk (w, b) x D, alpha, feature, view, rgb, heads)
Fold fold_of(const pnr_config& c, const std::vector<int64_t>& v_off) {
  const int D = c.D;
  return Fold{v_off[2 * D + 4], v_off[2 * D + 5], v_off[2 * D + 2], v_off[2 * D + 3], v_off.back(), c.W, 3 + 6 * c.view_res};
}

// V on the host, from the tensors a build took: them, concatenated, then - for a forward program - the derived block.
std::vector<float> host_v(const pnr_config& c, const float* const* t, const std::vector<int64_t>& v_off, bool derived) {
  const int W2 = c.W / 2, Ed = 3 + 6 * c.view_res;
  std::vector<float> V((size_t)v_off.back() + (derived ? (size_t)W2 * (c.W + Ed + 1) : 0));
  for (size_t i = 0; i + 1 < v_off.size(); ++i) memcpy(V.data() + v_off[i], t[i], (v_off[i + 1] - v_off[i]) * 4);
  if (derived) {
    const Fold f = fold_of(c, v_off);
    for (int n = 0; n < W2; ++n)
      for (int k = 0; k <= c.W + Ed; ++k) fold_element(V.data(), f, n, k);
  }
  return V;
}

// A plan applied to V on the host (the device twin: pack_from_plan_kernel, consts_from_plan_kernel).  In the fp16
// modes a packed weight outside the fp16 range - after the fold - is refused.
int pack_host(const Builder& bld, const std::vector<float>& V, std::vector<uint16_t>& w, std::vector<float>& consts) {
  const Plan& pl = bld.plan;
  w.resize(pl.wpos.size());
  bool out_of_fp16_range = false;
  for (size_t p = 0; p < w.size(); ++p) {
    const float v = pl.wpos[p] < 0 ? 0.f : V[pl.wpos[p]];
    out_of_fp16_range |= !(v >= -65504.f && v <= 65504.f);   // also catches NaN
    w[p] = weight_part16(v, pl.wpart[p], bld.fmt);
  }
  if (out_of_fp16_range && bld.fmt == kFmtF16)
    return set_error(PNR_ERR_UNSUPPORTED, "%s: a weight is outside the fp16 range (|w| > 65504 or not finite): use "
                     "precision bf16x3", bld.what);
  consts.resize(pl.cpos.size());
  for (size_t c = 0; c < consts.size(); ++c) consts[c] = pl.cpos[c] < 0 ? 0.f : V[pl.cpos[c]];
  return PNR_OK;
}

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// A segment that reads columns [col0, col0 + k) of m against the activation operand columns a_hi / a_lo
Seg seg_tmem(const Mat& m, int col0, int k, int a_hi = kColAHi, int a_lo = kColALo) {
  return Seg{A_TMEM, m, col0, k, round_up(k, 16), a_hi, a_lo, false};
}


}  // namespace

extern "C" int pnr_version(void) { return PNR_VERSION; }
extern "C" const char* pnr_last_error(void) { return g_err; }
extern "C" int64_t pnr_launch_count(int32_t reset) {
  const int64_t v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

static int precision_passes(int precision) {
  return (precision == PNR_PREC_BF16X3 || precision == PNR_PREC_FP16X3) ? 3 : 1;
}
static int precision_fmt(int precision) {   // instruction-descriptor operand format: 0 = fp16, 1 = bf16
  return (precision == PNR_PREC_BF16X3 || precision == PNR_PREC_BF16) ? 1 : 0;
}

static bool is_hashgrid(const pnr_config& c) { return c.xyz_encoding == PNR_XYZ_HASHGRID; }

// Width of the trunk input (layer 0 and the skip layer's first columns): gamma(x) or the hash-grid features h(x)
static int trunk_input_width(const pnr_config& c) {
  return is_hashgrid(c) ? c.hash_levels * c.hash_features : 3 + 6 * c.xyz_res;
}

// K of the embedding operand the MMAs read: gamma(x)'s 63 columns padded to 64 (the whole region), h(x)'s E columns to
// a multiple of 16 (zero weight columns; the prologue writes zeros there)
static int trunk_input_kpad(const pnr_config& c) {
  return is_hashgrid(c) ? (trunk_input_width(c) + 15) / 16 * 16 : 64;
}

static int check_config(const pnr_config* cfg) {
  PNR_CHECK_ARG(cfg->D >= 3 && cfg->D <= 16, "pnr_create: D=%d outside [3,16]", cfg->D);
  PNR_CHECK_ARG(cfg->W == 64 || cfg->W == 128 || cfg->W == 256, "pnr_create: W=%d not in {64,128,256}", cfg->W);
  PNR_CHECK_ARG(cfg->xyz_res >= 0 && cfg->xyz_res <= 10, "pnr_create: xyz_res=%d outside [0,10]", cfg->xyz_res);
  PNR_CHECK_ARG(cfg->view_res >= 0 && cfg->view_res <= 4, "pnr_create: view_res=%d outside [0,4]", cfg->view_res);
  PNR_CHECK_ARG(cfg->num_classes >= 0 && cfg->num_classes <= 128, "pnr_create: num_classes=%d outside [0,128]", cfg->num_classes);
  PNR_CHECK_ARG(cfg->num_instances >= 0 && cfg->num_instances <= 128, "pnr_create: num_instances=%d outside [0,128]", cfg->num_instances);
  PNR_CHECK_ARG(cfg->precision >= 0 && cfg->precision <= 3, "pnr_create: bad precision %d", cfg->precision);
  PNR_CHECK_ARG(cfg->xyz_encoding == PNR_XYZ_FREQUENCY || cfg->xyz_encoding == PNR_XYZ_HASHGRID,
                "pnr_create: bad xyz_encoding %d", cfg->xyz_encoding);
  if (is_hashgrid(*cfg)) {   // the checks of pnr_hashgrid_encode, and the features must fit the 64-K embedding operand
    const int L = cfg->hash_levels, F = cfg->hash_features;
    PNR_CHECK_ARG(L >= 1 && L <= kHashMaxLevels && (F == 1 || F == 2 || F == 4 || F == 8),
                  "pnr_create: hash_levels=%d hash_features=%d (levels in [1,32], features in {1,2,4,8})", L, F);
    PNR_CHECK_ARG(L * F <= 64, "pnr_create: hash-grid features E=%d > 64 (hash_levels * hash_features)", L * F);
    PNR_CHECK_ARG(cfg->hash_log2_size >= 4 && cfg->hash_log2_size <= 28, "pnr_create: hash_log2_size=%d outside [4,28]",
                  cfg->hash_log2_size);
    PNR_CHECK_ARG(cfg->hash_base_resolution >= 1.0f && cfg->hash_per_level_scale >= 1.0f,
                  "pnr_create: hash_base_resolution / hash_per_level_scale < 1");
    PNR_CHECK_ARG((double)cfg->hash_base_resolution * pow((double)cfg->hash_per_level_scale, (double)(L - 1)) < 1048576.0,
                  "pnr_create: hash-grid finest resolution >= 2^20");
    for (int d = 0; d < 3; ++d)
      PNR_CHECK_ARG(cfg->hash_aabb[3 + d] > cfg->hash_aabb[d] && cfg->hash_aabb[3 + d] - cfg->hash_aabb[d] < 3.0e38f,
                    "pnr_create: hash_aabb axis %d: hi must exceed lo (a hash-grid network needs its aabb)", d);
  }
  return PNR_OK;
}

extern "C" int pnr_create(const pnr_config* cfg, pnr_ctx** out) {
  PNR_CHECK_ARG(cfg && out, "pnr_create: null pointer");
  if (const int rc = check_config(cfg)) return rc;
  int ndev = 0;
  PNR_CUDA(cudaGetDeviceCount(&ndev));
  PNR_CHECK_ARG(cfg->device >= 0 && cfg->device < ndev, "pnr_create: device %d of %d", cfg->device, ndev);
  cudaDeviceProp prop;
  PNR_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)
    return set_error(PNR_ERR_UNSUPPORTED, "pnr_create: device %d is sm_%d%d; libpnr is sm_90a only (no fallback path)",
                     cfg->device, prop.major, prop.minor);
  PNR_CHECK_ARG(cfg->device < kMaxDevices, "pnr_create: device ordinal %d >= %d", cfg->device, kMaxDevices);
  DeviceGuard guard(cfg->device);   // the caller's current device is restored on return
  pnr_ctx* c = new pnr_ctx();
  c->cfg = *cfg;
  c->passes = precision_passes(cfg->precision);
  c->fmt = precision_fmt(cfg->precision);
  if (is_hashgrid(*cfg)) hash_level_resolutions(cfg->hash_levels, cfg->hash_base_resolution, cfg->hash_per_level_scale, c->hash_res);
  cudaError_t e = cudaMalloc(&c->d_status, sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMemset(c->d_status, 0, sizeof(uint32_t));
  if (e != cudaSuccess) {
    delete c;
    return set_error(PNR_ERR_CUDA, "pnr_create: status word: %s", cudaGetErrorString(e));
  }
  *out = c;
  return PNR_OK;
}

// Frees the program's device buffers and forgets it (plain cudaFree: it synchronises with the device, so no launch still
// reads them).
static void release(PackedProgram& pp) {
  cudaFree(pp.d_wpacked);
  cudaFree(pp.d_consts);
  cudaFree(pp.d_widx);
  cudaFree(pp.d_wpart);
  cudaFree(pp.d_cidx);
  pp = PackedProgram();
}

extern "C" int pnr_destroy(pnr_ctx* ctx) {
  if (!ctx) return PNR_OK;
  DeviceGuard guard(ctx->cfg.device);
  for (PackedProgram& pp : ctx->prog) release(pp);
  cudaFree(ctx->d_V);
  cudaFree(ctx->d_status);
  delete ctx;
  return PNR_OK;
}

// Sticky status of the fused MLP launches enqueued so far on `stream` (synchronises that stream): bit 0 = a value
// written into a 16-bit operand rounded to inf (fp16 modes: |x| >= 65520) or was NaN (include/pnr.h) - the
// results of that launch are not trustworthy; re-run with PNR_PREC_BF16X3.  reset != 0 clears the word.
extern "C" int pnr_status(pnr_ctx* ctx, uint32_t* status_host, int32_t reset, void* stream) {
  PNR_CHECK_ARG(ctx && status_host, "pnr_status: null pointer");
  DeviceGuard guard(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  PNR_CUDA(cudaMemcpyAsync(status_host, ctx->d_status, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  if (reset) PNR_CUDA(cudaMemsetAsync(ctx->d_status, 0, sizeof(uint32_t), st));
  PNR_CUDA(cudaStreamSynchronize(st));
  return PNR_OK;
}

// The trunk layers of a network: weight [W, in] and bias [W] of layers 0..D-1, the first 2*D tensors of
// pnr_load_weights' list.  Layer 0 reads the trunk input, the skip layer D/2 + 1 [trunk input ; h].
struct Trunk {
  std::vector<Mat> w;
  std::vector<int32_t> b;   // first position in V
};

static int take_trunk(const pnr_config& c, const float* const* t, const int64_t* shapes, const char* what, Builder& bld,
                      Trunk& tr) {
  const int D = c.D, W = c.W, Ex = trunk_input_width(c), skip = D / 2;
  tr.w.resize(D);
  tr.b.resize(D);
  for (int i = 0; i < D; ++i) {
    const int in = i == 0 ? Ex : (i == skip + 1 ? W + Ex : W);
    if (shapes[4 * i] != W || shapes[4 * i + 1] != in || shapes[4 * i + 2] != W || shapes[4 * i + 3] != 1 || !t[2 * i] ||
        !t[2 * i + 1])
      return set_error(PNR_ERR_ARG, "%s: tensor %d: expected weight [%d,%d] + bias [%d,1]", what, 2 * i, W, in, W);
    tr.w[i] = Mat{bld.take_tensor(shapes, 2 * i), W, in};
    tr.b[i] = bld.take_tensor(shapes, 2 * i + 1);
  }
  return PNR_OK;
}

// Steps 0..D-1 of a program, the trunk's forward layers: ReLU activations into the A operand columns, the last layer's
// epilogue `last_kind`.  sigma_w_off >= 0: the last layer also accumulates the sigma head, whose weights are at that
// constant offset.  slots: layer i keeps what its epilogue produces in stash slot i (H_i; dZ_{D-1} for the last layer)
// and, below the last, its sign pattern in slot i - the backward program's forward half.
static bool add_trunk_steps(const pnr_config& c, const Trunk& tr, uint8_t last_kind, int sigma_w_off, bool slots,
                            Builder& bld) {
  const int D = c.D, W = c.W, Ex = trunk_input_width(c), Ekpad = trunk_input_kpad(c), skip = D / 2;
  bld.prog.Lx = is_hashgrid(c) ? 0 : c.xyz_res;
  bld.prog.Ld = c.view_res;
  bld.prog.passes = bld.passes;
  for (int i = 0; i < D; ++i) {
    EpiDesc ed{};
    ed.kind = i == D - 1 ? last_kind : EPI_RELU_TO_A;
    if (sigma_w_off >= 0) {
      ed.sigma = i == D - 1 ? 1 : 0;
      ed.aux_off = (uint16_t)sigma_w_off;
    }
    if (slots) {
      ed.n_valid = i == D - 1 ? 0 : (uint16_t)(i + 1);   // sign-pattern slot + 1
      ed.out_off1 = (uint16_t)(i + 1);                   // stash slot + 1: H_i, or dZ_{D-1} for i = D-1
    }
    ed.dst_col = kColAHi;
    ed.dst_lo_col = kColALo;
    ed.bias_off = (uint16_t)bld.add_consts(tr.b[i], W, W);
    std::vector<Seg> segs;
    if (i == 0) {
      segs.push_back(Seg{A_EMB, tr.w[i], 0, Ex, Ekpad, 0, 0, false});
    } else if (i == skip + 1) {
      segs.push_back(Seg{A_EMB, tr.w[i], 0, Ex, Ekpad, 0, 0, true});
      segs.push_back(seg_tmem(tr.w[i], Ex, W));
    } else {
      segs.push_back(seg_tmem(tr.w[i], 0, W));
    }
    if (!bld.add_step(segs, W, kColAcc, ed, i == 0)) return false;
  }
  return true;
}

// Host only (no CUDA call): checks the tensor list against cfg, builds the per-tile program and its plan.  Shared by
// pnr_load_weights and pnr_program_host.
static int build_program(const pnr_config& c, const float* const* t, const int64_t* shapes, int32_t n,
                         Builder& bld) {
  const int D = c.D, W = c.W, W2 = W / 2, C = c.num_classes, K = c.num_instances, Ed = 3 + 6 * c.view_res;
  const int expected = 2 * D + 8 + (C > 0 ? 4 : 0) + (K > 0 ? 4 : 0);
  PNR_CHECK_ARG(n == expected, "pnr_load_weights: got %d tensors, expected %d", n, expected);
  Trunk trunk;
  if (const int rc = take_trunk(c, t, shapes, "pnr_load_weights", bld, trunk)) return rc;
  int ti = 2 * D;
  auto take = [&](int out, int in, Mat* m, int32_t* bias) -> bool {
    if (shapes[2 * ti] != out || shapes[2 * ti + 1] != in) return false;
    if (shapes[2 * ti + 2] != out || shapes[2 * ti + 3] != 1) return false;
    if (!t[ti] || !t[ti + 1]) return false;
    *m = Mat{bld.take_tensor(shapes, ti), out, in};
    *bias = bld.take_tensor(shapes, ti + 1);
    ti += 2;
    return true;
  };
#define PNR_TAKE(out, in, m, b)                                                                        \
  if (!take(out, in, m, b))                                                                            \
    return set_error(PNR_ERR_ARG, "pnr_load_weights: tensor %d: expected weight [%d,%d] + bias [%d,1]", \
                     ti, out, in, out)
  Mat m_sig, m_feat, m_view, m_rgb, m_s1, m_s2, m_i1, m_i2;
  int32_t b_sig, b_feat, b_view, b_rgb, b_s1 = -1, b_s2 = -1, b_i1 = -1, b_i2 = -1;
  PNR_TAKE(1, W, &m_sig, &b_sig);
  PNR_TAKE(W, W, &m_feat, &b_feat);
  PNR_TAKE(W2, W + Ed, &m_view, &b_view);
  PNR_TAKE(3, W2, &m_rgb, &b_rgb);
  if (C > 0) { PNR_TAKE(W2, W, &m_s1, &b_s1); PNR_TAKE(C, W2, &m_s2, &b_s2); }
  if (K > 0) { PNR_TAKE(W2, W, &m_i1, &b_i1); PNR_TAKE(K, W2, &m_i2, &b_i2); }
#undef PNR_TAKE

  const int sig_w_off = bld.add_consts(m_sig.first, W, W);
  bld.prog.sigma_bias_off = bld.add_consts(b_sig, 1, 4);
  const int rgb_w_off = bld.add_consts(m_rgb.first, 3 * W2, 3 * W2);
  bld.prog.rgb_bias_off = bld.add_consts(b_rgb, 3, 4);

  bool ok = add_trunk_steps(c, trunk, EPI_RELU_TO_A, sig_w_off, false, bld);
  // the view step reads the fold (Fold): V's derived block, after the last tensor
  const int32_t fold_first = (int32_t)bld.v_off.back();
  const Mat m_fold{fold_first, W2, W + Ed};
  auto add_view = [&](int acc_col) {  // view branch [h, gamma(d)] -> relu -> rgb (CUDA cores) ; writes rgb + sigma
    EpiDesc ed{};
    ed.kind = EPI_VIEW_RGB;
    ed.bias_off = (uint16_t)bld.add_consts(fold_first + W2 * (W + Ed), W2, W2);
    ed.aux_off = (uint16_t)rgb_w_off;
    std::vector<Seg> segs;
    segs.push_back(seg_tmem(m_fold, 0, W, kColAHi, kColALo));
    segs.push_back(Seg{A_DIR, m_fold, W, Ed, 32, 0, 0, true});
    // (Accumulating the view step in the UPPER half of the accumulator region, so that the next tile's first layer
    // can be issued right behind the view MMAs, was measured: the stall only moves in front of the view step -
    // the tile boundary is bound by the serial epilogues of view + layer 0, 71.6 k vs 71.9 k cycles per tile.)
    // ONE N = W/2 half: as two N = 64 halves the view step's 108 MMAs cost ~66 cycles each for half the columns
    // (an M=128 N=64 K=16 MMA is no faster than 0.84 of an N=128 one: profiles/r01_mma_rate_probe.log) - 7-8 k cycles
    // of tensor pipe at the one place of the tile where nothing else can be issued.  What the halves bought, the view
    // epilogue's first part overlapping the second half's MMAs, is worth less than that.
    ok = ok && bld.add_step(segs, W2, acc_col, ed, false, nullptr, W2 <= 128 ? W2 : 0);
  };
  // heads: hidden layer -> logits
  auto add_head = [&](const Mat& m1, int32_t b1, const Mat& m2, int32_t b2, int nout, int out_off) {
    EpiDesc e1{};
    e1.kind = EPI_RELU_TO_A;
    e1.dst_col = kColHeadHi;        // head hidden activations (K <= 128) live in the upper half of the
    e1.dst_lo_col = kColHeadLo;     // accumulator region while it is free
    e1.bias_off = (uint16_t)bld.add_consts(b1, W2, W2);
    ok = ok && bld.add_step({seg_tmem(m1, 0, W, kColAHi, kColALo)}, W2, kColAcc, e1, false);
    const int npad = round_up(nout, 16);
    EpiDesc e2{};
    e2.kind = EPI_LOGITS;
    e2.n_valid = (uint16_t)nout;
    e2.out_off = (uint16_t)out_off;
    e2.bias_off = (uint16_t)bld.add_consts(b2, nout, npad);
    ok = ok && bld.add_step({seg_tmem(m2, 0, W2, kColHeadHi, kColHeadLo)}, npad, kColAcc, e2, false);
  };
  if (C > 0 && K > 0 && 2 * W2 == W && W >= 128) {
    // Both heads: the view step runs first (it is the last reader of the trunk output), then ONE W-wide hidden
    // step computes both heads' hidden layers ([W_s1 ; W_i1], ReLU) in place of the trunk activations - a full-size
    // layer at trunk efficiency instead of two N = W/2 steps whose halves are issue-bound - and ONE logits step whose
    // halves are the two (block-diagonal) logit layers, zero blocks skipped: h0 = semantic logits from hidden
    // columns [0, W/2), h1 = instance logits from [W/2, W).  Per tile: 11 steps instead of 13, and the serial chain
    // hidden -> epilogue -> logits -> epilogue runs once, not twice (r2 timeline: ~30 k of a cfg3 tile's ~99 k
    // cycles went into the two head chains for ~10 k cycles of tensor work).
    // (The view step accumulating in the UPPER accumulator half, so that the hidden step's first half can start right
    // behind the view MMAs, was measured on the cfg3 frame: 411.8 vs 408.9 ms - no gain, not kept.)
    add_view(kColAcc);
    std::vector<int32_t> hid_w((size_t)W * W);   // [W_s1 ; W_i1]
    for (int r = 0; r < W; ++r)
      for (int k = 0; k < W; ++k) hid_w[(size_t)r * W + k] = r < W2 ? m_s1.at(r, k) : m_i1.at(r - W2, k);
    const Mat m_hid{0, W, W, hid_w.data()};
    EpiDesc eh{};
    eh.kind = EPI_RELU_TO_A;
    eh.dst_col = kColAHi;
    eh.dst_lo_col = kColALo;
    eh.bias_off = (uint16_t)bld.add_consts(b_s1, W2, W2);
    bld.add_consts(b_i1, W2, W2);                         // contiguous: [b_s1 ; b_i1]
    ok = ok && bld.add_step({seg_tmem(m_hid, 0, W, kColAHi, kColALo)}, W, kColAcc, eh, false);
    const int n_s = round_up(C, 16), n_i = round_up(K, 16);
    EpiDesc el{};
    el.kind = EPI_LOGITS;
    el.n_valid = (uint16_t)C;
    el.out_off = 4;
    el.n_valid1 = (uint16_t)K;
    el.out_off1 = (uint16_t)(4 + C);
    el.bias_off = (uint16_t)bld.add_consts(b_s2, C, n_s);
    bld.add_consts(b_i2, K, n_i);                         // contiguous: bias of column n_s + j
    const std::vector<Seg> seg_i{seg_tmem(m_i2, 0, W2, kColAHi + W2 / 2, kColALo + W2 / 2)};
    ok = ok && bld.add_step({seg_tmem(m_s2, 0, W2, kColAHi, kColALo)}, n_s + n_i, kColAcc, el, false, &seg_i, n_s);
  } else {
    if (ok && C > 0) add_head(m_s1, b_s1, m_s2, b_s2, C, 4);
    if (ok && K > 0) add_head(m_i1, b_i1, m_i2, b_i2, K, 4 + C);
    add_view(kColAcc);
  }
  return bld.finish(ok, "pnr_load_weights");
}

// Backward program of the trunk (mlp_program.h, "BACKWARD"): t / shapes = the trunk's weight, bias pairs (the first
// 2*D tensors of pnr_load_weights' list).  Forward steps 0..D-1 (sign patterns kept, the last one loads the incoming
// gradient), then for l = D-1..0 the gradient w.r.t. layer l's input: g_l [128, W] x W_l [W, in_l], i.e. a step whose
// weight matrix is W_l transposed; the embedded-input columns of layer 0 and of the skip layer go to the output rows.
// forward_only: just the trunk, whose last layer writes its activations to the output rows (EPI_ACT_OUT).
// Stash slots (MlpParams::stash): H_i of forward layer i < D-1 in slot i; the pre-activation gradient dZ_j in slot
// 2D-2-j (the order they are produced in: dZ_{D-1} by the last forward layer's epilogue, then D-2 .. 0).
static int build_backward_program(const pnr_config& c, const float* const* t, const int64_t* shapes, int32_t n,
                                  Builder& bld, bool forward_only = false) {
  const int D = c.D, W = c.W, Ex = trunk_input_width(c), Ekpad = trunk_input_kpad(c), skip = D / 2;
  PNR_CHECK_ARG(n >= 2 * D, "backward program: got %d tensors, the trunk has %d", n, 2 * D);
  if (bld.passes != 3)
    return set_error(PNR_ERR_UNSUPPORTED, "backward program: precision must be fp16x3 or bf16x3");
  if (D - 1 > kMaxMaskSlots)
    return set_error(PNR_ERR_UNSUPPORTED, "backward program: D=%d needs %d sign-pattern slots, %d fit", D, D - 1, kMaxMaskSlots);
  Trunk trunk;
  if (const int rc = take_trunk(c, t, shapes, "backward program", bld, trunk)) return rc;
  bool ok = add_trunk_steps(c, trunk, forward_only ? EPI_ACT_OUT : EPI_LOADG_TO_A, -1, !forward_only, bld);
  std::vector<int32_t> wt;   // W_l transposed: [in_l, W] row-major (packed inside add_step, so one buffer serves all)
  for (int l = forward_only ? -1 : D - 1; l >= 0 && ok; --l) {
    const int in = trunk.w[l].in;
    wt.assign((size_t)in * W, 0);
    for (int o = 0; o < W; ++o)
      for (int k = 0; k < in; ++k) wt[(size_t)k * W + o] = trunk.w[l].at(o, k);
    auto grad_out = [&](const int32_t* rows, bool accumulate) {  // embedded-input columns -> output rows
      EpiDesc eo{};
      eo.kind = EPI_GRAD_OUT;
      eo.n_valid = (uint16_t)Ex;
      eo.n_valid1 = accumulate ? 1 : 0;
      eo.out_off = 0;
      // one N = Ekpad half: two N = 32 halves would double the MMA count for the same tensor time per MMA
      return bld.add_step({seg_tmem(Mat{0, Ex, W, rows}, 0, W)}, Ekpad, kColAcc, eo, false, nullptr, Ekpad);
    };
    auto grad_h = [&](const int32_t* rows) {                     // hidden columns, gated by layer l-1's sign pattern
      EpiDesc em{};
      em.kind = EPI_MASK_TO_A;
      em.n_valid = (uint16_t)l;                                  // slot (l - 1) + 1
      em.out_off1 = (uint16_t)(2 * D - 2 - (l - 1) + 1);          // stash slot + 1 of dZ_{l-1}
      em.dst_col = kColAHi;
      em.dst_lo_col = kColALo;
      return bld.add_step({seg_tmem(Mat{0, W, W, rows}, 0, W)}, W, kColAcc, em, false);
    };
    if (l == 0) {
      ok = grad_out(wt.data(), true);
    } else if (l == skip + 1) {   // input = [embedded xyz ; h]: the embedded part first (the next step overwrites g_l)
      ok = grad_out(wt.data(), false) && grad_h(wt.data() + (size_t)Ex * W);
    } else {
      ok = grad_h(wt.data());
    }
  }
  return bld.finish(ok, "backward program");
}

// Program `kind` of a network, from the tensors of pnr_load_weights' list (the backward and trunk-forward programs read
// the trunk's only).
static int build_program_kind(ProgramKind kind, const pnr_config& c, const float* const* t, const int64_t* shapes,
                              int32_t n, Builder& bld) {
  return kind == kProgForward ? build_program(c, t, shapes, n, bld)
                              : build_backward_program(c, t, shapes, n, bld, kind == kProgTrunkForward);
}

// Gives the program the builder's program and plan, and device buffers for the stream and constants the caller packs.
static int place(PackedProgram& pp, Builder& bld) {
  release(pp);
  pp.n_w = bld.plan.wpos.size();
  pp.n_c = bld.plan.cpos.size();
  PNR_CUDA(cudaMalloc(&pp.d_wpacked, pp.n_w * 2));
  PNR_CUDA(cudaMalloc(&pp.d_consts, pp.n_c * 4));
  pp.launch.prog = bld.prog;
  pp.plan = std::move(bld.plan);
  return PNR_OK;
}

extern "C" int pnr_load_weights(pnr_ctx* ctx, const float* const* t, const int64_t* shapes, int32_t n) {
  PNR_CHECK_ARG(ctx && t && shapes, "pnr_load_weights: null pointer");
  const pnr_config& c = ctx->cfg;
  Builder bld(ctx->passes, ctx->fmt);
  if (const int rc = build_program(c, t, shapes, n, bld)) return rc;
  const std::vector<float> V = host_v(c, t, bld.v_off, true);
  std::vector<uint16_t> w;
  std::vector<float> consts;
  if (const int rc = pack_host(bld, V, w, consts)) return rc;
  DeviceGuard guard(c.device);
  ctx->loaded = false;
  for (PackedProgram& pp : ctx->prog) release(pp);   // the backward and trunk-forward programs follow on first use
  cudaFree(ctx->d_V);
  ctx->d_V = nullptr;
  ctx->v_off = bld.v_off;
  ctx->shapes.assign(shapes, shapes + 2 * n);
  PackedProgram& pp = ctx->prog[kProgForward];
  if (const int rc = place(pp, bld)) return rc;
  PNR_CUDA(cudaMalloc(&ctx->d_V, V.size() * 4));
  PNR_CUDA(cudaMemcpy(ctx->d_V, V.data(), V.size() * 4, cudaMemcpyHostToDevice));
  PNR_CUDA(cudaMemcpy(pp.d_wpacked, w.data(), pp.n_w * 2, cudaMemcpyHostToDevice));
  PNR_CUDA(cudaMemcpy(pp.d_consts, consts.data(), pp.n_c * 4, cudaMemcpyHostToDevice));
  pp.ready = true;
  ctx->loaded = true;
  return PNR_OK;
}

extern "C" int pnr_program_host(const pnr_config* cfg, const float* const* t, const int64_t* shapes, int32_t n,
                                int32_t flags, void* program, size_t program_cap, size_t* program_bytes, void* wpacked,
                                size_t wpacked_cap, size_t* wpacked_bytes, float* consts, size_t consts_cap,
                                size_t* n_consts) {
  PNR_CHECK_ARG(cfg && t && shapes && program_bytes && wpacked_bytes && n_consts, "pnr_program_host: null pointer");
  if (const int rc = check_config(cfg)) return rc;
  PNR_CHECK_ARG((flags & ~(PNR_PROGRAM_SPLIT_E1 | PNR_PROGRAM_NO_SPLIT | PNR_PROGRAM_BACKWARD | PNR_PROGRAM_VIEW_PRODUCERS)) == 0,
                "pnr_program_host: unknown flags 0x%x", flags);
  Builder bld(precision_passes(cfg->precision), precision_fmt(cfg->precision));
  if (flags & PNR_PROGRAM_NO_SPLIT) bld.split_e1 = false;
  if (flags & PNR_PROGRAM_SPLIT_E1) bld.split_e1 = true;
  if (flags & PNR_PROGRAM_VIEW_PRODUCERS) bld.view_on_producers = true;
  const ProgramKind kind = (flags & PNR_PROGRAM_BACKWARD) ? kProgBackward : kProgForward;
  if (const int rc = build_program_kind(kind, *cfg, t, shapes, n, bld)) return rc;
  std::vector<uint16_t> w;
  std::vector<float> cst;
  if (const int rc = pack_host(bld, host_v(*cfg, t, bld.v_off, kind == kProgForward), w, cst)) return rc;
  *program_bytes = sizeof(MlpProgram);
  *wpacked_bytes = w.size() * 2;
  *n_consts = cst.size();
  if (program) {
    PNR_CHECK_ARG(program_cap >= sizeof(MlpProgram), "pnr_program_host: program buffer too small");
    memcpy(program, &bld.prog, sizeof(MlpProgram));
  }
  if (wpacked) {
    PNR_CHECK_ARG(wpacked_cap >= *wpacked_bytes, "pnr_program_host: weight buffer too small");
    memcpy(wpacked, w.data(), *wpacked_bytes);
  }
  if (consts) {
    PNR_CHECK_ARG(consts_cap >= *n_consts, "pnr_program_host: constant buffer too small");
    memcpy(consts, cst.data(), *n_consts * 4);
  }
  return PNR_OK;
}

extern "C" int pnr_bind_hashgrid_table(pnr_ctx* ctx, const float* table) {
  PNR_CHECK_ARG(ctx, "pnr_bind_hashgrid_table: null context");
  if (!is_hashgrid(ctx->cfg)) return set_error(PNR_ERR_STATE, "pnr_bind_hashgrid_table: not a hash-grid context");
  PNR_CHECK_ARG(!table || hash_table_aligned(table, ctx->cfg.hash_features),
                "pnr_bind_hashgrid_table: table not aligned to its %d features (a float%d per corner)",
                ctx->cfg.hash_features, ctx->cfg.hash_features);
  ctx->hash_table = table;
  return PNR_OK;
}

// The trunk-input fields of a launch: a hash-grid context's table and level constants, or none (gamma(x)).
static int set_trunk_input(const pnr_ctx* ctx, MlpParams& p, const char* what) {
  p.hash_table = nullptr;
  if (!is_hashgrid(ctx->cfg)) return PNR_OK;
  if (ctx->hash_table == nullptr)
    return set_error(PNR_ERR_STATE, "%s: hash-grid network without a table (pnr_bind_hashgrid_table)", what);
  const pnr_config& c = ctx->cfg;
  p.hash_table = ctx->hash_table;
  p.hash_L = c.hash_levels; p.hash_F = c.hash_features; p.hash_T_log2 = c.hash_log2_size;
  memcpy(p.hash_aabb, c.hash_aabb, sizeof(p.hash_aabb));
  memcpy(p.hash_res, ctx->hash_res, sizeof(p.hash_res));
  return PNR_OK;
}

static int ensure_program(pnr_ctx* ctx, ProgramKind kind, cudaStream_t st);   // below, with the device-side updates

// The checks every fused-MLP launch makes, and the fields every launch of program `kind` sets: its packed stream and
// constants (built on first use), sample source, sizes, status word and trunk input.  The rest of the launch's
// MlpParams is zero: each entry point sets its own fields.  Needs the context's device current.
static int prepare_launch(pnr_ctx* ctx, ProgramKind kind, const char* what, const float* pts, const float* viewdirs,
                          const float* rays, const float* z, int64_t R, int32_t N, cudaStream_t st, MlpLaunch** out) {
  if (!ctx->loaded) return set_error(PNR_ERR_STATE, "%s: pnr_load_weights has not been called", what);
  PNR_CHECK_ARG(R > 0 && N >= 1, "%s: bad sizes R=%lld N=%d", what, (long long)R, N);
  if (const int rc = ensure_program(ctx, kind, st)) return rc;
  PackedProgram& pp = ctx->prog[kind];
  MlpParams& p = pp.launch.p;
  memset(&p, 0, sizeof(p));
  p.wpacked = pp.d_wpacked; p.consts = pp.d_consts;
  p.pts = pts; p.viewdirs = viewdirs; p.rays = rays; p.z = z;
  p.S = R * (int64_t)N; p.N = N;
  p.status = ctx->d_status;
  *out = &pp.launch;
  return set_trunk_input(ctx, p, what);
}

extern "C" int pnr_mlp_forward(pnr_ctx* ctx, const float* pts, const float* viewdirs, const float* rays,
                               const float* z, int64_t R, int32_t N, float* raw, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(ctx && raw, "pnr_mlp_forward: null pointer");
  PNR_CHECK_ARG((pts && viewdirs) || (!pts && rays && z), "pnr_mlp_forward: need (pts, viewdirs) or (rays, z)");
  DeviceGuard guard(ctx->cfg.device);   // launch on the context's device whatever the caller's current one is
  MlpLaunch* L;
  if (const int rc = prepare_launch(ctx, kProgForward, "pnr_mlp_forward", pts, viewdirs, rays, z, R, N,
                                    (cudaStream_t)stream, &L))
    return rc;
  L->p.CH = 4 + ctx->cfg.num_classes + ctx->cfg.num_instances;
  L->p.raw = raw;
  return launch_mlp(*L, ctx->passes, ctx->fmt, kMlpForward, (cudaStream_t)stream);
}

extern "C" int pnr_mlp_composite(pnr_ctx* ctx, const float* rays, const float* z, int64_t R, int32_t N,
                                 int32_t white_bkgd, int32_t mask_outside, const int32_t* sample_box,
                                 const int32_t* box_sem, const int32_t* box_inst, int32_t B,
                                 const pnr_composite_out* out, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(ctx && rays && z && out, "pnr_mlp_composite: null pointer");
  DeviceGuard guard(ctx->cfg.device);
  MlpLaunch* L;
  if (const int rc = prepare_launch(ctx, kProgForward, "pnr_mlp_composite", nullptr, nullptr, rays, z, R, N,
                                    (cudaStream_t)stream, &L))
    return rc;
  if (N % 32 != 0)
    return set_error(PNR_ERR_UNSUPPORTED, "pnr_mlp_composite: N=%d is not a multiple of 32 (use pnr_mlp_forward + pnr_composite)", N);
  PNR_CHECK_ARG(out->weights, "pnr_mlp_composite: out->weights is required");
  PNR_CHECK_ARG(!mask_outside || sample_box, "pnr_mlp_composite: mask_outside needs sample_box");
  const int C = ctx->cfg.num_classes, K = ctx->cfg.num_instances;
  MlpParams& p = L->p;
  p.CH = 4 + C + K;
  p.sample_box = sample_box; p.mask_outside = mask_outside; p.white_bkgd = white_bkgd;
  p.C = C; p.K = K;
  p.weights = out->weights; p.rgb_map = out->rgb_map; p.depth_map = out->depth_map; p.acc_map = out->acc_map;
  p.disp_map = out->disp_map; p.sem_map = C > 0 ? out->semantic_map : nullptr; p.inst_map = K > 0 ? out->instance_map : nullptr;
  if (const int rc = launch_mlp(*L, ctx->passes, ctx->fmt, kMlpComposite, (cudaStream_t)stream)) return rc;
  const bool fs = C > 0 && out->fixed_semantic_map && sample_box && box_sem;
  const bool fi = K > 0 && out->fixed_instance_map && sample_box && box_inst;
  if (fs || fi)
    return launch_fixed_maps(out->weights, sample_box, box_sem, box_inst, R, N, C, K, B,
                             fs ? out->fixed_semantic_map : nullptr, fi ? out->fixed_instance_map : nullptr,
                             (cudaStream_t)stream);
  return PNR_OK;
}

// ------------------------------------------------------------------------------------------------- device-side packing
// A training loop changes the weights every step; re-running the host builder (three programs, ~30 ms each) and
// copying the parameters to the host and back would cost more than the step itself.  So each plan is built once, and
// pnr_update_weights refreshes V from the caller's DEVICE tensors, folds (fold_kernel) and repacks every program with
// the pack / constants kernels: bit-identical to a fresh pnr_load_weights of the same values.
namespace {

__global__ void pack_from_plan_kernel(const float* __restrict__ V, const int32_t* __restrict__ idx,
                                      const uint8_t* __restrict__ part, size_t n, int fmt, uint16_t* __restrict__ out,
                                      uint32_t* status) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const float w = idx[p] < 0 ? 0.f : V[idx[p]];
  if (fmt == kFmtF16 && !(w >= -65504.f && w <= 65504.f) && status != nullptr) atomicOr(status, 2u);   // weight outside the fp16 range
  out[p] = weight_part16(w, part[p], fmt);
}

__global__ void consts_from_plan_kernel(const float* __restrict__ V, const int32_t* __restrict__ idx, size_t n,
                                        float* __restrict__ out) {
  const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = idx[p] < 0 ? 0.f : V[idx[p]];
}

// One thread per element of [W2, W + Ed + 1] (fold_element)
__global__ void fold_kernel(float* V, Fold f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int cols = f.W + f.Ed + 1;
  if (i < f.W / 2 * cols) fold_element(V, f, i / cols, i % cols);
}

}  // namespace

// Packs program `kind`'s stream and constants from V, on `st`; its plan moves to the device the first time.
static int refresh(pnr_ctx* ctx, ProgramKind kind, cudaStream_t st) {
  PackedProgram& pp = ctx->prog[kind];
  if (!pp.plan.wpos.empty()) {
    PNR_CUDA(cudaMalloc(&pp.d_widx, pp.n_w * 4));
    PNR_CUDA(cudaMalloc(&pp.d_wpart, pp.n_w));
    PNR_CUDA(cudaMalloc(&pp.d_cidx, pp.n_c * 4));
    PNR_CUDA(cudaMemcpy(pp.d_widx, pp.plan.wpos.data(), pp.n_w * 4, cudaMemcpyHostToDevice));
    PNR_CUDA(cudaMemcpy(pp.d_wpart, pp.plan.wpart.data(), pp.n_w, cudaMemcpyHostToDevice));
    PNR_CUDA(cudaMemcpy(pp.d_cidx, pp.plan.cpos.data(), pp.n_c * 4, cudaMemcpyHostToDevice));
    pp.plan = Plan();
  }
  pack_from_plan_kernel<<<(unsigned)((pp.n_w + 255) / 256), 256, 0, st>>>(ctx->d_V, pp.d_widx, pp.d_wpart, pp.n_w, ctx->fmt,
                                                                          reinterpret_cast<uint16_t*>(pp.d_wpacked), ctx->d_status);
  PNR_LAUNCH_CHECK("pack_from_plan_kernel");
  consts_from_plan_kernel<<<(unsigned)((pp.n_c + 255) / 256), 256, 0, st>>>(ctx->d_V, pp.d_cidx, pp.n_c, pp.d_consts);
  PNR_LAUNCH_CHECK("consts_from_plan_kernel");
  return PNR_OK;
}

extern "C" int pnr_update_weights(pnr_ctx* ctx, const float* const* device_tensors, int32_t n, void* stream) {
  PNR_CHECK_ARG(ctx && device_tensors, "pnr_update_weights: null pointer");
  if (!ctx->loaded) return set_error(PNR_ERR_STATE, "pnr_update_weights: pnr_load_weights has not been called (it fixes the shapes)");
  const int n_loaded = (int)ctx->v_off.size() - 1;
  PNR_CHECK_ARG(n == n_loaded, "pnr_update_weights: got %d tensors, pnr_load_weights had %d", n, n_loaded);
  for (int i = 0; i < n; ++i) PNR_CHECK_ARG(device_tensors[i], "pnr_update_weights: tensor %d is null", i);
  DeviceGuard guard(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n; ++i)
    PNR_CUDA(cudaMemcpyAsync(ctx->d_V + ctx->v_off[i], device_tensors[i], (size_t)(ctx->v_off[i + 1] - ctx->v_off[i]) * 4,
                             cudaMemcpyDeviceToDevice, st));
  const Fold f = fold_of(ctx->cfg, ctx->v_off);
  fold_kernel<<<(f.W / 2 * (f.W + f.Ed + 1) + 127) / 128, 128, 0, st>>>(ctx->d_V, f);
  PNR_LAUNCH_CHECK("fold_kernel");
  // the programs that exist follow; the others are packed from V when they are first built
  for (int k = 0; k < kNumPrograms; ++k)
    if (ctx->prog[k].ready)
      if (const int rc = refresh(ctx, (ProgramKind)k, st)) return rc;
  return PNR_OK;
}

// Program `kind` of a loaded context, built on first use and packed on the device from V.
static int ensure_program(pnr_ctx* ctx, ProgramKind kind, cudaStream_t st) {
  PackedProgram& pp = ctx->prog[kind];
  if (pp.ready) return PNR_OK;   // the forward program always is: pnr_load_weights builds it
  std::vector<const float*> tp(ctx->v_off.size() - 1);   // the loaded tensors, where they sit in V
  for (size_t i = 0; i < tp.size(); ++i) tp[i] = ctx->d_V + ctx->v_off[i];
  Builder bld(ctx->passes, ctx->fmt);
  if (const int rc = build_program_kind(kind, ctx->cfg, tp.data(), ctx->shapes.data(), (int32_t)tp.size(), bld)) return rc;
  if (const int rc = place(pp, bld)) return rc;
  if (const int rc = refresh(ctx, kind, st)) return rc;
  pp.ready = true;
  return PNR_OK;
}

// dL/d(embedded xyz) through the trunk (the tensor-core part of the MLP backward, SURVEY 8f rank 2): the forward
// trunk is recomputed per tile (sign patterns stay in shared memory), then the layers run in reverse on the same tiles
// with the transposed weight stream.  grad_h = dL/dh of the trunk output [R*N, W]; grad_emb [R*N, ld_emb], the first
// trunk_input_width columns of a row are the gradient (ld_emb = trunk_input_kpad with a 16-byte aligned base: vector
// stores).  For a hash-grid context that is dL/dh(x), which pnr_hashgrid_backward turns into the table's gradient.
// stash (nullable) [2D-1, R*N, W] fp32 receives every A operand on the way: H_i (i < D-1) in slot i, the
// pre-activation gradient dZ_j in slot 2D-2-j - the operands of the weight-gradient GEMMs dW_j = dZ_j^T H_{j-1}.
// grad_scale: a power of two the incoming gradient is multiplied by on load (every gradient leaving the kernel is
// divided by it again): gradients of a mean-reduced loss are ~1e-6, far below the normal range of the fp16 operand
// parts; scale so that max |grad_h| * grad_scale is a few hundred (the pass is linear, the scaling exact).
extern "C" int pnr_mlp_backward_trunk(pnr_ctx* ctx, const float* pts, const float* rays, const float* z, int64_t R,
                                      int32_t N, const float* grad_h, float grad_scale, float* grad_emb, int32_t ld_emb,
                                      float* stash, uint32_t* stash_absmax, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(ctx && grad_h && grad_emb, "pnr_mlp_backward_trunk: null pointer");
  PNR_CHECK_ARG(ld_emb >= trunk_input_width(ctx->cfg), "pnr_mlp_backward_trunk: ld_emb=%d < %d columns", ld_emb,
                trunk_input_width(ctx->cfg));
  int gexp = 0;
  PNR_CHECK_ARG(grad_scale > 0.f && grad_scale < 1.0e30f && grad_scale > 1.0e-30f && frexpf(grad_scale, &gexp) == 0.5f,
                "pnr_mlp_backward_trunk: grad_scale=%g must be a positive power of two", (double)grad_scale);
  PNR_CHECK_ARG(stash_absmax == nullptr || stash != nullptr, "pnr_mlp_backward_trunk: stash_absmax without a stash");
  PNR_CHECK_ARG(pts || (rays && z), "pnr_mlp_backward_trunk: need pts or (rays, z)");
  PNR_CHECK_ARG(stash == nullptr || (reinterpret_cast<uintptr_t>(stash) & 15) == 0,
                "pnr_mlp_backward_trunk: stash must be 16-byte aligned");
  DeviceGuard guard(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  MlpLaunch* L;
  if (const int rc = prepare_launch(ctx, kProgBackward, "pnr_mlp_backward_trunk", pts, nullptr, rays, z, R, N, st, &L))
    return rc;
  MlpParams& p = L->p;
  p.CH = ld_emb; p.raw = grad_emb;
  p.grad_in = grad_h;
  p.stash = stash;
  p.stash_absmax = stash_absmax;
  if (stash_absmax != nullptr)
    PNR_CUDA(cudaMemsetAsync(stash_absmax, 0, sizeof(uint32_t) * (size_t)(2 * ctx->cfg.D - 1), st));
  p.grad_scale = grad_scale;
  p.grad_unscale = 1.0f / grad_scale;
  return launch_mlp(*L, ctx->passes, ctx->fmt, kMlpBackward, st);
}

// The trunk's output activations h [R*N, W] (what alpha_linear, feature_linear and the heads read): the forward
// trunk on the same tiles, last layer written out.  The training forward needs it once per step: everything
// after the trunk is differentiated by the caller (torch), everything before it by pnr_mlp_backward_trunk.
extern "C" int pnr_mlp_trunk_forward(pnr_ctx* ctx, const float* pts, const float* rays, const float* z, int64_t R,
                                     int32_t N, float* h_out, void* stream) {
  if (R == 0) return PNR_OK;
  PNR_CHECK_ARG(ctx && h_out, "pnr_mlp_trunk_forward: null pointer");
  PNR_CHECK_ARG((reinterpret_cast<uintptr_t>(h_out) & 15) == 0, "pnr_mlp_trunk_forward: h_out must be 16-byte aligned");
  PNR_CHECK_ARG(pts || (rays && z), "pnr_mlp_trunk_forward: need pts or (rays, z)");
  DeviceGuard guard(ctx->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  MlpLaunch* L;
  if (const int rc = prepare_launch(ctx, kProgTrunkForward, "pnr_mlp_trunk_forward", pts, nullptr, rays, z, R, N, st, &L))
    return rc;
  L->p.CH = ctx->cfg.W; L->p.raw = h_out;
  L->p.grad_scale = L->p.grad_unscale = 1.0f;
  return launch_mlp(*L, ctx->passes, ctx->fmt, kMlpBackward, st);
}

namespace pnr {
size_t workspace_bytes_for(int64_t R, int N, int Ni, int CH);   // render.cu
int ctx_channels(const pnr_ctx* ctx) { return 4 + ctx->cfg.num_classes + ctx->cfg.num_instances; }
int ctx_classes(const pnr_ctx* ctx, int* C, int* K) {
  *C = ctx->cfg.num_classes;
  *K = ctx->cfg.num_instances;
  return PNR_OK;
}
}  // namespace pnr

extern "C" size_t pnr_workspace_bytes(const pnr_ctx* ctx, int64_t R, int32_t N, int32_t Ni) {
  if (!ctx || R <= 0 || N < 1) return 0;
  return workspace_bytes_for(R, N, Ni > 0 ? Ni : 0, ctx_channels(ctx));
}
