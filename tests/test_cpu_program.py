"""CPU tier: the host side of the fused MLP kernel.  `pnr_program_host` (the host-only twin of pnr_load_weights)
builds the per-tile program, the packed 16-bit weight stream and the constant table; this test REPLAYS that
program on the CPU - stage by stage, from the packed bytes, following the same StageDesc / EpiDesc semantics
the kernel interprets - and compares the result with the oracle's Network.forward.  It pins the weight packing
(tile order, hi/lo split, K padding), the feature_linear fold, the skip connection, the head wiring, the bias /
sigma / rgb constant offsets and the hazard-flag invariants without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import reference_renderer as O
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as S
from util import assert_close, rms

K_MAX_STAGES, K_MAX_STEPS = 256, 24
A_TMEM, A_EMB, A_DIR = 0, 1, 2
F_FIRST, F_WAIT_E0, F_WAIT_E1, F_COMMIT_ACC0, F_COMMIT_ACC1, F_COMMIT_WAR = 1, 2, 4, 8, 16, 32
F_WAIT_E1A = 1024
F_COMMIT_VIEW = 2048
PROGRAM_VIEW_PRODUCERS = 32
PROGRAM_SPLIT_E1, PROGRAM_NO_SPLIT = 4, 8
EPI_RELU_TO_A, EPI_VIEW_RGB, EPI_LOGITS = 0, 2, 3
EPI_MASK_TO_A, EPI_LOADG_TO_A, EPI_GRAD_OUT = 4, 5, 6          # backward programs
PROGRAM_BACKWARD = 16
COL_A_HI, COL_HEAD_HI = 256, 128


class StageDesc(C.Structure):
    _fields_ = [("gofs", C.c_uint32), ("bytes", C.c_uint32), ("n", C.c_uint16), ("acc_col", C.c_uint16),
                ("a_off", C.c_uint16), ("a_lo_off", C.c_uint16), ("flags", C.c_uint16), ("lo_off16", C.c_uint16),
                ("ksteps", C.c_uint8), ("a_kind", C.c_uint8)]


class IssueDesc(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("idesc", "b_lo_base", "b_inc", "lo_off16", "acc_col", "a_off", "a_lo_off", "flags_k",
                                          "needs")]


class EpiDesc(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("sigma", C.c_uint8)] + [(k, C.c_uint16) for k in
                ("n", "n0", "n_valid", "acc_col", "dst_col", "dst_lo_col", "bias_off", "aux_off", "out_off", "out_off1", "n_valid1", "n1a")]


class MlpProgram(C.Structure):
    _fields_ = [("n_stages", C.c_int32), ("n_steps", C.c_int32), ("n_consts", C.c_int32),
                ("sigma_bias_off", C.c_int32), ("rgb_bias_off", C.c_int32), ("Lx", C.c_int32), ("Ld", C.c_int32),
                ("passes", C.c_int32), ("acc_flip", C.c_int32), ("view_step", C.c_int32), ("st", StageDesc * K_MAX_STAGES), ("is_", IssueDesc * K_MAX_STAGES),
                ("ep", EpiDesc * K_MAX_STEPS)]


def build(cfg, net, flags: int = 0):
    host, shapes = [], []
    for lin in net._linears():
        w, b = lin.weight.detach().float().contiguous(), lin.bias.detach().float().contiguous()
        host += [w, b]
        shapes += [w.shape[0], w.shape[1], b.shape[0], 1]
    L = _capi.lib()
    pc = _capi.PnrConfig(cfg.D, cfg.W, cfg.xyz_res, cfg.view_res, cfg.num_classes, cfg.num_instances,
                         _capi.PREC[cfg.precision], 0)
    ptrs = (C.c_void_p * len(host))(*[t.data_ptr() for t in host])
    shp = (C.c_int64 * len(shapes))(*shapes)
    pb, wb, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
    _capi.check(L.pnr_program_host(C.byref(pc), ptrs, shp, len(host), flags, None, 0, C.byref(pb), None, 0,
                                   C.byref(wb), None, 0, C.byref(nc)), "pnr_program_host (sizes)")
    assert pb.value == C.sizeof(MlpProgram), "MlpProgram layout in this test is out of date"
    prog = MlpProgram()
    w16 = np.zeros(wb.value // 2, dtype=np.uint16)
    consts = np.zeros(nc.value, dtype=np.float32)
    _capi.check(L.pnr_program_host(C.byref(pc), ptrs, shp, len(host), flags, C.byref(prog), pb.value, C.byref(pb),
                                   w16.ctypes.data, wb.value, C.byref(wb), consts.ctypes.data, nc.value, C.byref(nc)),
                "pnr_program_host")
    return prog, w16, consts


def to_f32(u16: np.ndarray, bf16: bool) -> np.ndarray:
    if bf16:
        return (u16.astype(np.uint32) << 16).view(np.float32)
    return u16.view(np.float16).astype(np.float32)


def split16(x: np.ndarray, bf16: bool):
    """x = hi + lo + residual with both parts rounded to the 16-bit operand format (the kernel's split_x2)."""
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    dt = torch.bfloat16 if bf16 else torch.float16
    hi = t.to(dt).float()
    lo = (t - hi).to(dt).float()
    return hi.double().numpy(), lo.double().numpy()


REPLAY_DEFECTS = ("grad_hi_only", "mask_of_next_layer", "scale_left_in_dz0", "skip_overwritten")


def replay(prog, w16, consts, cfg, pts, viewdirs, operand_precision: bool = False, grad_in=None, emb_x=None,
           grad_scale: float = 1.0, stash=None, defect=None):
    """What the kernel computes for these samples, from the packed program.  Default: exact activations, float64
    (tests the program).  operand_precision=True also rounds the A operands like the tensor cores see them:
    fp32 activations split into 16-bit hi (+ lo in the x3 modes), products hi*Whi (+ lo*Whi + hi*Wlo).
    emb_x [S, E]: the embedding operand in place of gamma(pts) (a hash-grid network's h(x)).
    Backward programs: grad_in is multiplied by grad_scale as it is loaded and every gradient written is divided by it
    (pnr_mlp_backward_trunk); `stash` (a dict) receives every stash slot the program writes, keyed by slot
    (EpiDesc.out_off1 - 1): H_i in slot i < D-1, dZ_j in slot 2D-2-j.
    defect: one of REPLAY_DEFECTS, a kernel made wrong on purpose, for the tests that check a bound rejects it: the
    gradient operands keep only their hi part; dZ_0 gated by layer 1's mask instead of layer 0's; dZ_0 stashed
    without the division by grad_scale; layer 0's d(input) overwriting the skip layer's instead of adding to it."""
    assert defect is None or defect in REPLAY_DEFECTS
    S_ = pts.shape[0]
    bf16 = cfg.precision.startswith("bf16")
    emb = np.zeros((S_, 64))
    if emb_x is None:
        emb[:, :3 + 6 * cfg.xyz_res] = O.embed(pts, cfg.xyz_res).double().numpy()
    else:
        emb[:, :emb_x.shape[1]] = emb_x
    dirs = np.zeros((S_, 32)); dirs[:, :3 + 6 * cfg.view_res] = O.embed(viewdirs, cfg.view_res).double().numpy()
    act = {COL_A_HI: np.zeros((S_, 256)), COL_HEAD_HI: np.zeros((S_, 128))}
    acc = np.zeros((S_, 256))
    CH = 4 + cfg.num_classes + cfg.num_instances
    out = np.zeros((S_, CH if grad_in is None else 3 + 6 * cfg.xyz_res if emb_x is None else emb_x.shape[1]))
    sig = np.zeros(S_)
    masks = {}                       # backward programs: ReLU sign pattern per slot
    step = -1
    stages_of = []
    for i in range(prog.n_stages):
        sd = prog.st[i]
        if sd.flags & F_WAIT_E0:
            step += 1
            stages_of.append([])
        stages_of[step].append(i)
    assert len(stages_of) == prog.n_steps
    for s, idxs in enumerate(stages_of):
        ed = prog.ep[s]
        for i in idxs:
            sd = prog.st[i]
            n, kc = sd.n, sd.ksteps * 2
            base = sd.gofs // 2
            parts = 2 if prog.passes == 3 else 1
            assert sd.bytes == parts * n * kc * 16
            nh = n
            assert sd.lo_off16 == nh * kc
            hi = to_f32(w16[base:base + nh * kc * 8], bf16).reshape(kc, nh, 8).astype(np.float64)
            lo = np.zeros_like(hi)
            if parts == 2:
                lo0 = base + sd.lo_off16 * 8
                lo = to_f32(w16[lo0:lo0 + nh * kc * 8], bf16).reshape(kc, nh, 8).astype(np.float64)
            W, Wlo = hi.transpose(1, 0, 2).reshape(nh, kc * 8), lo.transpose(1, 0, 2).reshape(nh, kc * 8)   # [row, k]
            if sd.a_kind == A_TMEM:
                region = COL_A_HI if sd.a_off >= COL_A_HI else COL_HEAD_HI
                k0 = (sd.a_off - region) * 2
                assert sd.a_lo_off - sd.a_off in (128, 64)          # lo parts sit one region further
                A = act[region][:, k0:k0 + kc * 8]
            elif sd.a_kind == A_EMB:
                A = emb[:, sd.a_off * 2:sd.a_off * 2 + kc * 8]
            else:
                A = dirs[:, sd.a_off * 2:sd.a_off * 2 + kc * 8]
            assert A.shape[1] == kc * 8
            if sd.flags & F_FIRST:
                acc[:, sd.acc_col:sd.acc_col + n] = 0.0
            if operand_precision:
                a_hi, a_lo = split16(A, bf16)
                if defect == "grad_hi_only" and s >= cfg.D:      # the backward steps: A is a gradient
                    a_lo = np.zeros_like(a_lo)
                prod = a_hi @ W.T
                if prog.passes == 3:
                    prod = prod + a_lo @ W.T + a_hi @ Wlo.T
                acc[:, sd.acc_col:sd.acc_col + n] += prod
            else:
                acc[:, sd.acc_col:sd.acc_col + n] += A @ (W + Wlo).T
            # issue table = the same stage, pre-digested
            d = prog.is_[i]
            assert d.acc_col == sd.acc_col and d.a_off == sd.a_off and d.lo_off16 == sd.lo_off16
            assert d.flags_k == (sd.flags | (sd.ksteps << 16) | (sd.a_kind << 24))
            assert d.b_lo_base == (nh << 16) and d.b_inc == 2 * nh
            assert (d.idesc >> 17) & 0x3F == n >> 3 and (d.idesc >> 24) & 0x1F == 8
            assert (d.idesc >> 7) & 7 == int(bf16)
        n = ed.n
        v = acc[:, ed.acc_col:ed.acc_col + n] + consts[ed.bias_off:ed.bias_off + n][None]
        if ed.kind == EPI_MASK_TO_A:         # gradient w.r.t. a hidden layer's output, gated by its sign pattern
            v = acc[:, ed.acc_col:ed.acc_col + n]
            slot = ed.n_valid if (defect == "mask_of_next_layer" and ed.n_valid == 1) else ed.n_valid - 1
            act[ed.dst_col][:, :n] = np.where(masks[slot][:, :n], v, 0.0) if ed.n_valid else v
            if stash is not None and ed.out_off1:
                keep = defect == "scale_left_in_dz0" and ed.n_valid == 1
                stash[ed.out_off1 - 1] = act[ed.dst_col][:, :n] / (1.0 if keep else grad_scale)
        elif ed.kind == EPI_LOADG_TO_A:      # last forward layer: the incoming gradient gated by its own pattern
            act[ed.dst_col][:, :n] = np.where(v > 0.0, grad_in[:, :n] * grad_scale, 0.0)
            if stash is not None and ed.out_off1:
                stash[ed.out_off1 - 1] = act[ed.dst_col][:, :n] / grad_scale
        elif ed.kind == EPI_GRAD_OUT:
            v = acc[:, ed.acc_col:ed.acc_col + ed.n_valid] / grad_scale
            add = ed.n_valid1 and defect != "skip_overwritten"
            out[:, ed.out_off:ed.out_off + ed.n_valid] = v + (out[:, ed.out_off:ed.out_off + ed.n_valid] if add else 0.0)
        elif ed.kind == EPI_RELU_TO_A:
            v = np.maximum(v, 0.0)
            if ed.sigma:
                sig = v @ consts[ed.aux_off:ed.aux_off + n].astype(np.float64)
            if grad_in is not None and ed.n_valid:
                masks[ed.n_valid - 1] = v > 0.0
            if stash is not None and ed.out_off1:
                stash[ed.out_off1 - 1] = v.copy()
            act[ed.dst_col][:, :n] = v
        elif ed.kind == EPI_VIEW_RGB:
            v = np.maximum(v, 0.0)
            wr = consts[ed.aux_off:ed.aux_off + 3 * n].astype(np.float64).reshape(3, n)
            out[:, :3] = v @ wr.T + consts[prog.rgb_bias_off:prog.rgb_bias_off + 3][None]
            out[:, 3] = sig + consts[prog.sigma_bias_off]
        else:
            out[:, ed.out_off:ed.out_off + ed.n_valid] = v[:, :ed.n_valid]
            if ed.n_valid1:        # the second half is a logit layer of its own (columns [n0, n))
                out[:, ed.out_off1:ed.out_off1 + ed.n_valid1] = v[:, ed.n0:ed.n0 + ed.n_valid1]
    return out, stages_of


def check_invariants(prog, stages_of):
    """Every step signals each accumulator half once, waits for the previous step's epilogues once, and releases
    the activation columns its first epilogue overwrites once."""
    for s, idxs in enumerate(stages_of):
        fl = [prog.st[i].flags for i in idxs]
        assert sum(bool(f & F_WAIT_E0) for f in fl) == 1 and fl[0] & F_WAIT_E0
        assert sum(bool(f & F_WAIT_E1) for f in fl) == 1 and sum(bool(f & F_WAIT_E1A) for f in fl) == 1
        if s == prog.view_step:      # its epilogue runs on the producer warps: one commit, to its own barrier
            assert fl[-1] & F_COMMIT_VIEW and not any(f & (F_COMMIT_ACC0 | F_COMMIT_ACC1 | F_COMMIT_WAR) for f in fl)
            assert s == prog.n_steps - 1 and prog.ep[s].n0 == prog.ep[s].n
            continue
        assert not any(f & F_COMMIT_VIEW for f in fl)
        assert sum(bool(f & F_COMMIT_ACC1) for f in fl) == 1 and fl[-1] & F_COMMIT_ACC1
        assert sum(bool(f & F_COMMIT_ACC0) for f in fl) <= 1
        assert sum(bool(f & F_COMMIT_WAR) for f in fl) == 1
        for i in idxs:
            sd = prog.st[i]
            assert sd.bytes <= 32768 and sd.n % 16 == 0 and 16 <= sd.n <= 128 and 1 <= sd.ksteps <= 8
    # hand-off counts of the issue table: E0 of every earlier step of the tile, E1 parts one step behind until the
    # stage that carries the matching wait flag
    for s, idxs in enumerate(stages_of):
        ed = prog.ep[s]
        assert 0 < ed.n0 <= ed.n1a <= ed.n and ed.n1a % 16 == 0
        seen_a = seen_b = False
        for i in idxs:
            f = prog.st[i].flags
            seen_a |= bool(f & F_WAIT_E1A)
            seen_b |= bool(f & F_WAIT_E1)
            needs = prog.is_[i].needs
            assert needs & 0xFF == s + 1
            assert (needs >> 8) & 0xFF == s + int(seen_a) and (needs >> 16) & 0xFF == s + int(seen_b)
            assert (needs >> 24) in (0, 1) and (prog.view_step >= 0 or needs >> 24 == 0)
            assert not (seen_b and not seen_a)            # "E1 done" is never required before "E1 part a done"


@pytest.mark.parametrize("preset,over", [
    ("cfg1", {}), ("cfg2", {}), ("cfg3", {}), ("cfg2", dict(precision="bf16x3")), ("cfg2", dict(precision="fp16")),
    ("cfg2", dict(D=5, W=128, num_classes=7, num_instances=3)), ("cfg1", dict(xyz_res=4, view_res=2))])
def test_program_replay_matches_oracle_network(preset, over):
    cfg = make_cfg(preset, **over)
    net = S.init_network_weights(make_network(cfg), seed=3)
    prog, w16, consts = build(cfg, net)
    assert prog.passes == (3 if cfg.precision.endswith("x3") else 1)
    g = torch.Generator().manual_seed(5)
    pts = (torch.rand(257, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(257, 3, generator=g), dim=-1)
    got, stages_of = replay(prog, w16, consts, cfg, pts, vd)
    check_invariants(prog, stages_of)
    onet = O.Network(cfg)
    onet.load_state_dict(net.state_dict())
    with torch.no_grad():
        ref = onet(pts, vd).double()
    got = torch.from_numpy(got)
    # the replay keeps activations exact, so only the 16-bit split of the WEIGHTS separates it from fp32:
    # 2^-22 (fp16 hi+lo), 2^-17 (bf16 hi+lo), 2^-11 (one fp16 part) per weight
    tol = {"fp16x3": 2e-5, "bf16x3": 1e-4, "fp16": 4e-3, "bf16": 3e-2}[cfg.precision]
    C_, K_ = cfg.num_classes, cfg.num_instances
    for name, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4)), ("sem", slice(4, 4 + C_)), ("inst", slice(4 + C_, 4 + C_ + K_))):
        if ref[:, sl].numel():
            assert_close(got[:, sl], ref[:, sl], rms(ref[:, sl]), f"{preset} {over} {name}", rel=tol)


@pytest.mark.parametrize("precision,bound", [("fp16x3", 2e-5), ("bf16x3", 1e-4), ("fp16", 1e-2), ("bf16", 6e-2)])
def test_operand_precision_of_each_mode(precision, bound):
    """The error the 16-bit operand split itself causes (activations AND weights rounded as the tensor cores see
    them, accumulation exact), relative to the per-tensor RMS: the x3 modes sit inside the 1e-4 parity tolerance
    with margin, the 1-pass modes do not - which is why fp16x3 is the default and the others are labelled."""
    cfg = make_cfg("cfg2", precision=precision)
    net = S.init_network_weights(make_network(cfg), seed=1)
    prog, w16, consts = build(cfg, net)
    g = torch.Generator().manual_seed(9)
    pts = (torch.rand(512, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(512, 3, generator=g), dim=-1)
    got, _ = replay(prog, w16, consts, cfg, pts, vd, operand_precision=True)
    onet = O.Network(cfg)
    onet.load_state_dict(net.state_dict())
    with torch.no_grad():
        ref = onet(pts, vd).double()
    got = torch.from_numpy(got)
    worst = max(float(((got[:, sl] - ref[:, sl]).abs().max() / rms(ref[:, sl]))) for sl in (slice(0, 3), slice(3, 4)))
    assert worst <= bound, f"{precision}: {worst:.3e} > {bound:.1e}"
    if precision in ("fp16", "bf16"):
        assert worst > 1e-4          # and really outside the tolerance: the mode must stay labelled "fast"


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg1", {}), ("cfg2", dict(precision="fp16")), ("cfg1", dict(D=3, W=128, xyz_res=4))])
def test_view_on_producers_program(preset, over):
    """The variant whose view epilogue runs on the producer warps: same stages, packed weights, constants and replayed
    outputs as the standard program; only the view step's commits and the hand-off counts differ."""
    cfg = make_cfg(preset, **over)
    net = S.init_network_weights(make_network(cfg), seed=3)
    std, w16, consts = build(cfg, net)
    vp, w16v, constsv = build(cfg, net, flags=PROGRAM_VIEW_PRODUCERS)
    assert std.view_step == -1 and vp.view_step == vp.n_steps - 1 and vp.n_stages == std.n_stages
    assert np.array_equal(w16, w16v) and np.array_equal(consts, constsv)
    g = torch.Generator().manual_seed(5)
    pts = (torch.rand(130, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(130, 3, generator=g), dim=-1)
    a, stages_of = replay(vp, w16v, constsv, cfg, pts, vd)
    b, _ = replay(std, w16, consts, cfg, pts, vd)
    assert np.array_equal(a, b)
    check_invariants(vp, stages_of)
    v = [prog_needs >> 24 for prog_needs in (vp.is_[i].needs for i in range(vp.n_stages))]
    assert v[-1] == 1 and v == sorted(v)                 # from the first stage that reuses the view columns on
    if cfg.W >= 256:
        assert v[0] == 0                                 # the first half of layer 0 lands in the other accumulator half
    cfg_h = make_cfg("cfg3")
    with_heads, _, _ = build(cfg_h, S.init_network_weights(make_network(cfg_h), seed=0), flags=PROGRAM_VIEW_PRODUCERS)
    assert with_heads.view_step == -1                                    # the view step is not the last one there


def trunk_grad_oracle(cfg, net, pts, grad_h):
    """dL/d(embedded xyz) by autograd through the oracle network's trunk (float64)."""
    onet = O.Network(cfg).double()
    onet.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    ex = O.embed(pts, cfg.xyz_res).double().requires_grad_(True)
    h = ex
    min_z = torch.full((pts.shape[0],), float("inf"), dtype=torch.float64)
    for i, lin in enumerate(onet.pts_linears):
        pre = lin(h)
        min_z = torch.minimum(min_z, pre.detach().abs().min(dim=1).values)
        h = torch.relu(pre)
        if i == onet.skip:
            h = torch.cat([ex, h], -1)
    h.backward(grad_h.double())
    return ex.grad, min_z


def assert_grad_close(got, ref, min_z, what, rel, kink=1e-6):
    """relu' is discontinuous: a sample with a pre-activation within rounding distance of zero may take the other
    branch (one gated unit = an O(1e-3) step in its gradient).  Those rows (|z| < kink somewhere in the trunk's
    2048 units; kink ~ 10x the rounding error of z in the mode under test) only have to be sane; every other row is
    held to `rel` of the gradient's RMS."""
    strict = min_z >= kink
    assert strict.float().mean() > 0.4, f"{what}: {int((~strict).sum())} of {len(strict)} rows sit on a ReLU kink"
    assert_close(got[strict], ref[strict], rms(ref), what, rel=rel)
    if (~strict).any():
        assert_close(got[~strict], ref[~strict], rms(ref), what + " (rows on a ReLU kink)", rel=1.0)


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg3", dict(precision="bf16x3")), ("cfg1", dict(D=5, W=128)),
                                         ("cfg1", dict(xyz_res=4, D=3, W=64))])
def test_backward_program_replay_matches_autograd(preset, over):
    """The backward program of the trunk (forward steps that keep their ReLU sign patterns, then the layers in reverse
    with transposed weights) replayed on the CPU = autograd through the oracle's trunk."""
    cfg = make_cfg(preset, **over)
    net = S.init_network_weights(make_network(cfg), seed=4)
    prog, w16, consts = build(cfg, net, flags=PROGRAM_BACKWARD)
    assert prog.n_steps == 2 * cfg.D + 1
    g = torch.Generator().manual_seed(6)
    pts = (torch.rand(200, 3, generator=g) * 2 - 1) * 4
    grad_h = torch.randn(200, cfg.W, generator=g)
    got, stages_of = replay(prog, w16, consts, cfg, pts, torch.zeros_like(pts), grad_in=grad_h.double().numpy())
    check_invariants(prog, stages_of)
    ref, min_z = trunk_grad_oracle(cfg, net, pts, grad_h)
    tol = {"fp16x3": 2e-5, "bf16x3": 1e-4}[cfg.precision]
    kink = {"fp16x3": 1e-6, "bf16x3": 2e-5}[cfg.precision]
    assert_grad_close(torch.from_numpy(got), ref, min_z, f"{preset} {over} d_emb", tol, kink)
    # with the operands rounded like the tensor cores see them (gradients split hi/lo as activations are)
    got_op, _ = replay(prog, w16, consts, cfg, pts, torch.zeros_like(pts), operand_precision=True, grad_in=grad_h.double().numpy())
    assert_grad_close(torch.from_numpy(got_op), ref, min_z, f"{preset} {over} d_emb (operand precision)", 1e-4, kink)


def test_backward_program_limits():
    cfg = make_cfg("cfg2", precision="fp16")
    net = S.init_network_weights(make_network(cfg), seed=0)
    with pytest.raises(_capi.PnrError, match="x3"):
        build(cfg, net, flags=PROGRAM_BACKWARD)
    cfg = make_cfg("cfg2", D=12)
    with pytest.raises(_capi.PnrError, match="slots"):
        build(cfg, S.init_network_weights(make_network(cfg), seed=0), flags=PROGRAM_BACKWARD)


def test_program_host_rejects_bad_input():
    cfg = make_cfg("cfg1")
    net = S.init_network_weights(make_network(cfg), seed=0)
    L = _capi.lib()
    pc = _capi.PnrConfig(cfg.D, cfg.W, cfg.xyz_res, cfg.view_res, 0, 0, _capi.PREC["fp16x3"], 0)
    w = net._linears()[0].weight.detach().float().contiguous()
    ptrs = (C.c_void_p * 2)(w.data_ptr(), w.data_ptr())
    shp = (C.c_int64 * 4)(w.shape[0], w.shape[1], w.shape[0], 1)
    pb, wb, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
    rc = L.pnr_program_host(C.byref(pc), ptrs, shp, 2, 0, None, 0, C.byref(pb), None, 0, C.byref(wb), None, 0, C.byref(nc))
    assert rc != 0 and b"tensors" in L.pnr_last_error()
    bad = _capi.PnrConfig(cfg.D, 100, cfg.xyz_res, cfg.view_res, 0, 0, _capi.PREC["fp16x3"], 0)
    rc = L.pnr_program_host(C.byref(bad), ptrs, shp, 2, 0, None, 0, C.byref(pb), None, 0, C.byref(wb), None, 0, C.byref(nc))
    assert rc != 0 and b"W=100" in L.pnr_last_error()
