"""CPU tier of the 16-bit operand split of the fused MLP kernel: the residual model against the bytes.

The x3 modes split every operand x = hi + lo, both parts rounded to nearest even in the operand format (split_x2 in
sm90.cuh for the activations, weight_part16 in mlp_program.h for the weights); the 1-pass modes keep hi.  With p
significand bits (11 in fp16, 8 in bf16) hi leaves at most 2^-p |x|, and lo, rounded from a value below 2^-p |x|, at
most 2^-2p |x| more.  fp16 also has a floor: below 2^-14 it is subnormal with a fixed spacing of 2^-24, so a part that
lands there leaves up to 2^-25 whatever |x|.  The lo part of a fp16 split is subnormal once |x - hi| < 2^-14, i.e. from
|x| ~ 2^-3 down, and the floor exceeds 2^-23 |x| below |x| = 2^-2: a 1e-4 activation is carried to ~2^-12 relative,
like one fp16 part.  The residual r = |x - hi - lo| and r1 = |x - hi|:
    fp16x3  r <= max(2^-23 |x|, 2^-25)     bf16x3  r <= 2^-17 |x|
    fp16    r1 <= max(2^-11 |x|, 2^-25)    bf16    r1 <= 2^-8 |x|
(bf16 keeps fp32's exponent range: no floor at the magnitudes a network holds).

Checked for floats from every binade 2^-30 .. 2^15, both signs, on the packed weight stream of `pnr_program_host` and on
the restated split of the activations (test_cpu_program.split16, what the program replay rounds with): every residual
lies within the model, every term of the model is reached, the fp16 floor included, so a model without the floor or a
split that truncates fails."""
import math

import numpy as np
import pytest
import torch

from oracle_bound import backward_bound, encoding, forward_bound, twin, view_encoding
from oracle_hashgrid import SCENE_AABB, hash_cfg, oracle_like
from panopticnerf_b200 import make_cfg, make_network, synthetic as S
from test_cpu_hashgrid_network import build
from test_cpu_program import F_WAIT_E0, PROGRAM_BACKWARD, REPLAY_DEFECTS, replay, split16, to_f32

# (relative, floor) of r (both parts) and of r1 (hi alone)
RESIDUAL = {"fp16": ((2.0 ** -23, 2.0 ** -25), (2.0 ** -11, 2.0 ** -25)), "bf16": ((2.0 ** -17, 0.0), (2.0 ** -8, 0.0))}
BINADES = range(-30, 16)


def binade_samples(per=1424, seed=0):
    """sign x 2^e x (1 + u) for every binade e of BINADES, below 65504 in the top one."""
    g = np.random.default_rng(seed)
    e = np.repeat(np.array(BINADES, dtype=np.float64), per)
    m = 1.0 + g.random(e.shape) * np.where(e == 15, 0.999, 1.0)
    return (np.where(g.random(e.shape) < 0.5, -1.0, 1.0) * np.ldexp(m, e.astype(int))).astype(np.float32)


def residual_model(x, fmt, parts=2):
    """The bound of |x - hi - lo| (parts = 2) or of |x - hi| (parts = 1) in operand format `fmt`."""
    rel, floor = RESIDUAL[fmt][2 - parts]
    return np.maximum(rel * np.abs(x), floor)


def _check_residuals(x, hi, lo, fmt):
    """hi + lo against the model; returns the residuals r and r1."""
    x = x.astype(np.float64)
    r, r1 = np.abs(x - hi - lo), np.abs(x - hi)
    assert (r <= residual_model(x, fmt)).all(), f"{fmt}: |x - hi - lo| outside the model"
    assert (r1 <= residual_model(x, fmt, parts=1)).all(), f"{fmt}: |x - hi| outside the model"
    return r, r1


def _check_model_is_reached(x, r, r1, fmt):
    """The relative terms are reached in the normal binades, and (fp16) the absolute floor where the lo part, or the hi
    part, is subnormal: a model without the floor, or a split that truncates, fails."""
    ax = np.abs(x.astype(np.float64))
    (rel, _), (rel1, _) = RESIDUAL[fmt]
    normal = ax >= (2.0 ** -2 if fmt == "fp16" else 2.0 ** -126)    # fp16: where the floor is below 2^-23 |x|
    assert (r[normal] / ax[normal]).max() > 0.9 * rel and (r1[normal] / ax[normal]).max() > 0.9 * rel1
    if fmt == "fp16":
        sub_lo = (ax < 2.0 ** -4) & (ax >= 2.0 ** -14)
        sub_hi = ax < 2.0 ** -14
        for part in (sub_lo, sub_hi):
            assert r[part].max() > 0.9 * 2.0 ** -25, "the 2^-25 floor is not reached"
            assert (r[part] > rel * ax[part]).any(), "2^-23 |x| alone holds where the floor should"
        assert r1[sub_hi].max() > 0.9 * 2.0 ** -25


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_packed_weight_parts_follow_the_residual_model(fmt):
    """Trunk layer 1 of a W = 256 network holds the samples; its hi / lo images are read back from the packed stream."""
    cfg = make_cfg("cfg2", D=3, precision=fmt + "x3")
    net = S.init_network_weights(make_network(cfg), seed=0)
    x = binade_samples()
    x = np.concatenate([x, np.zeros(256 * 256 - x.size, np.float32)])
    with torch.no_grad():
        net.pts_linears[1].weight.copy_(torch.from_numpy(x.reshape(256, 256)))
    prog, w16, _ = build(cfg, net)
    hi, lo = np.full((256, 256), np.nan), np.full((256, 256), np.nan)
    step = -1
    for i in range(prog.n_stages):
        sd = prog.st[i]
        step += bool(sd.flags & F_WAIT_E0)
        if step != 1:
            continue
        kc, base = sd.ksteps * 2, sd.gofs // 2
        k0 = (sd.a_off - 256) * 2
        for img, off in ((hi, base), (lo, base + sd.lo_off16 * 8)):
            part = to_f32(w16[off:off + sd.n * kc * 8], fmt == "bf16").reshape(kc, sd.n, 8).astype(np.float64)
            img[sd.acc_col:sd.acc_col + sd.n, k0:k0 + kc * 8] = part.transpose(1, 0, 2).reshape(sd.n, kc * 8)
    assert not np.isnan(hi).any() and not np.isnan(lo).any()
    hi, lo = hi.reshape(-1), lo.reshape(-1)
    # the packer and the activations' split_x2 round alike, bit for bit
    h2, l2 = split16(x, fmt == "bf16")
    assert np.array_equal(hi, h2) and np.array_equal(lo, l2)
    r, r1 = _check_residuals(x, hi, lo, fmt)
    _check_model_is_reached(x, r, r1, fmt)


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_activation_split_follows_the_residual_model(fmt):
    """split_x2 of the activations (restated: round to nearest even, twice, with subnormals), both signs."""
    x = binade_samples(per=4096, seed=1)
    hi, lo = split16(x, fmt == "bf16")
    r, r1 = _check_residuals(x, hi, lo, fmt)
    _check_model_is_reached(x, r, r1, fmt)


# ------------------------------------------------------------------------------------------------ bound vs replay
TWIN_LAYERS = {"early": 0, "skip": 1, "last": 2}        # D = 3: layer 0, the skip layer and the last trunk layer
TABLES = (1e-4, 1e-2, 1.0)                               # HashGrid's own init, and two larger tables


def regimes():
    """(name, hash table scale or None, point scale, twin layer or None, k; k = -1: the largest upward twin)."""
    out = [("default", None, 4.0, None, 0)]
    for lname, layer in TWIN_LAYERS.items():
        out += [(f"down-{lname}-k{k}", None, 4.0, layer, k) for k in (4, 8, 12, 16)]
        out += [(f"up-{lname}", None, 4.0, layer, -1)]
    out += [(f"table-{a:g}", a, None, None, 0) for a in TABLES]
    out += [("kitti360", None, 300.0, None, 0)]         # |p| up to 300 m: gamma(x) arguments up to 2^9 x 300
    return out


REGIMES = regimes()
# The worst |err| / B of the replay is 1/64 .. 1/16 in most regimes.  It is lower where many units sit within their
# bound of a ReLU kink, whose either branch the bound must allow: the bf16 modes (1/100 in bf16x3, 1/250 in bf16) and
# layer 0 twinned down by 2^16 (1/2900), where the floor makes layer 1's error 2^-9 of its values.
TIGHT = 1.0 / 4096


def make_regime(precision, regime, seed=1, **over):
    """cfg and network (CPU, fp32) of one regime, before its twin is applied (apply_twin)."""
    name, table, pscale, layer, k = regime
    over = dict(dict(D=3, W=256), **over, precision=precision)
    if table is not None:
        cfg = hash_cfg("cfg2", hash_levels=16, hash_features=2, hash_log2_size=12, **over)
    else:
        cfg = make_cfg("cfg2", **over)
    net = S.init_network_weights(make_network(cfg), seed=seed)
    if table is not None:
        with torch.no_grad():
            g = torch.Generator().manual_seed(seed + 100)
            net.xyz_encoder.table.copy_((torch.rand(net.xyz_encoder.table.shape, generator=g) * 2 - 1) * table)
    return cfg, net


def regime_points(regime, n, seed):
    """Sample points of a regime (inside the hash grid's box for the table regimes) and unit view directions."""
    g = torch.Generator().manual_seed(seed)
    if regime[1] is not None:
        lo, hi = torch.tensor(SCENE_AABB[:3]), torch.tensor(SCENE_AABB[3:])
        pts = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    else:
        pts = (torch.rand(n, 3, generator=g) * 2 - 1) * regime[2]
    return pts, torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)


def trunk_input(cfg, net, pts):
    """The float64 trunk input and the kernel's error of it: h(x) of the fp32 oracle encoder (exact), or gamma(x)."""
    if getattr(cfg, "xyz_encoding", "frequency") == "hashgrid":
        with torch.no_grad():
            ex = oracle_like(net, cfg).xyz_encoder(pts.cpu()).double()
        return ex, torch.zeros_like(ex)
    return encoding(pts.cpu(), cfg.xyz_res)


def up_k(net, ex, layer):
    """The largest k that keeps trunk layer `layer`'s weights, biases and (float64) activations times 2^k below 2^14,
    inside the fp16 range check (|x| >= 65520) with room for samples the float64 pass did not see."""
    h, skip = ex, len(net.pts_linears) // 2
    for i, lin in enumerate(net.pts_linears[:layer + 1]):
        h = torch.relu(torch.nn.functional.linear(h, lin.weight.detach().double(), lin.bias.detach().double()))
        if i == skip:
            h = torch.cat([ex, h], -1)
    lin = net.pts_linears[layer]
    m = max(float(lin.weight.abs().max()), float(lin.bias.abs().max()), float(h.abs().max()))
    return int(math.floor(math.log2(2.0 ** 14 / m)))


def apply_twin(net, regime, ex):
    """The regime's twin; returns the network and the k applied (negative: upward)."""
    name, table, pscale, layer, k = regime
    if layer is None:
        return net, 0
    if k < 0:
        k = -up_k(net, ex, layer)
        assert k <= -4, f"{name}: no room for an upward twin"
    return twin(net, layer, k), k


def ratio(got, ref, B):
    """|got - ref| / B per element (0 where both are 0, inf for an error where B = 0); NaN patterns must coincide."""
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), "NaN patterns differ"
    err = torch.nan_to_num(got - ref).abs()
    B = torch.nan_to_num(B)
    return torch.where(B > 0, err / torch.where(B > 0, B, torch.ones_like(B)), torch.where(err > 0, torch.inf, 0.0))


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3", "fp16", "bf16"])
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_bound_holds_and_is_tight_on_the_replay(regime, precision):
    """oracle_bound against the program replay with operands rounded as the tensor cores see them and exact
    accumulation (the bound's accumulation term at 0): every element within B, and the worst at least TIGHT of B."""
    cfg, net = make_regime(precision, regime, W=128)
    pts, vd = regime_points(regime, 512, seed=5)
    ex, e_ex = trunk_input(cfg, net, pts)
    ed, e_ed = view_encoding(vd, cfg.view_res)
    ref0 = forward_bound(net, precision, ex, e_ex, ed, e_ed)[0]
    net, k = apply_twin(net, regime, ex)
    ref, B, _, _ = forward_bound(net, precision, ex, e_ex, ed, e_ed, acc=False)
    assert torch.equal(ref, ref0), "a twin must leave the float64 network unchanged"
    prog, w16, consts = build(cfg, net)
    # the replay's gamma(x) / gamma(d) are torch's fp32 sin / cos (within 1 ulp); h(x) is the fp32 oracle encoder
    got, _ = replay(prog, w16, consts, cfg, pts, vd, operand_precision=True,
                    emb_x=ex.numpy() if regime[1] is not None else None)
    worst = float(ratio(torch.from_numpy(got), ref, B).max())
    print(f"{regime[0]} k={k} {precision}: worst |err|/B = {worst:.3g}")
    assert worst <= 1.0, f"{regime[0]} {precision}: an element outside the bound ({worst:.3g})"
    assert worst >= TIGHT, f"{regime[0]} {precision}: the bound is loose ({worst:.3g})"


# ------------------------------------------------------------------------------------------------ backward bound vs replay
GRADS = ("unit", "tiny-unscaled", "spread")


def default_grad_scale(grad_h):
    """The power of two Network.backward_trunk picks: max |grad_h| * grad_scale ~ 256."""
    m = float(grad_h.abs().max())
    return 2.0 ** max(-100, min(100, round(math.log2(256.0 / m))))


def grad_regime(name, n, W, seed):
    """(grad_h [n, W], grad_scale).  unit: O(1) at the default scale; tiny-unscaled: 2^-20 O(1) with grad_scale = 1, so
    the fp16 parts of every gradient are subnormal; spread: columns over 2^-12 .. 2^4, default scale.  No entry is 0:
    a nonzero dZ_{D-1} is then exactly the last layer's mask."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, W, generator=g)
    x = torch.where(x == 0, torch.ones_like(x), x)
    if name == "tiny-unscaled":
        return x * 2.0 ** -20, 1.0
    if name == "spread":
        x = x * torch.exp2(torch.linspace(-12.0, 4.0, W))[torch.randperm(W, generator=g)]
    return x, default_grad_scale(x)


def fp16_safe_scale(b, gs):
    """The largest power of two <= gs that keeps every float64 dZ_j (j < D-1: the loaded one is at most ~256) times
    the scale below 2^14, inside the fp16 range check with room to spare."""
    m = max(float(d.abs().max()) for d in b["dZ"])
    return min(gs, 2.0 ** math.floor(math.log2(2.0 ** 14 / m))) if m > 0 else gs


def stash_masks(H, dZ_last):
    """The kernel's D ReLU masks from its stash: H_i > 0 for i < D-1, dZ_{D-1} != 0 for the last layer."""
    return [(h > 0).double() for h in H] + [(dZ_last != 0).double()]


def backward_ratios(b, dZ, d_in):
    """Worst |err| / B per dZ_j and of d(trunk input)."""
    out = {f"dZ{j}": float(ratio(dZ[j], b["dZ"][j], b["B_dZ"][j]).max()) for j in range(len(dZ))}
    out["d_in"] = float(ratio(d_in, b["d_in"], b["B_in"]).max())
    return out


def _replay_backward(cfg, net, regime, pts, ex, grad_h, gs, defect=None):
    prog, w16, consts = build(cfg, net, flags=PROGRAM_BACKWARD)
    stash = {}
    d_in, _ = replay(prog, w16, consts, cfg, pts, torch.zeros_like(pts), operand_precision=True,
                     grad_in=grad_h.double().numpy(), emb_x=ex.numpy() if regime[1] is not None else None,
                     grad_scale=gs, stash=stash, defect=defect)
    D = cfg.D
    H = [torch.from_numpy(stash[i]) for i in range(D - 1)]
    dZ = [torch.from_numpy(stash[2 * D - 2 - j]) for j in range(D)]
    return torch.from_numpy(d_in)[:, :ex.shape[1]], H, dZ


def _backward_case(precision, regime, grad, n=512, defect=None):
    cfg, net = make_regime(precision, regime, W=128)
    pts, _ = regime_points(regime, n, seed=5)
    ex, e_ex = trunk_input(cfg, net, pts)
    net, k = apply_twin(net, regime, ex)
    grad_h, gs = grad_regime(grad, n, cfg.W, seed=7)
    d_in, H, dZ = _replay_backward(cfg, net, regime, pts, ex, grad_h, gs, defect)
    masks = stash_masks(H, dZ[-1])
    b = backward_bound(net, precision, ex, e_ex, grad_h, gs, masks, acc=False)
    if precision == "fp16x3" and fp16_safe_scale(b, gs) < gs:      # the kernel would flag this scale: rerun below it
        gs = fp16_safe_scale(b, gs)
        d_in, H, dZ = _replay_backward(cfg, net, regime, pts, ex, grad_h, gs, defect)
        b = backward_bound(net, precision, ex, e_ex, grad_h, gs, masks, acc=False)
    return backward_ratios(b, dZ, d_in), f"{regime[0]} k={k} {precision} {grad} gs=2^{int(math.log2(gs))}"


@pytest.mark.parametrize("grad", GRADS)
@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_backward_bound_holds_and_is_tight_on_the_replay(regime, precision, grad):
    """oracle_bound.backward_bound against the backward program's replay (operands rounded as the tensor cores see
    them, exact accumulation), pinned to the masks of the replay's own stash: every dZ_j slot and every element of
    d(trunk input) within B, and the worst at least TIGHT of B."""
    worst, name = _backward_case(precision, regime, grad)
    print(f"{name}: " + " ".join(f"{g}={v:.3g}" for g, v in worst.items()))
    assert max(worst.values()) <= 1.0, f"{name}: an element outside the bound {worst}"
    assert max(worst.values()) >= TIGHT, f"{name}: the bound is loose {worst}"


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("defect", REPLAY_DEFECTS)
def test_backward_bound_rejects_a_defective_kernel(defect, precision):
    """Each deliberate defect of the replay (a 1-pass gradient operand, a mask one layer off, grad_scale left in the
    dZ_0 slot, the skip layer's d(input) overwritten by layer 0's) takes some element outside the bound."""
    worst, name = _backward_case(precision, REGIMES[0], "unit", defect=defect)
    print(f"{defect} {name}: " + " ".join(f"{g}={v:.3g}" for g, v in worst.items()))
    assert max(worst.values()) > 1.0, f"{defect} {name}: the bound does not see it {worst}"
