"""GPU: the range check of the fused MLP kernel (bit 0 of pnr_status) at every operand it guards, and the NaN inputs and
parameters it must let through to the outputs, in every instantiation (forward from points and from rays, the
compositing epilogue, the trunk forward and backward programs, pnr_render_fused) and precision.

The reference is the oracle network in float64, fed the same fp32 weights and inputs.  It decides, per case, whether
the bit must be set (some value the kernel converts to a 16-bit operand rounds to inf in that format, or is NaN) and
what the outputs must be (within the path's tolerance of float64, NaN exactly where the oracle has NaN).

Cases at the fp16 threshold are exact in fp32 and float64: unit j of layers 0 .. k-1 carries the coordinate x0 (weight
1 on one chain column, zeros elsewhere in its row, bias 0) and layer k adds a bias of 65000, so its pre-activation is
x0 + 65000 = 65519 (hi part 65504, lo part 15: clear) or 65520 (rounds to inf in fp16: set)."""
import math

import pytest
import torch
import torch.nn.functional as F

import panopticnerf_b200 as PN
from oracle import reference_renderer as O
from oracle_hashgrid import hash_cfg, oracle_like
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as S
from test_gpu_config_space import _dyadic_rays, _inputs, _oracle64
from util import rel_err, rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRECS = ["fp16x3", "fp16", "bf16x3", "bf16"]
# the x3 tolerances of test_gpu_config_space; bf16x3 at 3e-4 here: the hash-grid probes carry a feature of 65519 into
# layer 0 at full weight, ~2^-17 of which lands on outputs whose RMS is far smaller
X3_TOL = {"fp16x3": 2e-5, "bf16x3": 3e-4}
# the 1-pass bounds of test_cpu_program, bf16 at 1e-1: ~2^-9 per operand, and in the head probes (whose trunk output
# column j is read by the chain alone) sigma sums fewer, larger terms (7e-2 of its RMS measured on an H100)
FAST_BOUND = {"fp16": 1e-2, "bf16": 1e-1}
HEADS = dict(num_classes=5, num_instances=6)
CHAIN_J = 5                                    # the chain unit
S_SMALL, BAD = 256, 100                        # samples of a small launch (four tiles) and the probe sample


# ------------------------------------------------------------------------------------------------ float64 reference
def _half(prec):
    return torch.float16 if prec.startswith("fp16") else torch.bfloat16


def _forward64(onet, ex, ed):
    """The oracle network's forward in float64 from its embeddings, and every value the forward program writes into a
    16-bit operand: both embeddings, each trunk activation and each head's hidden activation (the view layer's hidden
    units, sigma and the outputs are fp32 in the kernel)."""
    ops, h = [ex, ed], ex
    for i, lin in enumerate(onet.pts_linears):
        h = F.relu(lin(h))
        ops.append(h)
        if i == onet.skip:
            h = torch.cat([ex, h], -1)
    outs = [onet.rgb_linear(F.relu(onet.views_linears[0](torch.cat([onet.feature_linear(h), ed], -1)))),
            onet.alpha_linear(h)]
    for name in ("semantic_linears", "instance_linears"):
        if hasattr(onet, name):
            a = F.relu(getattr(onet, name)[0](h))
            ops.append(a)
            outs.append(getattr(onet, name)[1](a))
    return torch.cat(outs, -1), ops


def _ref(net_cpu, cfg, pts, vd):
    """float64 outputs [S, CH] and operands of the network at fp32 points / directions."""
    with torch.no_grad():
        if getattr(cfg, "xyz_encoding", "frequency") == "hashgrid":
            onet = oracle_like(net_cpu, cfg, torch.float64)
            ex = oracle_like(net_cpu, cfg).xyz_encoder(pts).double()     # the fp32 encoder: the kernel's gather
        else:
            onet = _oracle64(cfg, net_cpu)
            ex = O.embed(pts.double(), cfg.xyz_res)
        return _forward64(onet, ex, O.embed(vd.double(), cfg.view_res))


def _flagged(ops, prec):
    """Must bit 0 be set: does some operand value round to inf in the 16-bit format, or is it NaN?"""
    return any(bool((~torch.isfinite(o.float().to(_half(prec)))).any()) for o in ops)


def _check(got, ref, prec, what):
    """NaN exactly where float64 has NaN; the rest within the path's tolerance (x3: per channel group of its RMS;
    1-pass: the operand-precision bound)."""
    got = got.detach().cpu().double().reshape(ref.shape)
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), f"{what}: NaN pattern differs from float64"
    for c0, c1 in ((0, 3), (3, 4), (4, ref.shape[1])):
        if c1 <= c0:
            continue
        r = ref[:, c0:c1]
        floor = max(rms(torch.nan_to_num(r)), 1e-6)
        e = rel_err(got[:, c0:c1], r, floor)
        tol = X3_TOL.get(prec, FAST_BOUND.get(prec))
        assert e <= tol, f"{what} channels {c0}:{c1}: rel err {e:.3e} > {tol:.1e}"


def _net(cfg, seed=3):
    return S.init_network_weights(make_network(cfg), seed=seed)


def _to_dev(net_cpu, cfg):
    net = make_network(cfg)
    net.load_state_dict(net_cpu.state_dict())
    return net.to(DEV)


def _status(net, reset=True):
    return net.range_status(reset=reset)


# ------------------------------------------------------------------------------------------------ exact threshold probes
def _chain(net, k, head=None, j=CHAIN_J, top=65000.0, r=CHAIN_J + 1):
    """Unit j of trunk layers 0 .. k-1 (all of them with `head`) carries x0; layer k (or the head's hidden layer) gets
    bias `top` on it.  No other unit reads the chain, but one: unit r of the next trunk layer (sigma, after the last
    one) reads its end with weight 2^-8, so that a dropped lo part of 15 shows in the outputs.  That weight is a power
    of two, whose fp16 lo part is 0: a weight with a subnormal lo part would lose up to 2^-25 of itself times 65519,
    a limit of the operand format that would swamp the check of the kernel."""
    last = net.D - 1 if head is not None else k

    def col(i):                                   # the chain's input column of trunk layer i
        return 0 if i == 0 else (net.in_dim + j if i == net.skip + 1 else j)
    with torch.no_grad():
        for i in range(last + 1):
            lin = net.pts_linears[i]
            lin.weight[:, col(i)] = 0.0
            lin.weight[j].zero_()
            lin.weight[j, col(i)] = 1.0
            lin.bias[j] = 0.0
        if last + 1 < net.D:
            nxt = net.pts_linears[last + 1]
            nxt.weight[:, col(last + 1)] = 0.0
            nxt.weight[r, col(last + 1)] = 2.0 ** -8
        else:                                     # the readers of the trunk output
            for name in ("alpha_linear", "feature_linear", "semantic_linears.0", "instance_linears.0"):
                if hasattr(net, name.split(".")[0]):
                    net.get_submodule(name).weight[:, j] = 0.0
            if head is None:
                net.alpha_linear.weight[0, j] = 2.0 ** -8
        if head is None:
            net.pts_linears[k].bias[j] = top
        else:
            lin = getattr(net, head)[0]
            lin.weight[j].zero_()
            lin.weight[j, j] = 1.0
            lin.bias[j] = top
    return net


# name: cfg overrides, where the value sits ("x": the x0 column of gamma(x) itself, "d": of gamma(d), "chain": x0 + 65000
# at trunk layer k or a head's hidden layer), and whether the samples come as rays
PROBES = {
    "gamma_x_pts": dict(site="x"),
    "gamma_x_rays": dict(site="x", rays=True),
    "gamma_d_pts": dict(site="d"),
    "trunk_regs_W256": dict(site="chain", k=2),
    "trunk_last_sigma": dict(site="chain", k=7),
    "trunk_W64": dict(site="chain", k=2, over=dict(W=64)),
    "trunk_W128": dict(site="chain", k=2, over=dict(W=128)),
    "skip_layer": dict(site="chain", k=5),
    "semantic_hidden": dict(site="chain", head="semantic_linears", over=HEADS),
    "instance_hidden": dict(site="chain", head="instance_linears", over=HEADS),
}


def _probe_inputs(site, value, base, n=S_SMALL, bad=BAD):
    """pts / viewdirs with the probed coordinate at `base` everywhere and at `value` in sample `bad`."""
    pts, vd = _inputs(n, seed=11)
    col = vd if site == "d" else pts
    col[:, 0] = base
    col[bad, 0] = value
    return pts, vd


def _probe_rays(value, base, R=64, N=4, bad=25):
    """Rays along +z whose origin x is `base` (`value` for ray `bad`): every point's x0 is the origin's, exactly."""
    rays, z, _, _ = _dyadic_rays(R, N, seed=12)
    rays[:, 3:] = torch.tensor([0.0, 0.0, 1.0])
    rays[:, 0] = base
    rays[bad, 0] = value
    pts = (rays[:, None, :3] + rays[:, None, 3:] * z[..., None]).reshape(-1, 3)
    vd = rays[:, None, 3:].expand(-1, N, -1).reshape(-1, 3).contiguous()
    return rays, z, pts, vd


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", list(PROBES))
def test_threshold_at_every_guarded_operand(name, prec):
    """65519 in the operand: clear, and carried exactly (outputs within tolerance of float64); 65520 in one sample: set
    in the fp16 modes, every other sample unchanged bit for bit; the bf16 modes hold both values."""
    pr = PROBES[name]
    cfg = make_cfg("cfg2", precision=prec, **pr.get("over", {}))
    net_cpu = _net(cfg)
    chain = pr["site"] == "chain"
    if chain:
        _chain(net_cpu, pr.get("k"), pr.get("head"))
    base, over_v = (519.0, 520.0) if chain else (65519.0, 65520.0)
    net = _to_dev(net_cpu, cfg)
    outs = {}
    for v in (base, over_v):
        if pr.get("rays"):
            rays, z, pts, vd = _probe_rays(v, base)
            got = net.forward_rays(rays.to(DEV), z.to(DEV)).reshape(pts.shape[0], -1)
        else:
            pts, vd = _probe_inputs(pr["site"], v, base)
            got = net(pts.to(DEV), vd.to(DEV))
        ref, ops = _ref(net_cpu, cfg, pts, vd)
        want = _flagged(ops, prec)
        assert want == (v == over_v and prec.startswith("fp16")), "the probe does not reach the threshold"
        assert bool(_status(net) & 1) == want, f"{name} {prec} value {v}: status"
        if not want:
            _check(got, ref, prec, f"{name} {prec} value {v}")
        outs[v] = got.cpu()
    bad = (torch.arange(outs[base].shape[0]) // 4 == 25) if pr.get("rays") else (torch.arange(outs[base].shape[0]) == BAD)
    assert torch.equal(outs[base][~bad], outs[over_v][~bad]), "an overflow changed another sample"


@pytest.mark.parametrize("F_", [1, 2, 4, 8])
@pytest.mark.parametrize("thread", ["xyz", "dir"])
@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_threshold_in_hashgrid_features(thread, F_, prec):
    """One table entry of the level the xyz thread gathers (level 0) or the dir thread gathers (the last, E = 16: two
    core rows, one per thread) at 65519 / 65520, read with weight 1 by a sample on the grid's corner vertex."""
    L = 16 // F_
    cfg = hash_cfg("cfg2", hash_levels=L, hash_features=F_, hash_log2_size=14, precision=prec)
    net_cpu = _net(cfg)
    lvl = 0 if thread == "xyz" else L - 1
    g = torch.Generator().manual_seed(5)
    lo, hi = torch.tensor(cfg.hash_aabb[:3]), torch.tensor(cfg.hash_aabb[3:])
    pts = lo + (hi - lo) * (0.1 + 0.8 * torch.rand(S_SMALL, 3, generator=g))
    pts[BAD] = lo                                                  # on the corner vertex of every level
    vd = F.normalize(torch.randn(S_SMALL, 3, generator=g), dim=-1)
    row = _corner_row(net_cpu, cfg, pts[BAD:BAD + 1], lvl, F_)
    net = _to_dev(net_cpu, cfg)
    for v in (65519.0, 65520.0):
        with torch.no_grad():
            net_cpu.xyz_encoder.table[lvl, row, F_ - 1] = v
            net.xyz_encoder.table.copy_(net_cpu.xyz_encoder.table)
        got = net(pts.to(DEV), vd.to(DEV))
        ref, ops = _ref(net_cpu, cfg, pts, vd)
        assert float(ops[0][BAD, lvl * F_ + F_ - 1]) == v                # exact blend: the feature is the entry
        want = _flagged(ops, prec)
        assert want == (v == 65520.0 and prec == "fp16x3")
        assert bool(_status(net) & 1) == want, f"{thread} F={F_} {prec} {v}"
        if not want:
            _check(got, ref, prec, f"hash {thread} F={F_} {prec} {v}")


def _corner_row(net_cpu, cfg, p, lvl, F_):
    """Index of the table row at level `lvl` that point p reads with weight 1 (found through the oracle encoder)."""
    enc = oracle_like(net_cpu, cfg).xyz_encoder
    T = enc.table.shape[1]
    with torch.no_grad():
        enc.table.zero_()
        enc.table[lvl, :, F_ - 1] = torch.arange(T, dtype=torch.float32)
        row = float(enc(p)[0, lvl * F_ + F_ - 1])
    assert row == int(row)
    return int(row)


# ------------------------------------------------------------------------------------------------ no false positives
FP32_OUTPUTS = {
    "sigma_raw_1e6": lambda n: n.alpha_linear.bias.fill_(1e6),
    "rgb_raw_1e6": lambda n: n.rgb_linear.bias.fill_(1e6),
    "logits_1e6": lambda n: (n.semantic_linears[1].bias.fill_(1e6), n.instance_linears[1].bias.fill_(-1e6)),
    "view_hidden_1e5": lambda n: n.views_linears[0].bias.__setitem__(0, 1e5),
}


@pytest.mark.parametrize("name", list(FP32_OUTPUTS) + ["hashgrid_outside_aabb"])
def test_fp32_values_leave_the_bit_clear(name):
    """sigma, rgb and logits of 1e6 and a view-layer hidden value of 1e5 are fp32 in the kernel, never 16-bit operands;
    hash-grid points far outside the box are clamped to it by design.  fp16x3: clear, and within tolerance."""
    if name == "hashgrid_outside_aabb":
        cfg = hash_cfg("cfg2", hash_levels=8, hash_features=2, hash_log2_size=14, **HEADS)
        net_cpu = _net(cfg)
        pts, vd = _inputs(S_SMALL, seed=4)
        pts = pts * 1e4                                            # |x| up to 4e4, far outside the box
    else:
        cfg = make_cfg("cfg2", **HEADS)
        net_cpu = _net(cfg)
        with torch.no_grad():
            FP32_OUTPUTS[name](net_cpu)
        pts, vd = _inputs(S_SMALL, seed=4)
    net = _to_dev(net_cpu, cfg)
    got = net(pts.to(DEV), vd.to(DEV))
    ref, ops = _ref(net_cpu, cfg, pts, vd)
    assert not _flagged(ops, "fp16x3")
    assert _status(net) == 0
    _check(got, ref, "fp16x3", name)
    if name != "hashgrid_outside_aabb":
        assert float(ref.abs().max()) > 1e3                        # the large value reaches the outputs


# ------------------------------------------------------------------------------------------------ non-finite inputs
INPUTS = [(w, v) for w in ("pts", "viewdirs", "ray_origin", "ray_direction", "z") for v in ("nan", "inf", "-inf")]
INPUTS.append(("zero_direction", "0"))


def _bad_inputs(what, value, R=64, N=4, r=25, i=2):
    """Clean and bad inputs of one launch (pts mode or rays mode), and the samples the bad value touches."""
    v = float(value)
    if what in ("pts", "viewdirs"):
        pts, vd = _inputs(S_SMALL, seed=6)
        bp, bv = pts.clone(), vd.clone()
        (bp if what == "pts" else bv)[BAD, 1] = v
        rows = torch.arange(S_SMALL) == BAD
        return dict(pts=pts, vd=vd), dict(pts=bp, vd=bv), rows
    rays, z, _, _ = _dyadic_rays(R, N, seed=7)
    br, bz = rays.clone(), z.clone()
    if what == "ray_origin":
        br[r, 1] = v
    elif what == "ray_direction":
        br[r, 4] = v
    elif what == "zero_direction":
        br[r, 3:] = 0.0
    else:
        bz[r, i] = v
    rows = torch.arange(R * N) // N == r
    if what == "z":
        rows = torch.arange(R * N) == r * N + i
    return dict(rays=rays, z=z), dict(rays=br, z=bz), rows


def _pts_of(inp):
    """The kernel's points and directions of a launch, in fp32 as it forms them (o + d*z separately rounded)."""
    if "pts" in inp:
        return inp["pts"], inp["vd"]
    rays, z = inp["rays"], inp["z"]
    N = z.shape[1]
    pts = (rays[:, None, :3] + rays[:, None, 3:] * z[..., None]).reshape(-1, 3)
    d = rays[:, 3:].double()
    vd = (d / d.norm(dim=-1, keepdim=True))[:, None].expand(-1, N, -1).reshape(-1, 3)
    return pts, vd


def _forward(net, inp):
    if "pts" in inp:
        return net(inp["pts"].to(DEV), inp["vd"].to(DEV))
    R, N = inp["z"].shape
    return net.forward_rays(inp["rays"].to(DEV), inp["z"].to(DEV)).reshape(R * N, -1)


_NETS = {}


def _heads_net(prec):
    """One network with both heads per precision, shared by the non-finite input cases."""
    if prec not in _NETS:
        cfg = make_cfg("cfg2", precision=prec, **HEADS)
        net_cpu = _net(cfg)
        _NETS[prec] = (cfg, net_cpu, _to_dev(net_cpu, cfg))
    return _NETS[prec]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("what,value", INPUTS, ids=[f"{w}-{v}" for w, v in INPUTS])
def test_non_finite_input_is_reported_and_reaches_the_outputs(what, value, prec):
    """NaN / +-Inf in pts, viewdirs, a ray's origin or direction or z, and a zero-length direction (d/|d| = 0/0): bit 0
    set in every precision, NaN in exactly the channels float64 makes NaN (a bad direction: rgb, not sigma or the
    logits), every other sample bit-identical to the launch without the bad value."""
    cfg, net_cpu, net = _heads_net(prec)
    clean, bad, rows = _bad_inputs(what, value)
    ref_clean = _forward(net, clean).cpu()
    assert _status(net) == 0
    got = _forward(net, bad).cpu()
    pts, vd = _pts_of(bad)
    ref, ops = _ref(net_cpu, cfg, pts, vd)
    assert _flagged(ops, prec)
    assert _status(net) & 1, f"{what}={value} {prec}: not reported"
    assert bool(torch.isnan(ref[rows]).any()) and not bool(torch.isnan(ref[~rows]).any())
    if what in ("viewdirs", "zero_direction"):
        assert bool(torch.isnan(ref[rows][:, :3]).all()) and not bool(torch.isnan(ref[rows][:, 3:]).any())
    _check(got, ref, prec, f"{what}={value} {prec}")
    assert torch.equal(got[~rows], ref_clean[~rows]), "a bad sample changed another sample"


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("prec", ["fp16x3", "bf16"])
def test_non_finite_hashgrid_point_is_reported(prec, value):
    """The hash grid clamps every point into its box by design (a NaN one to the corner (0,0,0), whose features are
    finite): a non-finite point is flagged before the clamp, and every other sample is unchanged."""
    cfg = hash_cfg("cfg2", hash_levels=8, hash_features=2, hash_log2_size=14, precision=prec)
    net = _net(cfg).to(DEV)
    pts, vd = (t.to(DEV) for t in _inputs(S_SMALL, seed=19))
    clean = net(pts, vd)
    assert _status(net) == 0
    bp = pts.clone()
    bp[BAD, 1] = float(value)
    got = net(bp, vd)
    assert _status(net) & 1
    keep = torch.arange(S_SMALL, device=DEV) != BAD
    assert torch.equal(got[keep], clean[keep])


# name: cfg overrides, the module path of the layer whose bias (unit 3, or its only unit) becomes NaN
BIASES = {
    "trunk_regs": ({}, "pts_linears.2"),
    "trunk_last_sigma": ({}, "pts_linears.7"),
    "skip_layer": ({}, "pts_linears.5"),
    "trunk_W64": (dict(W=64), "pts_linears.2"),
    "view_hidden": ({}, "views_linears.0"),
    "semantic_hidden": ({}, "semantic_linears.0"),
    "instance_hidden": ({}, "instance_linears.0"),
    "sigma": ({}, "alpha_linear"),
    "logits": ({}, "semantic_linears.1"),
}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", list(BIASES))
def test_nan_bias_reaches_the_outputs(name, prec):
    """A NaN bias (any mode: biases are fp32 constants nothing else checks): NaN where float64 has NaN, never a silently
    dead unit; the bit set where the NaN enters an operand (trunk and head hidden layers), clear where it stays fp32
    (the view layer's hidden units, sigma, the logits)."""
    over, path = BIASES[name]
    cfg = make_cfg("cfg2", precision=prec, **HEADS, **over)
    net_cpu = _net(cfg)
    with torch.no_grad():
        b = net_cpu.get_submodule(path).bias
        b[min(3, b.shape[0] - 1)] = float("nan")
    net = _to_dev(net_cpu, cfg)
    pts, vd = _inputs(S_SMALL, seed=8)
    got = net(pts.to(DEV), vd.to(DEV))
    ref, ops = _ref(net_cpu, cfg, pts, vd)
    assert bool(torch.isnan(ref).any())
    assert bool(_status(net) & 1) == _flagged(ops, prec), f"{name} {prec}"
    _check(got, ref, prec, f"NaN bias {name} {prec}")


@pytest.mark.parametrize("how", ["loaded", "updated"])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_nan_weight_in_bf16_modes(prec, how):
    """A NaN trunk weight in the bf16 modes (neither the load nor the device-side update refuses one: the bf16 range
    holds every finite weight): reported, and NaN in the outputs as in float64."""
    cfg = make_cfg("cfg2", precision=prec, **HEADS)
    net_cpu = _net(cfg)
    pts, vd = _inputs(S_SMALL, seed=9)
    if how == "loaded":
        with torch.no_grad():
            net_cpu.pts_linears[2].weight[3, 7] = float("nan")
        net = _to_dev(net_cpu, cfg)
    else:
        net = _to_dev(net_cpu, cfg)
        net(pts.to(DEV), vd.to(DEV))
        assert _status(net) == 0
        with torch.no_grad():
            net_cpu.pts_linears[2].weight[3, 7] = float("nan")
            net.pts_linears[2].weight[3, 7] = float("nan")
    got = net(pts.to(DEV), vd.to(DEV))
    ref, ops = _ref(net_cpu, cfg, pts, vd)
    assert _flagged(ops, prec) and _status(net) == 1
    _check(got, ref, prec, f"NaN weight ({how}) {prec}")


# ------------------------------------------------------------------------------------------------ every instantiation
def _comp_rays(R=8, N=32):
    rays, z, _, _ = _dyadic_rays(R, N, seed=13)
    return rays, torch.sort(z, -1).values


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("bad", ["origin_70000", "z_nan"])
def test_compositing_epilogue_reports_one_bad_ray(bad, prec):
    """pnr_mlp_composite (N % 32 == 0) with one bad ray among eight: reported where an operand overflows (a finite
    origin x of 70000 in the fp16 modes, a NaN depth in all), every other ray's maps and weights bit for bit those of
    the launch without it."""
    cfg, net_cpu, net = _heads_net(prec)
    rays, z = _comp_rays()
    br, bz = rays.clone(), z.clone()
    if bad == "origin_70000":
        br[3, 0] = 70000.0
    else:
        bz[3, 5] = float("nan")
    clean = net.forward_composite(rays.to(DEV), z.to(DEV))
    assert _status(net) == 0
    got = net.forward_composite(br.to(DEV), bz.to(DEV))
    _, ops = _ref(net_cpu, cfg, *_pts_of(dict(rays=br, z=bz)))
    want = _flagged(ops, prec)
    assert want == (bad == "z_nan" or prec.startswith("fp16"))
    assert bool(_status(net) & 1) == want
    keep = torch.arange(8) != 3
    for k, v in clean.items():
        n = v.shape[0]
        sel = keep if n == 8 else torch.arange(n) // 32 != 3
        assert torch.equal(got[k][sel.to(DEV)], v[sel.to(DEV)]), k


def _trunk_ops64(net_cpu, cfg, pts, grad_h, scale):
    """float64 trunk: output h, dL/d(trunk input), and the values the backward program writes into operands: the
    embedding, H_0 .. H_{D-2} and every dZ_j * scale."""
    onet = _oracle64(cfg, net_cpu)
    ex = O.embed(pts.double(), cfg.xyz_res).requires_grad_(True)
    h, pres = ex, []
    for i, lin in enumerate(onet.pts_linears):
        pre = lin(h)
        pre.retain_grad()
        pres.append(pre)
        h = F.relu(pre)
        if i == onet.skip:
            h = torch.cat([ex, h], -1)
    h.backward(grad_h.double())
    fwd = [ex.detach()] + [F.relu(p.detach()) for p in pres[:-1]]
    dz = [p.grad * scale for p in pres]
    return h.detach(), ex.grad, fwd, dz


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_trunk_forward_program(prec):
    """pnr_mlp_trunk_forward (the backward programs' forward trunk): 65519 in gamma(x) clear and within tolerance,
    65520 set in fp16x3 only, a NaN point set in both with that sample's h NaN and the others unchanged."""
    cfg = make_cfg("cfg2", precision=prec)
    net_cpu = _net(cfg)
    net = _to_dev(net_cpu, cfg)
    pts, _ = _probe_inputs("x", 65519.0, 65519.0)
    h0 = net.trunk_forward(pts=pts.to(DEV)).cpu()
    assert _status(net) == 0
    href, _, fwd, _ = _trunk_ops64(net_cpu, cfg, pts, torch.zeros(S_SMALL, cfg.W), 1.0)
    _check(h0, href, prec, "trunk forward 65519")
    for v, want in ((65520.0, prec == "fp16x3"), (float("nan"), True)):
        bp = pts.clone()
        bp[BAD, 0] = v
        h = net.trunk_forward(pts=bp.to(DEV)).cpu()
        _, _, fwd, _ = _trunk_ops64(net_cpu, cfg, bp, torch.zeros(S_SMALL, cfg.W), 1.0)
        assert _flagged(fwd, prec) == want
        assert bool(_status(net) & 1) == want, f"trunk forward {v} {prec}"
        keep = torch.arange(S_SMALL) != BAD
        assert torch.equal(h[keep], h0[keep])
        if v != v:
            assert bool(torch.isnan(h[BAD]).all())


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_backward_program_gradient_range(prec):
    """pnr_mlp_backward_trunk: one entry of grad_h * grad_scale = 2^16 (at a unit the last layer keeps, so that it
    enters the operand) sets the bit in fp16x3, 2^15 leaves it clear (float64 confirms no lower layer's |dZ * scale|
    reaches 2^15) and matches float64; a NaN there is reported in both modes, with NaN in exactly the gradient entries
    float64 makes NaN and every other sample unchanged."""
    cfg = make_cfg("cfg2", precision=prec)
    net_cpu = _net(cfg)
    net = _to_dev(net_cpu, cfg)
    pts, _ = _inputs(S_SMALL, seed=10)
    scale = 4.0
    g = torch.randn(S_SMALL, cfg.W, generator=torch.Generator().manual_seed(11)) * 1e-2
    h, _, _, _ = _trunk_ops64(net_cpu, cfg, pts, g, scale)
    unit = int(torch.argmax(h[BAD]))                              # active in the last layer
    assert float(h[BAD, unit]) > 0
    clean = net.backward_trunk(g.to(DEV), pts=pts.to(DEV), grad_scale=scale).cpu()
    assert _status(net) == 0
    for v in (2.0 ** 15 / scale, 2.0 ** 16 / scale, float("nan")):
        gb = g.clone()
        gb[BAD, unit] = v
        got = net.backward_trunk(gb.to(DEV), pts=pts.to(DEV), grad_scale=scale).cpu()
        _, gref, fwd, dz = _trunk_ops64(net_cpu, cfg, pts, gb, scale)
        want = _flagged(fwd + dz, prec)
        assert want == (v != v or (v == 2.0 ** 16 / scale and prec == "fp16x3"))
        assert bool(_status(net) & 1) == want, f"backward {v} {prec}"
        keep = torch.arange(S_SMALL) != BAD
        assert torch.equal(got[keep], clean[keep])
        if v == 2.0 ** 15 / scale:
            assert max(float(d[BAD].abs().max()) for d in dz[:-1]) < 2.0 ** 15
            assert bool((got.double() - gref).abs().max() <= 1e-4 * float(gref.abs().max()))
        if v != v:
            assert torch.equal(torch.isnan(got[BAD]), torch.isnan(gref[BAD]))
            assert bool(torch.isnan(got[BAD]).any())


@pytest.mark.parametrize("prec", PRECS)
def test_render_fused_raises_on_overflow(prec):
    """pnr_render_fused through Renderer.render: a ray whose origin x is 70000 (near / far given, no primitives, no fine
    pass) raises in the fp16 modes and renders in the bf16 modes."""
    cfg = make_cfg("cfg2", precision=prec, N_importance=0)
    net = S.init_network_weights(make_network(cfg), seed=2).to(DEV)
    R = 64
    rays = torch.cat([torch.randn(R, 3, generator=torch.Generator().manual_seed(1)),
                      torch.tensor([[0.6, 0.0, 0.8]]).expand(R, 3)], -1)
    rays[17, 0] = 70000.0
    batch = dict(rays=rays.to(DEV), near=torch.full((R,), 0.5, device=DEV), far=torch.full((R,), 4.0, device=DEV))
    renderer = PN.make_renderer(cfg, net)
    if prec.startswith("fp16"):
        with pytest.raises(_capi.PnrError, match="activation left the range"):
            renderer.render(batch)
    else:
        out = renderer.render(batch)
        assert bool(torch.isfinite(out["rgb_map"]).all())
    assert _status(net) == 0


# ------------------------------------------------------------------------------------------------ placement
@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_bad_sample_anywhere_in_a_large_launch(prec):
    """S = 64 * sms * 2 + 17 samples on a grid of sms CTAs (round-robin tiles, a ragged last tile): a NaN point, and in
    fp16x3 a coordinate of 65520, at sample 0, 63, 64, in the last CTA's last tile and at S - 1 is reported and stays in
    its row; the prefix launch of S - 1 samples (whose tail rows repeat sample S - 2, never S - 1) is clear."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S_ = 64 * sms * 2 + 17
    cfg = make_cfg("cfg2", precision=prec)
    net = S.init_network_weights(make_network(cfg), seed=3).to(DEV)
    pts, vd = (t.to(DEV) for t in _inputs(S_, seed=14))
    clean = net(pts, vd)
    assert _status(net) == 0
    values = [float("nan")] + ([65520.0] if prec == "fp16x3" else [])
    for pos in (0, 63, 64, 64 * (2 * sms - 1) + 5, S_ - 1):
        for v in values:
            bp = pts.clone()
            bp[pos, 0] = v
            got = net(bp, vd)
            assert _status(net) & 1, f"sample {pos} value {v}"
            keep = torch.arange(S_, device=DEV) != pos
            assert torch.equal(got[keep], clean[keep]), f"sample {pos} value {v}"
            if v != v:
                assert bool(torch.isnan(got[pos]).all())
            if pos == S_ - 1:
                assert torch.equal(net(bp[:-1].contiguous(), vd[:-1].contiguous()), clean[:-1])
                assert _status(net) == 0, "the prefix launch read past its samples"


# ------------------------------------------------------------------------------------------------ the sticky word
def test_status_is_sticky_until_read_with_reset():
    cfg = make_cfg("cfg2")
    net = S.init_network_weights(make_network(cfg), seed=3).to(DEV)
    pts, vd = (t.to(DEV) for t in _inputs(S_SMALL, seed=15))
    bp = pts.clone()
    bp[BAD, 2] = float("nan")
    net(bp, vd)
    for _ in range(2):
        net(pts, vd)
    assert _status(net, reset=False) == 1 and _status(net, reset=False) == 1
    assert _status(net) == 1 and _status(net) == 0
    net(pts, vd)
    assert _status(net) == 0


def test_coarse_and_fine_contexts_keep_separate_words():
    """An overflow in the fine network alone sets only its word, and Renderer.render still raises."""
    cfg = make_cfg("cfg1", N_importance=16)
    coarse = S.init_network_weights(make_network(cfg), seed=1).to(DEV)
    fine = S.init_network_weights(make_network(cfg), seed=2)
    with torch.no_grad():
        fine.pts_linears[1].bias[3] = 70000.0
    fine = fine.to(DEV)
    pts, vd = (t.to(DEV) for t in _inputs(S_SMALL, seed=16))
    coarse(pts, vd)
    fine(pts, vd)
    assert _status(coarse) == 0 and _status(fine) == 1
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, rows=2).items()}
    with pytest.raises(_capi.PnrError, match="activation left the range"):
        PN.make_renderer(cfg, coarse, fine).render(batch)
    assert _status(coarse) == 0


def test_cuda_graph_replay_sets_the_bit_each_time():
    """A CUDA graph captured around a flagged launch sets the bit again on every replay after a reset; replayed on clean
    inputs in the same buffers it leaves it clear."""
    cfg = make_cfg("cfg1")
    net = S.init_network_weights(make_network(cfg), seed=1).to(DEV)
    pts, vd = (t.to(DEV) for t in _inputs(S_SMALL, seed=17))
    clean = pts.clone()
    pts[BAD, 0] = float("inf")
    net(pts, vd)
    torch.cuda.synchronize()
    assert _status(net) == 1
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            out = net(pts, vd)
    torch.cuda.current_stream().wait_stream(side)
    assert _status(net) == 0                                        # capture launches nothing
    for _ in range(2):
        graph.replay()
        assert _status(net) == 1
        assert bool(torch.isnan(out[BAD]).all())
    pts.copy_(clean)
    graph.replay()
    assert _status(net) == 0 and bool(torch.isfinite(out).all())


# ------------------------------------------------------------------------------------------------ bit 1
WEIGHTS = [65505.0, -65505.0, math.inf, -math.inf, math.nan]


@pytest.mark.parametrize("prec", ["fp16x3", "fp16"])
def test_update_reports_a_packed_weight_outside_fp16(prec):
    """pnr_update_weights in the fp16 modes: bit 1 for a packed weight of +-65505, +-Inf or NaN, and for a fold that
    overflows though its inputs are in range; check_range raises the weight message; the bit survives a later valid
    update until it is read.  +-65504 leaves it clear and is packed exactly: it multiplies a semantic hidden unit that
    carries the integer x0 = 519 (the chain of the threshold probes), and the outputs are within tolerance of float64."""
    cfg = make_cfg("cfg2", precision=prec, **HEADS)
    net_cpu = _chain(_net(cfg), None, head="semantic_linears", top=0.0)
    net = _to_dev(net_cpu, cfg)
    pts, vd = _probe_inputs("x", 519.0, 519.0)
    gp, gv = pts.to(DEV), vd.to(DEV)
    net(gp, gv)
    assert _status(net) == 0
    w = net.semantic_linears[1].weight
    keep = float(w.detach()[0, CHAIN_J])
    for v in WEIGHTS:
        with torch.no_grad():
            w[0, CHAIN_J] = v
        net(gp, gv)
        assert _status(net, reset=False) & 2, f"weight {v}"
        with torch.no_grad():
            w[0, CHAIN_J] = keep                                        # a valid update: the bit stays until read
        net(gp, gv)
        assert _status(net, reset=False) & 2
        with pytest.raises(_capi.PnrError, match="outside the fp16 range"):
            net.check_range()
        assert _status(net) == 0
    for v in (65504.0, -65504.0):
        with torch.no_grad():
            w[0, CHAIN_J] = v
            net_cpu.semantic_linears[1].weight[0, CHAIN_J] = v
        got = net(gp, gv)
        assert _status(net) == 0, f"weight {v}"
        ref, _ = _ref(net_cpu, cfg, pts, vd)
        _check(got, ref, prec, f"weight {v}")
    with torch.no_grad():
        net.feature_linear.weight.fill_(300.0)
        net.views_linears[0].weight[:, :cfg.W].fill_(300.0)      # folded: 256 * 300 * 300 = 2.3e7
    net(gp, gv)
    assert _status(net) & 2
