"""GPU: the trunk backward (pnr_mlp_backward_trunk) element by element against the float64 bound of
tests/oracle_bound.backward_bound, pinned to the kernel's own ReLU masks, and the trunk's weight gradients
(network_backward: pnr_wgrad on the stash) against the float64 pinned reference.

Regimes: those of tests/test_cpu_operand_split.py (default init; layer 0, the skip layer and the last layer twinned
down by 2^4 .. 2^16 and up to the fp16 range; hash tables of +-1e-4, +-1e-2, +-1; KITTI-360 coordinates), in fp16x3 and
bf16x3, crossed with three grad_h regimes (`grad_regime`: O(1) at the default grad_scale; 2^-20 O(1) unscaled, whose fp16
parts are subnormal; columns spread over 2^-12 .. 2^4).  Every case is checked in this order, so that a failure names
its link:
  1. the stash's H_i (i < D-1) within the forward bound of layer i's activation;
  2. the decision guard: the kernel's masks (H_i > 0; dZ_{D-1} != 0, grad_h has no zero) agree with the sign of the
     float64 pre-activation wherever it clears its bound (the flips within the bound are counted and printed);
  3. the last layer's mask equals pnr_mlp_trunk_forward's h > 0 bit for bit, and the dZ_{D-1} slot is M_{D-1} grad_h
     bit for bit;
  4. every dZ_j slot and d(trunk input) within backward_bound, NaN patterns equal.
Range check: where float64 says a scaled intermediate dZ_j reaches 65520 (fp16x3, down twins at the default scale), bit 0
of pnr_status must be set; the case then reruns at the largest scale that keeps every scaled dZ_j below 2^14, with status
0, and that run is held to the bound.
grad_emb and the stash are views inside larger NaN-filled buffers: nothing outside them may be written.
The worst |err| / B of every link is printed (pytest -s)."""
import math

import pytest
import torch

from oracle_bound import backward_bound, wgrad_bound
from oracle_hashgrid import hash_cfg
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as S
from test_cpu_operand_split import (GRADS, REGIMES, apply_twin, backward_ratios, default_grad_scale, fp16_safe_scale,
                                    grad_regime, make_regime, ratio, regime_points, stash_masks, trunk_input)
from test_gpu_config_space import _dyadic_rays

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRECISIONS = ["fp16x3", "bf16x3"]
N = 64 * 132 * 2 + 17                       # more tiles than an H100 SXM has SMs, twice over, plus a tail
COUNTS = [1, 63, 64, 65, 127, 128, 129]     # shorter runs: prefixes of the same samples
PAD = 1024                                  # NaN floats before and after each output view
CHUNK = 256                                 # samples per chunk of the float64 bound


def run_backward(net, grad_h, gs, pts=None, rays=None, z=None):
    """pnr_mlp_backward_trunk through the C ABI, grad_emb and the stash as views inside larger NaN-filled buffers.
    Returns (d(trunk input) [S, E], stash [2D-1, S, W], range status of the launch)."""
    R, Nz, S_ = (pts.shape[0], 1, pts.shape[0]) if pts is not None else (z.shape[0], z.shape[1], z.numel())
    D, W, Ex = net.D, net.W, net.in_dim
    ld = (Ex + 15) // 16 * 16
    eb = torch.full((S_ * ld + 2 * PAD,), float("nan"), device=DEV)
    sb = torch.full(((2 * D - 1) * S_ * W + 2 * PAD,), float("nan"), device=DEV)
    emb = eb[PAD:PAD + S_ * ld].view(S_, ld)
    st = sb[PAD:PAD + (2 * D - 1) * S_ * W].view(2 * D - 1, S_, W)
    ctx = net.pack(torch.device(DEV))
    net.range_status()
    f32 = torch.float32
    _capi.check(_capi.lib().pnr_mlp_backward_trunk(
        ctx, _capi.ptr(pts, f32, "pts"), _capi.ptr(rays, f32, "rays"), _capi.ptr(z, f32, "z"), R, Nz,
        grad_h.data_ptr(), float(gs), emb.data_ptr(), ld, st.data_ptr(), None, _capi.stream_ptr()), "pnr_mlp_backward_trunk")
    status = net.range_status()
    for buf, n, what in ((eb, S_ * ld, "grad_emb"), (sb, (2 * D - 1) * S_ * W, "stash")):
        assert bool(torch.isnan(buf[:PAD]).all() and torch.isnan(buf[PAD + n:]).all()), f"{what}: written outside its rows"
    return emb[:, :Ex], st, status


def pinned_bound(name, net, precision, ex, e_ex, grad_h, gs, st, h_fwd):
    """Links 1-3 of the module docstring; returns backward_bound pinned to the kernel's masks."""
    D = net.D
    H = [st[i].double() for i in range(D - 1)]
    masks = stash_masks(H, st[D - 1])
    b = backward_bound(net, precision, ex.to(DEV), e_ex.to(DEV), grad_h.to(DEV), gs, masks, chunk=CHUNK)
    rH = {f"H{i}": float(ratio(H[i], b["H"][i], b["E_H"][i]).max()) for i in range(D - 1)}
    assert max(rH.values()) <= 1.0, f"{name}: a stash H slot outside the forward bound {rH}"
    flips = 0
    for i in range(D):
        differ = (masks[i] > 0) != (b["pre"][i] > 0)
        clear = b["pre"][i].abs() > b["E_pre"][i]
        assert not bool((differ & clear).any()), f"{name}: layer {i}'s mask contradicts a pre-activation clear of its bound"
        flips += int(differ.sum())
    assert torch.equal(st[D - 1] != 0, h_fwd > 0), f"{name}: the last layer's mask differs from trunk_forward's h > 0"
    assert torch.equal(st[D - 1], torch.where(h_fwd > 0, grad_h, torch.zeros_like(grad_h))), f"{name}: dZ_{D - 1} slot"
    b["report"] = f"flips={flips} " + " ".join(f"{k}={v:.3g}" for k, v in rH.items())
    return b


def check_within(name, b, d_in, st):
    """Link 4: every dZ_j slot and d(trunk input) within the bound."""
    D = len(b["dZ"])
    r = backward_ratios(b, [st[2 * D - 2 - j].double() for j in range(D)], d_in.double())
    print(f"BWD {name}: {b['report']} " + " ".join(f"{k}={v:.3g}" for k, v in r.items()))
    assert max(r.values()) <= 1.0, f"{name}: an element outside the bound {r}"


def check_case(name, net, precision, ex, e_ex, grad_h, gs, pts=None, rays=None, z=None):
    """One kernel run through links 1-4 and the range check; returns (d_in, stash, grad_scale) of the run held to the
    bound."""
    d_in, st, status = run_backward(net, grad_h, gs, pts=pts, rays=rays, z=z)
    with torch.no_grad():
        h_fwd = net.trunk_forward(pts=pts, rays=rays, z=z)
    b = pinned_bound(name, net, precision, ex, e_ex, grad_h, gs, st, h_fwd)
    over = max(float(d.abs().max()) for d in b["dZ"]) * gs
    if precision == "fp16x3" and over >= 65520.0:
        assert status & 1, f"{name}: a scaled dZ reaches {over:.4g}, but the range check is clear"
    if precision == "fp16x3" and over >= 2.0 ** 14:
        gs = fp16_safe_scale(b, gs)
        name = f"{name} rerun gs=2^{int(math.log2(gs))}"
        d_in, st2, status = run_backward(net, grad_h, gs, pts=pts, rays=rays, z=z)
        assert torch.equal(st2[:net.D - 1], st[:net.D - 1]), f"{name}: the forward half depends on grad_scale"
        st = st2
        b = pinned_bound(name, net, precision, ex, e_ex, grad_h, gs, st, h_fwd)
    assert status == 0, f"{name}: range status {status}"
    check_within(name, b, d_in, st)
    return d_in, st, gs


def _setup(precision, regime, n=N, **over):
    cfg, net = make_regime(precision, regime, **over)
    pts, _ = regime_points(regime, n, seed=11)
    ex, e_ex = trunk_input(cfg, net, pts)
    net, k = apply_twin(net, regime, ex)
    return cfg, net.to(DEV), k, pts, ex, e_ex


@pytest.mark.parametrize("grad", GRADS)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_backward_within_the_bound(regime, precision, grad):
    """Points mode, D = 3, W = 256: the whole run against the bound, and shorter runs as prefixes of it, bit for bit
    for d(trunk input) and for the stash."""
    cfg, net, k, pts, ex, e_ex = _setup(precision, regime)
    grad_h, gs = grad_regime(grad, N, cfg.W, seed=13)
    gp, gg = pts.to(DEV), grad_h.to(DEV)
    d_in, st, gs = check_case(f"{regime[0]} k={k} {precision} {grad}", net, precision, ex, e_ex, gg, gs, pts=gp)
    for m in COUNTS:
        d_m, st_m, _ = run_backward(net, gg[:m].contiguous(), gs, pts=gp[:m].contiguous())
        assert torch.equal(d_m, d_in[:m]) and torch.equal(st_m, st[:, :m]), f"{regime[0]}: {m} samples are not a prefix"


@pytest.mark.parametrize("grad", GRADS)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("D", [8, 9])
def test_deep_backward_within_the_bound(D, precision, grad):
    """The default network (D = 8) and the deepest the backward program accepts (D = 9), default init."""
    cfg, net, k, pts, ex, e_ex = _setup(precision, REGIMES[0], D=D)
    grad_h, gs = grad_regime(grad, N, cfg.W, seed=17)
    check_case(f"D{D} {precision} {grad}", net, precision, ex, e_ex, grad_h.to(DEV), gs, pts=pts.to(DEV))


ENTRY = {"rays": dict(rays=True), "L16F1": dict(hash=(16, 1)), "L16F2": dict(hash=(16, 2)), "L8F4": dict(hash=(8, 4)),
         "L8F8": dict(hash=(8, 8)), "xyz_res0": dict(xyz_res=0), "W64": dict(W=64), "W128": dict(W=128)}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("entry", list(ENTRY))
def test_backward_entry_points_within_the_bound(entry, precision):
    """Rays mode (points o + d z exact in fp32, formed in the kernel), hash grids with F = 1, 2, 4, 8 (table +-1e-2),
    xyz_res = 0, W = 64 and 128; D = 3, O(1) gradients at the default scale."""
    over = dict(ENTRY[entry])
    grid = over.pop("hash", None)
    rays_mode = over.pop("rays", False)
    if grid:
        cfg = hash_cfg("cfg2", hash_levels=grid[0], hash_features=grid[1], hash_log2_size=12, D=3, W=256,
                       precision=precision)
        net = S.init_network_weights(make_network(cfg), seed=1)
        with torch.no_grad():
            g = torch.Generator().manual_seed(101)
            net.xyz_encoder.table.copy_((torch.rand(net.xyz_encoder.table.shape, generator=g) * 2 - 1) * 1e-2)
        pts, _ = regime_points(("table", 1e-2, None, None, 0), N, seed=11)
    else:
        cfg = make_cfg("cfg2", **dict(dict(D=3, W=256), **over, precision=precision))
        net = S.init_network_weights(make_network(cfg), seed=1)
        pts, _ = regime_points(REGIMES[0], N, seed=11)
    if rays_mode:
        rays, z, pts, _ = _dyadic_rays(1301, 13, seed=12)
        kw = dict(rays=rays.to(DEV), z=z.to(DEV))
    else:
        kw = dict(pts=pts.to(DEV))
    ex, e_ex = trunk_input(cfg, net, pts)
    net = net.to(DEV)
    name = f"{entry} {precision}"
    grad_h, gs = grad_regime("unit", pts.shape[0], cfg.W, seed=19)
    gg = grad_h.to(DEV)
    d_in, st, gs = check_case(name, net, precision, ex, e_ex, gg, gs, **kw)
    if rays_mode:       # the kernel forms the same points as the points mode: the same bits
        d_p, st_p, _ = run_backward(net, gg, gs, pts=pts.to(DEV))
        assert torch.equal(d_p, d_in) and torch.equal(st_p, st), f"{name}: rays and points modes differ"
        n5 = 5 * 13
        d_r, st_r, _ = run_backward(net, gg[:n5].contiguous(), gs, rays=kw["rays"][:5].contiguous(), z=kw["z"][:5].contiguous())
        assert torch.equal(d_r, d_in[:n5]) and torch.equal(st_r, st[:, :n5]), f"{name}: 5 rays are not a prefix"


# ------------------------------------------------------------------------------------------------ weight gradients
WG_TOL = {"fp16x3": 1e-4, "bf16x3": 2e-4}      # test_gpu_backward.test_network_backward_every_parameter's tol x RMS


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_trunk_weight_gradients_within_the_bound(regime, precision, monkeypatch):
    """network_backward's pts_linears gradients per element against dW_j = dZ_j^T X_{j-1}, db_j = sum dZ_j in float64,
    pinned to the kernel's masks, within the sum of: pnr_wgrad's own bound on the operands it was given (the stash and
    the encoder's output), the stash's propagated error B_dZ^T (|X| + B_X) + |dZ|^T B_X, and for layer 0's and the skip
    layer's embedded columns the error of pnr_encode (sincosf, 2 ulp: the routine of the fused kernel's gamma(x)); a
    hash grid's h(x) is exact.  Also prints the ratio the RMS-scaled check tol max(|ref|, RMS(ref)) reaches on the
    same elements."""
    from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
    from panopticnerf_b200.lib.train import network_backward
    from panopticnerf_b200.lib.train.mlp_backward import _pow2_from_max
    cfg, net, k, pts, ex, e_ex = _setup(precision, regime)
    name = f"{regime[0]} k={k} {precision}"
    D, skip = cfg.D, cfg.D // 2
    rec = {}
    orig = net.backward_trunk

    def spy(grad_h, **kw):
        out = orig(grad_h, **kw)
        rec["grad_h"], rec["st"], rec["mx"] = grad_h.detach().clone(), out[1], out[2]
        return out
    monkeypatch.setattr(net, "backward_trunk", spy)
    g = torch.Generator().manual_seed(23)
    vd = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=-1)
    d_raw = torch.randn(N, 4, generator=g)
    gp = pts.to(DEV)
    grads = network_backward(net, d_raw.to(DEV), pts=gp, viewdirs=vd.to(DEV))
    status = net.range_status()
    grad_h, st = rec["grad_h"], rec["st"]
    gs = default_grad_scale(grad_h)
    with torch.no_grad():
        h_fwd = net.trunk_forward(pts=gp)
    b = pinned_bound(name, net, precision, ex, e_ex, grad_h, gs, st, h_fwd)
    if precision == "fp16x3" and max(float(d.abs().max()) for d in b["dZ"]) * gs >= 65520.0:
        assert status & 1, f"{name}: a scaled dZ overflows, but the range check is clear"
        print(f"WGRAD {name}: flagged by the range check (a scaled dZ reaches 65520)")
        return                   # the wrapper's scale follows grad_h alone: these gradients are flagged, not bounded
    assert status == 0, f"{name}: range status {status}"
    with torch.no_grad():
        ex_k = net.xyz_encoder(gp) if net.hashgrid else P.embed(gp, net.Lx)
    exd, e_exd = ex.to(DEV), e_ex.to(DEV)
    scales = _pow2_from_max(rec["mx"][D - 1:])[::-1] if precision == "fp16x3" else [None] * D
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    worst, rms_check = {}, {}
    for j in range(D):
        dZk, dZr, BdZ = st[2 * D - 2 - j].double(), b["dZ"][j], b["B_dZ"][j]
        if j == 0:
            Xk, Xr, BX = ex_k.double(), exd, e_exd
        elif j == skip + 1:
            Xk = torch.cat([ex_k.double(), st[j - 1].double()], 1)
            Xr, BX = torch.cat([exd, b["H"][j - 1]], 1), torch.cat([e_exd, b["E_H"][j - 1]], 1)
        else:
            Xk, Xr, BX = st[j - 1].double(), b["H"][j - 1], b["E_H"][j - 1]
        sc = float(scales[j]) if scales[j] is not None else 1.0
        bW, bb = wgrad_bound(dZk.abs().T @ Xk.abs(), dZk.abs().sum(0), Xk.abs().sum(0), N, cfg.W, precision, sc, sms)
        bW = bW + BdZ.T @ (Xr.abs() + BX) + dZr.abs().T @ BX
        bb = bb + BdZ.sum(0)
        for what, got, ref, B in ((f"W{j}", grads[f"pts_linears.{j}.weight"], dZr.T @ Xr, bW),
                                  (f"b{j}", grads[f"pts_linears.{j}.bias"], dZr.sum(0), bb)):
            err = (got.double() - ref).abs()
            worst[what] = float(ratio(got.double(), ref, B).max())
            floor = WG_TOL[precision] * torch.maximum(ref.abs(), ref.pow(2).mean().sqrt())
            rms_check[what] = float((err / floor).max())
    print(f"WGRAD {name}: " + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    print(f"WGRAD-RMS {name}: " + " ".join(f"{k}={v:.3g}" for k, v in rms_check.items()))
    assert max(worst.values()) <= 1.0, f"{name}: a weight gradient outside its bound {worst}"
