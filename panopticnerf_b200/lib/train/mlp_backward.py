"""Backward of `Network.forward` (SURVEY 8(f) rank 2): dL/d(parameters) from dL/draw.

The work is split where the network splits:
  * the trunk (`pts_linears`: D of the network's GEMM layers, ~80 % of its FLOPs) runs on the fused tensor-core kernel:
    `pnr_mlp_trunk_forward` gives the trunk output h, `pnr_mlp_backward_trunk` recomputes the trunk per tile, runs
    the layers in reverse with the transposed weight stream and keeps every operand of the weight-gradient GEMMs
    (activations H_i, pre-activation gradients dZ_j) in one fp32 stash;
  * every weight / bias gradient - the trunk's dW_j = dZ_j^T H_{j-1} on that stash and those of the layers after the
    trunk - is a split-K GEMM over the samples on the tensor cores (`wgrad` -> pnr_wgrad, csrc/wgrad_wgmma.cu);
  * the layers after the trunk (alpha / feature / view / rgb / the two heads: small GEMMs with K <= W) are
    differentiated layer by layer by autograd on h, each node's forward and input-gradient GEMM on `linear3x` ->
    pnr_linear (csrc/linear_wgmma.cu).  No library GEMM is left on this path.
Nothing here imports the oracle; tests compare every parameter's gradient with autograd through the oracle network."""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from ... import _capi
from ..networks.renderer import panopticnerf_renderer as P

_WGRAD_WS: Dict[Tuple[int, int], torch.Tensor] = {}     # (device, stream) -> scratch of pnr_wgrad (partial products)


def _rows(t: torch.Tensor, name: str) -> torch.Tensor:
    """[S, n] fp32 CUDA matrix whose rows are contiguous (any row stride: column blocks of a wider matrix are views)."""
    if not t.is_cuda:
        raise _capi.PnrError(f"{name} must be a CUDA tensor (panopticnerf_b200 has no CPU fallback)")
    if t.dtype != torch.float32 or t.dim() != 2:
        raise _capi.PnrError(f"{name} must be a 2-D float32 tensor, got {t.dtype} {tuple(t.shape)}")
    if (t.shape[1] > 1 and t.stride(1) != 1) or (t.shape[0] > 1 and t.stride(0) < t.shape[1]):
        t = t.contiguous()
    return t


def wgrad(dz: torch.Tensor, x: torch.Tensor, bias: bool = True, precision: str = "bf16x3",
          scale: Optional[torch.Tensor] = None):
    """(dW [No, Ni], db [No] or None) = (dz^T @ x, dz.sum(0)) for dz [S, No], x [S, Ni] (fp32, No <= 256): the weight
    and bias gradient of y = x W^T + b from dz = dL/dy, on the tensor cores (pnr_wgrad: 16-bit hi / lo operand parts,
    fp32 accumulation in registers, deterministic).  Ni > 256 (the skip and view layers' concatenated inputs) is
    covered by one call per 256-column block of x; neither dz^T nor a split copy of an operand is materialised.
    precision "bf16x3": ~2^-17 per product, no scaling needed; "fp16x3": ~2^-21 per product with `scale`, a device
    scalar power of two (`_pow2_scale(dz)`) that keeps the fp16 parts of tiny gradients normal."""
    dz, x = _rows(dz, "wgrad: dz"), _rows(x, "wgrad: x")
    S_, No = dz.shape
    Ni = x.shape[1]
    if x.shape[0] != S_ or x.device != dz.device:
        raise _capi.PnrError(f"wgrad: dz {tuple(dz.shape)} on {dz.device} vs x {tuple(x.shape)} on {x.device}")
    if No > 256:
        raise _capi.PnrError(f"wgrad: {No} output features (the library handles layers up to 256 wide)")
    if precision not in ("fp16x3", "bf16x3"):
        raise _capi.PnrError(f"wgrad: precision {precision!r} (the training path runs in the x3 precisions)")
    L = _capi.lib()
    dW = torch.empty(No, Ni, dtype=torch.float32, device=dz.device)
    db = torch.empty(No, dtype=torch.float32, device=dz.device) if bias else None
    ld_dz = dz.stride(0) if S_ > 1 else No
    ld_x = x.stride(0) if S_ > 1 else Ni
    with torch.cuda.device(dz.device):
        stream = _capi.stream_ptr()
        key = (dz.device.index, stream)
        ws = _WGRAD_WS.get(key)
        if ws is None:
            ws = _WGRAD_WS[key] = torch.empty(int(L.pnr_wgrad_workspace_bytes(256, 256)), dtype=torch.uint8, device=dz.device)
        for c0 in range(0, Ni, 256):
            n = min(256, Ni - c0)
            _capi.check(L.pnr_wgrad(dz.data_ptr(), ld_dz, No, x.data_ptr() + 4 * c0, ld_x, n, S_, _capi.PREC[precision],
                                    _capi.ptr(scale, torch.float32, "scale"), dW.data_ptr() + 4 * c0, Ni,
                                    db.data_ptr() if (bias and c0 == 0) else None, 0, ws.data_ptr(), ws.numel(), stream),
                        "pnr_wgrad")
    return dW, db


_LINEAR_WS: Dict[Tuple[int, int], torch.Tensor] = {}    # (device, stream) -> scratch of pnr_linear (packed weights)


def _pow2_scale(g: torch.Tensor) -> torch.Tensor:
    """Device scalar 2^k that brings max |g| to ~256 (1 when g is all zero / not finite): computed on the device, no
    host synchronisation.  The scaled product is divided by it again in the kernel - exact, it only keeps the fp16
    operand parts of tiny gradients out of the subnormal range."""
    m = torch.linalg.vector_norm(g, ord=float('inf'))                 # max |.| without an |g| temporary
    ok = (m > 0) & torch.isfinite(m)
    k = torch.clamp(torch.round(torch.log2(256.0 / torch.where(ok, m, torch.ones_like(m)))), -100.0, 100.0)
    return torch.where(ok, torch.exp2(k), torch.ones_like(k)).to(torch.float32).reshape(1)


def _pow2_scales(t: torch.Tensor):
    """`_pow2_scale` of every slice t[i] of a [n, S, W] tensor, from one reduction: a list of n device scalars."""
    return _pow2_from_max(torch.linalg.vector_norm(t, ord=float('inf'), dim=(1, 2)))   # max |.| without an |t| temporary


def _pow2_from_max(m: torch.Tensor):
    """A list of device scalars 2^k, one per entry of m [n] (max |.| of n tensors), bringing each maximum to ~256."""
    ok = (m > 0) & torch.isfinite(m)
    k = torch.clamp(torch.round(torch.log2(256.0 / torch.where(ok, m, torch.ones_like(m)))), -100.0, 100.0)
    v = torch.where(ok, torch.exp2(k), torch.ones_like(k)).to(torch.float32).contiguous()
    return [v[i:i + 1] for i in range(v.shape[0])]


def linear3x(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, relu: bool = False,
             transposed: bool = False, precision: str = "fp16x3", scale: Optional[torch.Tensor] = None,
             out_cols: int = 0) -> torch.Tensor:
    """act(x @ weight.T + bias) [S, N] for x [S, K], weight [N, K] - or x @ weight for weight [K, N] with
    transposed=True (the input gradient of a linear layer) - on the tensor cores (pnr_linear, csrc/linear_wgmma.cu:
    16-bit hi / lo operand parts, hi.hi + lo.hi + hi.lo, fp32 accumulation).  K <= 512; more than 256 outputs run as
    one call per 256-column block of the result.
    scale: device scalar power of two applied to x inside the kernel and removed from the result (gradients).
    out_cols > N: the result is returned inside a [S, out_cols] buffer whose extra columns are zero (rows padded to a
    multiple of 4 floats keep the kernels on their 16-byte load / store paths)."""
    x = _rows(x, "linear3x: x")
    w = _rows(weight, "linear3x: weight")
    S_, K = x.shape
    N = w.shape[1] if transposed else w.shape[0]
    if (w.shape[0] if transposed else w.shape[1]) != K or w.device != x.device:
        raise _capi.PnrError(f"linear3x: x {tuple(x.shape)} vs weight {tuple(weight.shape)} (transposed={transposed})")
    if precision not in ("fp16x3", "bf16x3"):
        raise _capi.PnrError(f"linear3x: precision {precision!r} (the training path runs in the x3 precisions)")
    if K > 512:
        raise _capi.PnrError(f"linear3x: K = {K} inputs (pnr_linear handles up to 512)")
    L = _capi.lib()
    ld_y = max(N, int(out_cols))
    y = torch.empty(S_, ld_y, dtype=torch.float32, device=x.device)
    if ld_y > N:
        y[:, N:].zero_()
    b = bias.detach().to(torch.float32).contiguous() if bias is not None else None
    ld_w = w.stride(0) if w.shape[0] > 1 else w.shape[1]
    with torch.cuda.device(x.device):
        stream = _capi.stream_ptr()
        key = (x.device.index, stream)
        ws = _LINEAR_WS.get(key)
        if ws is None:
            ws = _LINEAR_WS[key] = torch.empty(int(L.pnr_linear_workspace_bytes(256, 512)), dtype=torch.uint8, device=x.device)
        for c0 in range(0, N, 256):      # more than 256 outputs (the view layer's 283-wide input gradient): column blocks
            n = min(256, N - c0)
            w_ptr = w.data_ptr() + 4 * (c0 if transposed else c0 * ld_w)
            _capi.check(L.pnr_linear(x.data_ptr(), x.stride(0) if S_ > 1 else K, K, w_ptr, ld_w, int(transposed),
                                     (b.data_ptr() + 4 * c0) if b is not None else None, n, S_, int(relu), _capi.PREC[precision],
                                     _capi.ptr(scale, torch.float32, "scale"), y.data_ptr() + 4 * c0, ld_y, ws.data_ptr(), ws.numel(),
                                     stream), "pnr_linear")
    return y


class _Linear3x(torch.autograd.Function):
    """F.linear whose three GEMMs run on the library's tensor-core kernels: forward and dL/dx through pnr_linear
    (the network's operand format; the gradient scaled by a power of two), dL/dW and dL/db through pnr_wgrad."""

    @staticmethod
    def forward(ctx, x, weight, bias, precision):
        # x may carry zero columns behind the layer's inputs (rows padded to a multiple of 4 floats: `_tail`)
        ctx.save_for_backward(x, weight)
        ctx.precision = precision
        return linear3x(x[:, :weight.shape[1]], weight, bias, precision=precision)

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        g = _rows(g, "gradient")          # column blocks of dL/draw arrive as row-strided views: read in place, no copy
        sc = _pow2_scale(g) if ctx.precision == "fp16x3" else None      # one scale for both gradient GEMMs of the layer
        dx = (linear3x(g, weight, transposed=True, precision=ctx.precision, scale=sc, out_cols=x.shape[1])
              if ctx.needs_input_grad[0] else None)
        dW, db = wgrad(g, x[:, :weight.shape[1]], precision=ctx.precision, scale=sc)
        return dx, dW, db, None


def _lin(layer, x, precision):
    return _Linear3x.apply(x, layer.weight, layer.bias, precision)


def _tail(net, h: torch.Tensor, ed: torch.Tensor) -> torch.Tensor:
    """raw from the trunk output: the reference Network.forward after `pts_linears` (same module names)."""
    pr = net.precision if net.precision in ("fp16x3", "bf16x3") else "fp16x3"
    sigma = _lin(net.alpha_linear, h, pr)
    feat = _lin(net.feature_linear, h, pr)
    pad = (-(feat.shape[1] + ed.shape[1])) % 4            # rows of the concatenated input padded to 16 bytes
    parts = [feat, ed] + ([feat.new_zeros(feat.shape[0], pad)] if pad else [])
    g = F.relu(_lin(net.views_linears[0], torch.cat(parts, -1), pr))
    outs = [_lin(net.rgb_linear, g, pr), sigma]
    if net.C > 0:
        outs.append(_lin(net.semantic_linears[1], F.relu(_lin(net.semantic_linears[0], h, pr)), pr))
    if net.K > 0:
        outs.append(_lin(net.instance_linears[1], F.relu(_lin(net.instance_linears[0], h, pr)), pr))
    return torch.cat(outs, -1)


def network_backward(net, d_raw: torch.Tensor, pts: Optional[torch.Tensor] = None, viewdirs: Optional[torch.Tensor] = None,
                     rays: Optional[torch.Tensor] = None, z: Optional[torch.Tensor] = None,
                     return_input_grad: bool = False) -> Dict[str, torch.Tensor]:
    """{parameter name: gradient} of `net` for dL/draw = d_raw [S, 4+C+K], samples given as (pts, viewdirs) [S,3] each
    or as (rays [R,6], z [R,N]).  With return_input_grad also 'embedded_xyz': dL/d(trunk input) [S, net.in_dim] (gamma(x),
    or h(x) of a hash-grid network, whose table gradient 'xyz_encoder.table' comes from it through pnr_hashgrid_backward)."""
    if pts is None:
        o, d = rays[:, None, :3], rays[:, None, 3:]
        pts_ = (o + d * z[..., None]).reshape(-1, 3)                 # the kernel forms the same points (mul, then add)
        vd = (rays[:, 3:] / rays[:, 3:].norm(dim=-1, keepdim=True))[:, None, :].expand(-1, z.shape[1], -1).reshape(-1, 3)
    else:
        pts_, vd = pts.reshape(-1, 3), viewdirs.reshape(-1, 3)
    S_ = pts_.shape[0]
    d_raw = d_raw.reshape(S_, -1).to(torch.float32)
    h = net.trunk_forward(pts=pts, rays=rays, z=z).requires_grad_(True)
    ed = P.embed(vd.contiguous(), net.Ld)
    tail_named = [(n, p) for n, p in net.named_parameters() if not n.startswith(("pts_linears.", "xyz_encoder."))]
    with torch.enable_grad():
        raw = _tail(net, h, ed)
        g = torch.autograd.grad(raw, [h] + [p for _, p in tail_named], d_raw, allow_unused=True)
    grads = {n: (gi if gi is not None else torch.zeros_like(p)) for (n, p), gi in zip(tail_named, g[1:])}
    d_emb, st, st_max = net.backward_trunk(g[0].contiguous(), pts=pts, rays=rays, z=z, stash=True, absmax=True)
    if net.hashgrid:             # h(x) of the same points (pnr_hashgrid_encode: the features the fused kernel gathered)
        with torch.no_grad():
            ex = net.xyz_encoder(pts_.contiguous())
        grads["xyz_encoder.table"] = net.xyz_encoder.table_grad(pts_, d_emb)
    else:
        ex = P.embed(pts_.contiguous(), net.Lx)
    D = net.D
    pr = net.precision if net.precision in ("fp16x3", "bf16x3") else "fp16x3"
    # fp16 parts: one power-of-two scale per dZ_j, from the maxima the backward kernel collected while writing the stash
    scales = _pow2_from_max(st_max[D - 1:])[::-1] if pr == "fp16x3" else [None] * D
    for j in range(D):
        dZ = st[2 * D - 2 - j]
        if j == net.skip + 1:        # input [gamma(x) or h(x), H_{j-1}]: two column blocks of dW, no concatenated copy
            dWx, db = wgrad(dZ, ex, precision=pr, scale=scales[j])
            dW = torch.cat([dWx, wgrad(dZ, st[j - 1], bias=False, precision=pr, scale=scales[j])[0]], -1)
        else:
            dW, db = wgrad(dZ, ex if j == 0 else st[j - 1], precision=pr, scale=scales[j])
        grads[f"pts_linears.{j}.weight"], grads[f"pts_linears.{j}.bias"] = dW, db
    if return_input_grad:
        grads["embedded_xyz"] = d_emb
    return grads


class _NetworkFn(torch.autograd.Function):
    """raw = Network.forward(pts, viewdirs) on the fused kernel, differentiable w.r.t. the network's parameters."""

    @staticmethod
    def forward(ctx, net, pts, viewdirs, *params):
        ctx.net, ctx.names = net, [n for n, _ in net.named_parameters()]
        ctx.save_for_backward(pts, viewdirs)
        with torch.no_grad():
            return net.forward(pts, viewdirs)

    @staticmethod
    def backward(ctx, d_raw):
        pts, viewdirs = ctx.saved_tensors
        g = network_backward(ctx.net, d_raw.contiguous(), pts=pts.reshape(-1, 3).contiguous(),
                             viewdirs=viewdirs.reshape(-1, 3).contiguous())
        return (None, None, None) + tuple(g[n] for n in ctx.names)


class _NetworkRaysFn(torch.autograd.Function):
    """raw [R,N,CH] = Network.forward_rays(rays, z) on the fused kernel, differentiable w.r.t. the parameters."""

    @staticmethod
    def forward(ctx, net, rays, z, *params):
        ctx.net, ctx.names = net, [n for n, _ in net.named_parameters()]
        ctx.save_for_backward(rays, z)
        with torch.no_grad():
            return net.forward_rays(rays, z)

    @staticmethod
    def backward(ctx, d_raw):
        rays, z = ctx.saved_tensors
        g = network_backward(ctx.net, d_raw.contiguous(), rays=rays, z=z)
        return (None, None, None) + tuple(g[n] for n in ctx.names)


def network_forward_rays_autograd(net, rays: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """`net.forward_rays(rays, z)` (points and view directions formed in the kernel) with gradients to the parameters."""
    return _NetworkRaysFn.apply(net, rays.contiguous(), z.contiguous(), *[p for _, p in net.named_parameters()])


def training_step(net, rays: torch.Tensor, z: torch.Tensor, batch: Dict[str, torch.Tensor], weights=(1.0, 0.1, 1.0, 1.0),
                  white_bkgd: bool = False, sem_is_prob: bool = False, sample_box: Optional[torch.Tensor] = None,
                  box_sem: Optional[torch.Tensor] = None, mask_outside: bool = False):
    """One pass of the reference NetworkWrapper's job for one set of samples: raw = net(rays, z) (fused MLP kernel),
    maps = raw2outputs (compositing kernel), loss terms (loss kernel), and back: dL/dmaps (loss kernel) -> dL/draw
    (pnr_composite_backward) -> dL/dparameters (network_backward).  Leaves the gradients in `p.grad` like
    `loss.backward()` does; returns (total, terms).  Depths z are treated as constants (the sampler is not
    differentiated, as in the reference)."""
    from .losses import panoptic_losses
    raw = network_forward_rays_autograd(net, rays, z)
    out = P.raw2outputs_autograd(raw, z, rays[:, 3:].contiguous(), white_bkgd=white_bkgd, num_classes=net.C,
                                 num_instances=net.K, sample_box=sample_box, box_sem=box_sem, mask_outside=mask_outside)
    total, terms = panoptic_losses(out, batch, weights, sem_is_prob=sem_is_prob)
    total.backward()
    return total.detach(), terms


def network_forward_autograd(net, pts: torch.Tensor, viewdirs: torch.Tensor) -> torch.Tensor:
    """`net(pts, viewdirs)` whose result back-propagates into `net.parameters()` through `network_backward`."""
    return _NetworkFn.apply(net, pts, viewdirs, *[p for _, p in net.named_parameters()])
