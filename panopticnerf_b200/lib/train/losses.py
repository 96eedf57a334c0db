"""Loss side of the training path (SURVEY 8(f) rank 2; the reference's NetworkWrapper computes these terms with torch
ops on the rendered maps): photometric, depth, 2D pseudo-label cross-entropy on the rendered semantics, the
cross-entropy of the fixed (bounding-primitive) semantics and, optionally, the instance term (softmax cross-entropy of
the rendered instance logits against the dominant bounding primitive's slot) - values and map gradients from ONE
kernel family (`pnr_losses`), exposed as an autograd node so that `loss.backward()` continues into
`raw2outputs_autograd` (pnr_composite_backward)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import torch

from ... import _capi

_MAPS = ("rgb_map", "rgb_map0", "depth_map", "semantic_map", "fixed_semantic_map")


def _run(maps: Dict[str, Optional[torch.Tensor]], rgb_gt, depth_gt, label, label_weight, w, sem_is_prob: bool, eps: float,
         inst=None, inv_n=None):
    """inst = (instance_map, fixed_instance_map, w_inst, inst_min_weight) turns the instance term on: w then holds
    four weights and the result has a fifth term, the instance map's gradient and (n_inst, inst_label).
    inv_n = (inv_n_rgb, inv_n_depth, inv_n_sem): the normalisers of the first four terms given by the caller (a
    data-parallel shard uses 1 / the global batch's counts) instead of 1 / this batch's counts, which are then not
    read from the device."""
    ref = next(t for t in list(maps.values()) + [inst[0] if inst else None] if t is not None)
    dev, R = ref.device, ref.shape[0]
    keep = {k: (None if t is None else t.detach().to(torch.float32).contiguous()) for k, t in maps.items()}
    tg = {"rgb_gt": rgb_gt, "depth_gt": depth_gt, "label_weight": label_weight}
    keep.update({k: (None if t is None else t.detach().to(dev, torch.float32).contiguous()) for k, t in tg.items()})
    lab = None if label is None else label.detach().to(dev, torch.int32).contiguous()
    Cn = keep["semantic_map"].shape[1] if keep["semantic_map"] is not None else (
        keep["fixed_semantic_map"].shape[1] if keep["fixed_semantic_map"] is not None else 0)
    a = _capi.PnrLossArgs()
    a.R, a.C, a.sem_is_prob = R, Cn, int(bool(sem_is_prob))
    for k in _MAPS + ("rgb_gt", "depth_gt", "label_weight"):
        setattr(a, k, _capi.ptr(keep[k], torch.float32, k) if keep[k] is not None else None)
    a.label = _capi.ptr(lab) if lab is not None else None
    a.w_rgb, a.w_depth, a.w_sem, a.w_fix = [float(x) for x in w[:4]]
    if inv_n is None:
        n_depth = int((keep["depth_gt"] > 0).sum()) if keep["depth_gt"] is not None else 0
        n_sem = int(((lab >= 0) & (lab < Cn)).sum()) if lab is not None else 0
        inv_n = (1.0 / (3 * R), 1.0 / max(n_depth, 1), 1.0 / max(n_sem, 1))
    a.inv_n_rgb, a.inv_n_depth, a.inv_n_sem = (float(x) for x in inv_n)
    a.eps = float(eps)
    per_ray = torch.empty(R, 4, dtype=torch.float32, device=dev)
    grads = {k: (torch.empty_like(keep[k]) if keep[k] is not None else None) for k in _MAPS}
    a.per_ray = _capi.ptr(per_ray)
    for k in _MAPS:
        setattr(a, "d_" + k, _capi.ptr(grads[k]) if grads[k] is not None else None)
    extra = None
    if inst is not None:
        im, fim = (t.detach().to(torch.float32).contiguous() for t in inst[:2])
        per_ray_inst = torch.empty(R, dtype=torch.float32, device=dev)
        inst_label = torch.empty(R, dtype=torch.int32, device=dev)
        n_inst = torch.zeros(1, dtype=torch.int32, device=dev)
        grads["instance_map"] = torch.empty_like(im)
        a.K, a.w_inst, a.inst_min_weight = im.shape[1], float(inst[2]), float(inst[3])
        a.instance_map, a.fixed_instance_map = _capi.ptr(im, name="instance_map"), _capi.ptr(fim, name="fixed_instance_map")
        a.per_ray_inst, a.inst_label, a.n_inst = _capi.ptr(per_ray_inst), _capi.ptr(inst_label), _capi.ptr(n_inst)
        a.d_instance_map = _capi.ptr(grads["instance_map"])
        extra = (n_inst[0], inst_label, per_ray_inst)
    with torch.cuda.device(dev):
        _capi.check(_capi.lib().pnr_losses(C.byref(a), _capi.stream_ptr()), "pnr_losses")
    sums = per_ray.sum(0)
    terms = [sums[0] * a.inv_n_rgb, sums[1] * a.inv_n_depth, sums[2] * a.inv_n_sem, sums[3] * a.inv_n_sem]
    if extra is not None:        # mean over the counted rays, normalised on the device
        terms.append(extra[2].sum() / extra[0].clamp(min=1).to(torch.float32))
    terms = torch.stack(terms)
    total = (terms * torch.tensor([float(x) for x in w[:len(terms)]], device=dev)).sum()
    return total, terms, grads, extra


class PanopticLoss(torch.autograd.Function):
    """total, terms = PanopticLoss.apply(rgb_map, rgb_map0, depth_map, semantic_map, fixed_semantic_map, rgb_gt,
    depth_gt, label, label_weight, (w_rgb, w_depth, w_sem, w_fix), sem_is_prob, eps).  Maps may be None; `terms`
    (the four means, unweighted) is not differentiable.
    Trailing inv_n (see `_run`) and inst_scale - a device fp32 [1] tensor the caller may fill after the forward and
    before the backward, by which the instance map's gradient is multiplied (a data-parallel shard's
    n_inst / the global n_inst, known only once every shard's label pass ran) - default to this batch's normalisation.
    With the instance term - trailing arguments instance_map [R,K], fixed_instance_map [R,K], inst_min_weight and a
    fifth weight w_inst - it returns (total, terms[5], n_inst, inst_label): the number of counted rays (device int32
    scalar) and each ray's target slot (-1 = not counted), neither differentiable."""

    @staticmethod
    def forward(ctx, rgb_map, rgb_map0, depth_map, semantic_map, fixed_semantic_map, rgb_gt, depth_gt, label,
                label_weight, weights, sem_is_prob, eps, instance_map=None, fixed_instance_map=None, inst_min_weight=0.5,
                inv_n=None, inst_scale=None):
        maps = dict(zip(_MAPS, (rgb_map, rgb_map0, depth_map, semantic_map, fixed_semantic_map)))
        inst = None
        if instance_map is not None:
            if fixed_instance_map is None or len(weights) != 5:
                raise ValueError("PanopticLoss: the instance term needs fixed_instance_map and a fifth weight (w_inst)")
            inst = (instance_map, fixed_instance_map, weights[4], inst_min_weight)
        total, terms, grads, extra = _run(maps, rgb_gt, depth_gt, label, label_weight, weights, sem_is_prob, eps, inst,
                                          inv_n)
        ctx.grads = [grads[k] for k in _MAPS] + [grads.get("instance_map")]
        ctx.inst_scale = inst_scale
        ctx.n_in = 17 if (inv_n is not None or inst_scale is not None) else 15 if instance_map is not None else 12
        ctx.mark_non_differentiable(terms)
        if extra is None:
            return total, terms
        ctx.mark_non_differentiable(extra[0], extra[1])
        return total, terms, extra[0], extra[1]

    @staticmethod
    def backward(ctx, g_total, *_g_rest):
        g = tuple(None if g is None else g * g_total for g in ctx.grads)
        if g[5] is not None and ctx.inst_scale is not None:
            g = g[:5] + (g[5] * ctx.inst_scale,)
        return (g[:5] + (None,) * 7 + (g[5], None, None, None, None))[:ctx.n_in]


def panoptic_losses(out: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor],
                    weights: Tuple[float, ...] = (1.0, 0.1, 1.0, 1.0), sem_is_prob: bool = False,
                    eps: float = 1e-8, out_coarse: Optional[Dict[str, torch.Tensor]] = None, inst_min_weight: float = 0.5,
                    inv_n: Optional[Tuple[float, float, float]] = None, inst_scale: Optional[torch.Tensor] = None):
    """Convenience wrapper over a Renderer result: batch keys rgb (gt) [R,3], depth (gt, <= 0 = invalid) [R],
    pseudo_label [R] int (-1 = ignore), pseudo_weight [R] (optional).  Returns (total, {'rgb','depth','sem','fix'}).
    A fifth weight (w_inst) adds the instance term on out's instance_map / fixed_instance_map: the dict then also holds
    'inst', 'n_inst' and 'inst_label'.  inv_n, inst_scale: see PanopticLoss (defaults: this batch's own counts)."""
    g = out.get
    args = (g("rgb_map"), None if out_coarse is None else out_coarse.get("rgb_map"),
            g("depth_map") if "depth" in batch else None,
            g("semantic_map") if "pseudo_label" in batch else None,
            g("fixed_semantic_map") if "pseudo_label" in batch else None,
            batch.get("rgb"), batch.get("depth"), batch.get("pseudo_label"),
            batch.get("pseudo_weight"), tuple(weights), sem_is_prob, eps)
    if len(weights) == 5:
        if g("instance_map") is None or g("fixed_instance_map") is None:
            raise ValueError("panoptic_losses: w_inst given, but the result has no instance_map / fixed_instance_map "
                             "(num_instances > 0 and the primitives' box_inst are needed)")
        more = (inv_n, inst_scale) if (inv_n is not None or inst_scale is not None) else ()
        total, terms, n_inst, inst_label = PanopticLoss.apply(*args, g("instance_map"), g("fixed_instance_map"),
                                                              float(inst_min_weight), *more)
        d = dict(zip(("rgb", "depth", "sem", "fix", "inst"), terms.unbind(0)))
        d.update(n_inst=n_inst, inst_label=inst_label)
        return total, d
    more = (None, None, 0.5, inv_n, inst_scale) if (inv_n is not None or inst_scale is not None) else ()
    total, terms = PanopticLoss.apply(*args, *more)
    return total, dict(zip(("rgb", "depth", "sem", "fix"), terms.unbind(0)))
