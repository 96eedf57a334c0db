"""Float64 oracle of one `NetworkWrapper` iteration with every discontinuous decision supplied ("pinned").
TEST INFRASTRUCTURE ONLY; runs on the CPU or, in float64, on a GPU.

The chain is the oracle's: the network of `oracle/reference_renderer.Network` (or the hash-grid network of
`oracle_hashgrid.py`), `raw2outputs`, `oracle/reference_losses.losses` and `oracle_instance.instance_loss`, written
out again here so that each branch can take a supplied decision instead of its own:
  * every ReLU of the network (trunk layers, view layer, the two head hidden layers) is where(mask, pre, 0);
  * the density ReLU is where(mask, sigma, 0), on sigma + noise * raw_noise_std when there is noise;
  * the depth term is s * (depth - gt) with the sign s supplied;
  * max(p, eps) of the probability semantics and of the fixed semantics is where(branch, p, eps);
  * the instance target of each ray is supplied.
Without decisions (pins=None) each branch takes its own value and the chain is the plain oracle, bit for bit
(tests/test_cpu_train_chain.py).  With decisions from a device, a ReLU unit of width ~1e-5 around zero can no longer
flip a whole sample's row of dW, so every gradient can be compared element by element.

Margin guard: wherever a supplied decision disagrees with the chain's own value (a "flip"), that value must lie
within a margin of the switch point, or `PinError` is raised - a wrong mask from the device is caught, not adopted.
Margins: the ReLUs 3e-5 (fp16x3) / 1e-4 (bf16x3), the clearance `test_network_backward_every_parameter` asks of its
samples (100x / 10x the rounding of the mode); density 1e-4 of the pass's sigma RMS (the forward's tolerance); the
depth sign 1e-4 |depth|, the clamps and the instance target 1e-4 of the ray's opacity (the compositing tolerances).

Points and view directions are formed in fp32 as the fused kernel forms them (o + d z: mul, then add, each rounded;
d / sqrt((dx dx + dy dy) + dz dz), correctly rounded square root and division) and then cast; a hash-grid network's
h(x) is the fp32 oracle encoder's value (the kernel's bit for bit), cast, with the float64 table gradient of the
encoder (linear in the table, whose fp32 interpolation weights are exact)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import reference_renderer as O

F64 = torch.float64
RELU_MARGIN = {"fp16x3": 3e-5, "bf16x3": 1e-4}
STAGE_REL = 1e-4
EDITS = ("w_inst", "drop_coarse_rgb", "mask_forward_only", "head_rows")


class PinError(AssertionError):
    """A supplied decision disagrees with the oracle's own value outside the margin of its switch point."""


def _sqrt_rn(x: torch.Tensor) -> torch.Tensor:
    return torch.from_numpy(np.sqrt(x.detach().to(torch.float32).cpu().contiguous().numpy())).to(x.device)


def form_points(rays: torch.Tensor, z: torch.Tensor):
    """fp32 (pts, viewdirs) [R*N, 3] as `pnr_mlp_forward` forms them from rays [R,6] and depths z [R,N]."""
    rays, z = rays.to(torch.float32), z.to(torch.float32)
    R, N = z.shape
    o, d = rays[:, None, :3], rays[:, None, 3:]
    pts = (o + d * z[..., None]).reshape(-1, 3)
    dd = rays[:, 3:]
    n2 = dd[:, 0] * dd[:, 0]
    n2 = n2 + dd[:, 1] * dd[:, 1]
    n2 = n2 + dd[:, 2] * dd[:, 2]
    vd = dd / _sqrt_rn(n2)[:, None]
    return pts, vd[:, None, :].expand(R, N, 3).reshape(-1, 3)


class _Log:
    """Own decisions and flip counts of one chain run."""

    def __init__(self):
        self.own, self.flips = {}, {}

    def pin(self, key, where, value, own, pinned, margin, what):
        """The decision to use: `own` when pinned is None; else `pinned`, after the margin guard on its flips.
        value: what the switch point is measured on (|value| <= margin where a flip is allowed)."""
        self.own[key] = own
        if pinned is None:
            return own
        pinned = pinned.to(own.device).reshape(own.shape)
        flip = pinned != own
        n = int(flip.sum())
        if n:
            m = margin if not torch.is_tensor(margin) else margin.expand_as(value)[flip]
            far = value.detach()[flip].abs() > m
            if bool(far.any()):
                raise PinError(f"{what}: {int(far.sum())} of {n} supplied decisions differ from float64 where "
                               f"|value| = {float(value.detach()[flip].abs().max()):.3e} is beyond the margin")
        self.flips[where] = self.flips.get(where, 0) + n
        return pinned


def _embed_xyz(net, pts, dtype):
    if not hasattr(net, "xyz_encoder"):
        return O.embed(pts.to(dtype), net.Lx)
    from oracle import reference_panoptic as OP
    e = net.xyz_encoder
    p = pts.detach().to("cpu", torch.float32)
    with torch.no_grad():
        h32 = OP.hashgrid_encode(p, e.aabb.cpu(), e.table.detach().to("cpu", torch.float32), e.base, e.scale)
    h = OP.hashgrid_encode(p, e.aabb.cpu(), e.table, e.base, e.scale)       # the table's gradient, in its dtype
    dev = next(net.pts_linears.parameters()).device
    return (h32.to(dtype) + (h - h.detach()).to(dtype)).to(dev)


def _network(net, ex, ed, log, pins, margin, role):
    """Network.forward of the oracle with each ReLU pinned; pins: {layer name: mask [S, width]} or None."""
    pins = pins or {}

    def relu(pre, name):
        m = log.pin(f"{role}/{name}", role, pre, pre > 0, pins.get(name), margin, f"{role} {name}")
        return torch.where(m, pre, torch.zeros_like(pre))

    h = ex
    for i, lin in enumerate(net.pts_linears):
        h = relu(lin(h), f"pts_linears.{i}")
        if i == net.skip:
            h = torch.cat([ex, h], -1)
    sigma = net.alpha_linear(h)
    feat = net.feature_linear(h)
    g = relu(net.views_linears[0](torch.cat([feat, ed], -1)), "views_linears.0")
    outs = [net.rgb_linear(g), sigma]
    if net.C > 0:
        outs.append(net.semantic_linears[1](relu(net.semantic_linears[0](h), "semantic_linears.0")))
    if net.K > 0:
        outs.append(net.instance_linears[1](relu(net.instance_linears[0](h), "instance_linears.0")))
    return torch.cat(outs, -1)


def _onehot(weights, sample_box, table, n):
    """O._composite_onehot (same operations) on the device of the weights."""
    ids = O._box_ids(sample_box, table)
    valid = (ids >= 0) & (ids < n)
    out = torch.zeros(weights.shape[0], n + 1, dtype=weights.dtype, device=weights.device)
    out.scatter_add_(1, torch.where(valid, ids, torch.full_like(ids, n)), weights)
    return out[:, :n].contiguous()


def _composite(raw, z, rays_d, b, noise, log, pin, role, edit, C, K):
    """O.raw2outputs (same operations, same order) with the density ReLU pinned."""
    sb = b.get(f"sb_{role}")
    dists = z[:, 1:] - z[:, :-1]
    dists = torch.cat([dists, torch.full_like(z[:, :1], 1e10)], -1)
    dists = dists * torch.norm(rays_d[:, None, :], dim=-1)
    rgb = torch.sigmoid(raw[..., :3])
    sig = raw[..., 3]
    std = float(b.get("raw_noise_std", 0.0))
    if std > 0.0:
        sig = sig + noise * std
    margin = STAGE_REL * float(sig.detach().pow(2).mean().sqrt())
    live = log.pin(f"{role}/sigma", role, sig, sig > 0, pin, margin, f"{role} density")
    sig = torch.where(live, sig, torch.zeros_like(sig))
    if b.get("mask_outside") and sb is not None:
        inside = sb.to(sig.device) >= 0
        if edit == "mask_forward_only":        # masked values, but the gradient of the masked samples kept
            sig = sig + torch.where(inside, torch.zeros_like(sig), -sig).detach()
        else:
            sig = torch.where(inside, sig, torch.zeros_like(sig))
    alpha = 1.0 - torch.exp(-sig * dists)
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    weights = alpha * trans
    rgb_map = torch.sum(weights[..., None] * rgb, -2)
    depth_map = torch.sum(weights * z, -1)
    acc_map = torch.sum(weights, -1)
    if b.get("white_bkgd"):
        rgb_map = rgb_map + (1.0 - acc_map[..., None])
    out = {"rgb_map": rgb_map, "depth_map": depth_map, "acc_map": acc_map, "weights": weights, "sigma": sig, "dists": dists}
    if C > 0:
        s = raw[..., 4:4 + C]
        if b.get("sem_activation", "none") == "softmax":
            s = torch.softmax(s, -1)
        out["semantic_map"] = torch.sum(weights[..., None] * s, -2)
    if K > 0:
        out["instance_map"] = torch.sum(weights[..., None] * raw[..., 4 + C:4 + C + K], -2)
    if sb is not None and b.get("box_sem") is not None and C > 0:
        out["fixed_semantic_map"] = _onehot(weights, sb.to(weights.device), b["box_sem"].to(weights.device), C)
    if sb is not None and b.get("box_inst") is not None and K > 0:
        out["fixed_instance_map"] = _onehot(weights, sb.to(weights.device), b["box_inst"].to(weights.device), K)
    return out


def _losses(m1, m0, b, w, eps, log, pins, edit):
    """reference_losses.losses (same operations, same order) with the depth sign and both clamps pinned."""
    dev, dt = m1["rgb_map"].device, m1["rgb_map"].dtype
    R = m1["rgb_map"].shape[0]
    t = lambda k: None if b.get(k) is None else b[k].to(dev)
    rgb_gt, depth_gt, label, conf = t("rgb"), t("depth"), t("pseudo_label"), t("pseudo_weight")
    acc = m1["acc_map"].detach()
    zero = torch.zeros((), dtype=dt, device=dev)
    l_rgb = zero
    l_rgb = l_rgb + ((m1["rgb_map"] - rgb_gt) ** 2).sum() / (3 * R)
    if m0 is not None and edit != "drop_coarse_rgb":
        l_rgb = l_rgb + ((m0["rgb_map"] - rgb_gt) ** 2).sum() / (3 * R)
    l_depth = zero
    if depth_gt is not None:
        ok = depth_gt > 0
        diff = m1["depth_map"] - depth_gt.to(dt)
        s = log.pin("depth_sign", "loss", diff, torch.sign(diff.detach()), pins.get("depth_sign"),
                    STAGE_REL * m1["depth_map"].detach().abs(), "depth sign")
        l_depth = (diff * s.to(dt) * ok).sum() / max(int(ok.sum()), 1)
    l_sem = l_fix = zero
    sem, fix = m1.get("semantic_map"), m1.get("fixed_semantic_map")
    Cn = sem.shape[1] if sem is not None else (fix.shape[1] if fix is not None else 0)
    if label is not None and Cn > 0:
        has = (label >= 0) & (label < Cn)
        n = max(int(has.sum()), 1)
        lab = label.clamp(0, Cn - 1).long()
        conf = conf.to(dt) if conf is not None else torch.ones(R, dtype=dt, device=dev)

        def clamp(p, key):
            br = log.pin(key, "loss", p - eps, p.detach() >= eps, pins.get(key), STAGE_REL * acc, key.replace("_", " "))
            return torch.where(br, p, torch.full_like(p, eps))
        if sem is not None:
            if b.get("sem_activation", "none") == "softmax":
                p = sem.gather(1, lab[:, None])[:, 0]
                l_sem = (-torch.log(clamp(p, "sem_clamp")) * conf * has).sum() / n
            else:
                l_sem = (F.cross_entropy(sem, lab, reduction="none") * conf * has).sum() / n
        if fix is not None:
            p = fix.gather(1, lab[:, None])[:, 0]
            l_fix = (-torch.log(clamp(p, "fix_clamp")) * conf * has).sum() / n
    terms = torch.stack([l_rgb, l_depth, l_sem, l_fix])
    total = (terms * torch.tensor(w[:4], dtype=dt, device=dev)).sum()
    if len(w) < 5 or "instance_map" not in m1 or "fixed_instance_map" not in m1:
        return total, terms
    # oracle_instance.instance_loss with the target supplied
    im, fim = m1["instance_map"], m1["fixed_instance_map"].detach()
    thr = float(b.get("inst_min_weight", 0.5))
    mx = fim.max(1).values
    own = torch.where(mx >= thr, (fim == mx[:, None]).to(torch.int64).argmax(1), torch.full_like(mx, -1, dtype=torch.int64))
    top2 = fim.topk(min(2, fim.shape[1]), 1).values
    gap = torch.minimum((mx - thr).abs(), (top2[:, 0] - top2[:, -1]).abs() if fim.shape[1] > 1 else (mx - thr).abs())
    label_i = log.pin("inst_label", "loss", gap, own, None if pins.get("inst_label") is None else pins["inst_label"].long(),
                      STAGE_REL * acc, "instance target")
    ok = label_i >= 0
    n = int(ok.sum())
    ce = torch.logsumexp(im, 1) - im.gather(1, label_i.clamp(min=0)[:, None])[:, 0]
    inst = torch.where(ok, ce, torch.zeros_like(ce)).sum() / max(n, 1)
    w_inst = w[4] * (1.01 if edit == "w_inst" else 1.0)
    return total + w_inst * inst, torch.cat([terms, inst[None]])


def iteration(nets, b, pins=None, precision="fp16x3", edit=None, raw_from=None):
    """One iteration of the oracle chain on the depths a device sampled.
    nets = (coarse, fine) oracle networks in the chain's dtype (the same object twice for a shared network; fine None
    without a fine pass).  b: rays [R,6] fp32, z_coarse [R,N] and z_fine [R,N+Ni] fp32, sb_coarse / sb_fine int32 tags
    or None, box_sem / box_inst, C, K, options white_bkgd / mask_outside / raw_noise_std / noise_coarse / noise_fine /
    sem_activation, targets rgb / depth / pseudo_label / pseudo_weight, weights (4, or 5 with the instance term),
    inst_min_weight, eps.  pins: {"coarse" / "fine": {layer name or "sigma": mask}, "depth_sign", "sem_clamp",
    "fix_clamp", "inst_label"} or None.  edit: one of EDITS, a deliberate change of the reference (the comparison's
    power is tested with it).  raw_from: {role: raw [R,N,CH]} composited in place of the network's raw (the
    compositing and loss links on a device's own raw; the parameters then get no gradient).
    Returns {"maps": {role: maps}, "total", "terms", "raw": {role}, "d_raw": {role}, "grads": [{name: grad}] per
    distinct network, "own": the chain's own decisions (pins of the same layout), "flips": {role or "loss": count}}."""
    pins = pins or {}
    log = _Log()
    margin = RELU_MARGIN[precision]
    roles = ["coarse"] + (["fine"] if nets[1] is not None else [])
    maps, raws = {}, {}
    for role, net in zip(roles, nets):
        dt = next(net.pts_linears.parameters()).dtype
        dev = next(net.pts_linears.parameters()).device
        z = b[f"z_{role}"]
        R, N = z.shape
        pts, vd = form_points(b["rays"].to(dev), z.to(dev))
        ex, ed = _embed_xyz(net, pts, dt), O.embed(vd.to(dt), net.Ld)
        raw = _network(net, ex, ed, log, pins.get(role), margin, role).reshape(R, N, -1)
        if raw_from is not None:               # the compositing and loss links alone, on a device's raw
            raw = raw_from[role].detach().to(dev, dt).reshape(R, N, -1).requires_grad_(True)
        noise = b.get(f"noise_{role}")
        maps[role] = _composite(raw, z.to(dev, dt), b["rays"][:, 3:].to(dev, dt), b,
                                None if noise is None else noise.to(dev, dt), log, (pins.get(role) or {}).get("sigma"),
                                role, edit, net.C, net.K)
        raws[role] = raw
    m1, m0 = maps[roles[-1]], (maps["coarse"] if len(roles) == 2 else None)
    total, terms = _losses(m1, m0, b, tuple(b["weights"]), float(b.get("eps", 1e-8)), log, pins, edit)
    uniq = [nets[0]] + ([nets[1]] if nets[1] is not None and nets[1] is not nets[0] else [])
    params = [[p for _, p in n.named_parameters()] for n in uniq]
    flat = [p for ps in params for p in ps]
    g = torch.autograd.grad(total, flat + [maps[r]["weights"] for r in roles] + [raws[r] for r in roles], allow_unused=True)
    grads, k = [], 0
    for n, ps in zip(uniq, params):
        d = {}
        for (name, p), gi in zip(n.named_parameters(), g[k:k + len(ps)]):
            d[name] = gi if gi is not None else torch.zeros_like(p)
        grads.append(d)
        k += len(ps)
    if edit == "head_rows":                    # one head's gradient 1 % off on half its rows
        _head_rows(grads[-1])
    own = {}
    for key, v in log.own.items():
        if "/" in key:
            role, name = key.split("/", 1)
            own.setdefault(role, {})[name] = v
        else:
            own[key] = v
    raws = {r: raws[r].detach() for r in roles}
    return {"maps": maps, "total": total.detach(), "terms": terms.detach(), "raw": raws,
            "d_raw": {r: (torch.zeros_like(raws[r]) if x is None else x) for r, x in zip(roles, g[k + len(roles):])},
            "d_weights": {r: (torch.zeros_like(maps[r]["weights"]) if x is None else x) for r, x in zip(roles, g[k:k + len(roles)])},
            "grads": grads, "own": own,
            "flips": log.flips}


# ------------------------------------------------------------------------------------------------ the comparison
def rms(t: torch.Tensor) -> float:
    return float(t.double().pow(2).mean().sqrt()) if t.numel() else 0.0


def param_ratios(got, ref, tol, floor_only=False, extra=None):
    """{name: max |got - ref| / (tol max(|ref|, RMS(ref)))}: every element of every gradient within tol of itself or of
    its tensor's RMS, whichever is larger - the network backward's contract as `test_network_backward_every_parameter`
    asserts it.  floor_only=True holds every element to tol RMS(ref) alone.  extra: {name: per-element bound added}.
    A tensor whose reference is exactly zero must be exactly zero (ratio 0, else inf)."""
    out = {}
    extra = extra or {}
    for name, r in ref.items():
        if name.endswith(":atomic"):
            continue
        r = r.detach().double()
        a = got[name].detach().double().to(r.device)
        assert a.shape == r.shape, (name, a.shape, r.shape)
        if not bool(torch.isfinite(a).all()):
            out[name] = float("inf")
            continue
        s = rms(r)
        if s == 0.0:
            out[name] = 0.0 if bool((a == 0).all()) else float("inf")
            continue
        bound = tol * (torch.full_like(r, s) if floor_only else r.abs().clamp(min=s))
        if name in extra:
            bound = bound + extra[name].detach().double().to(r.device)
        out[name] = float(((a - r).abs() / bound).max())
    return out


def d_raw_bound(res, role, C, K):
    """The bound [R,N,CH] each element of a device's d(loss)/d(raw) is held to around the pinned chain's
    (res["d_raw"][role]): 1e-4 x the ray's largest |ref| in its channel group (rgb, sigma, semantic, instance),
    floored at 1e-6 of the group's RMS - the compositing backward's contract.  The sigma group adds what an fp32
    forward knows of the transmittance: each t_j = 1 - alpha_j + 1e-10 is stored to 2^-24 absolute and every factor is
    <= 1, so T_i and w_i = alpha_i T_i are known to (N + 1) 2^-24 absolute, and dL/dsigma_i =
    delta_i e_i (G_i T_i - sum_{j>i} G_j w_j / t_i), G = dL/dw, e_i = exp(-sigma_i delta_i), carries up to
    (N + 1) 2^-24 delta_i e_i (|G_i| + sum_{j>i} |G_j|).  That term decides on rays opaque from their first samples,
    whose whole sigma gradient is ~1e-10 and 1e-4 of it below what fp32 transmittances resolve."""
    ref = res["d_raw"][role]
    m = res["maps"][role]
    R, N = ref.shape[:2]
    G = res["d_weights"][role].abs()
    later = torch.flip(torch.cumsum(torch.flip(G, [-1]), -1), [-1]) - G
    e = torch.exp(-m["sigma"].detach() * m["dists"])
    bound = torch.zeros_like(ref)
    for sl in (slice(0, 3), slice(3, 4), slice(4, 4 + C), slice(4 + C, 4 + C + K)):
        r = ref[..., sl]
        if r.numel() == 0:
            continue
        per_ray = r.abs().reshape(R, -1).max(1).values.clamp(min=1e-6 * rms(r))
        bound[..., sl] = STAGE_REL * per_ray[:, None, None]
    bound[..., 3] += (N + 1) * 2.0 ** -24 * m["dists"] * e * (G + later)
    return bound


def d_raw_ratio(got, res, role, C, K):
    """max of |got - ref| / d_raw_bound over every element (a zero bound asks for an exact zero)."""
    ref = res["d_raw"][role]
    bound = d_raw_bound(res, role, C, K)
    err = (got.detach().double().to(ref.device).reshape(ref.shape) - ref).abs()
    if not bool((err[bound == 0] == 0).all()):          # nonzero where the reference group is exactly 0
        return float("inf")
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


def network_grads(nets, b, pins, upstream, precision="fp16x3", edit=None):
    """Gradients (one dict per distinct network) of sum over the passes of <raw, upstream[role]> through the pinned
    networks.  With upstream = a device's recorded d(loss)/d(raw) this is the float64 network backward of the
    device's own d_raw: the network-backward link alone.  (The whole chain's gradient differs from it exactly by this
    function applied to the difference of the two d_raw: the chain is linear in d_raw once the decisions are pinned.)
    edit="head_rows" applies that deliberate change here too."""
    log = _Log()
    roles = ["coarse"] + (["fine"] if nets[1] is not None else [])
    uniq = [nets[0]] + ([nets[1]] if nets[1] is not None and nets[1] is not nets[0] else [])
    total, exs, pts_all = 0.0, [], []
    for role, net in zip(roles, nets):
        dt = next(net.pts_linears.parameters()).dtype
        dev = next(net.pts_linears.parameters()).device
        pts, vd = form_points(b["rays"].to(dev), b[f"z_{role}"].to(dev))
        ex, ed = _embed_xyz(net, pts, dt), O.embed(vd.to(dt), net.Ld)
        if hasattr(net, "xyz_encoder"):
            exs.append(ex)
            pts_all.append(pts.detach().to("cpu", torch.float32))
        raw = _network(net, ex, ed, log, pins.get(role), RELU_MARGIN[precision], role)
        total = total + (raw.reshape(-1) * upstream[role].detach().to(raw).reshape(-1)).sum()
    flat = [p for n in uniq for _, p in n.named_parameters()]
    g = iter(torch.autograd.grad(total, flat + exs, allow_unused=True))
    out = [{k: (lambda gi, p: torch.zeros_like(p) if gi is None else gi)(next(g), p) for k, p in n.named_parameters()}
           for n in uniq]
    if edit == "head_rows":
        _head_rows(out[-1])
    if not exs:
        return out
    # an fp32 sum of n terms in any order (the table gradient's atomics) is within (n + 1) 2^-24 sum |term| of the
    # exact one; the terms of entry k are w_k(x) dL/dh(x), so sum |term| = the encoder's gradient on |dL/dh|
    from oracle import reference_panoptic as OP
    e = uniq[0].xyz_encoder
    T = e.table.detach().clone().requires_grad_(True)
    acc, n = 0.0, 0
    for (p, d) in zip(pts_all, g):
        h = OP.hashgrid_encode(p, e.aabb.cpu(), T, e.base, e.scale)
        acc = acc + (h * d.detach().abs().to(h)).sum()
        n += p.shape[0]
    (s_abs,) = torch.autograd.grad(acc, T)
    out[0]["xyz_encoder.table:atomic"] = (n + 1) * 2.0 ** -24 * s_abs
    return out


def _head_rows(d):
    key = "instance_linears.1.weight" if "instance_linears.1.weight" in d else "rgb_linear.weight"
    d[key] = d[key].clone()
    d[key][: (d[key].shape[0] + 1) // 2] *= 1.01


def maps_ratio(got, ref, raw, z, C, K, white_bkgd=False, softmax=False):
    """Each map element within 1e-4 x sum_i |w_i v_i| of its ray (the largest over the map's channels; fixed maps
    floored at the ray's largest weight) plus half an ulp of the value; weights within 1e-4 of the ray's largest:
    the compositing stage's tolerances (test_gpu_stage_limits.test_composite_per_ray_against_float64)."""
    w = ref["weights"].detach()
    R = w.shape[0]
    aw, raw, z = w.abs(), raw.detach(), z.to(w)
    s = {"rgb_map": (aw[..., None] * torch.sigmoid(raw[..., :3])).sum(1), "depth_map": (aw * z.abs()).sum(1),
         "acc_map": aw.sum(1)}
    if white_bkgd:
        s["rgb_map"] = s["rgb_map"] + s["acc_map"][:, None]
    if C > 0:
        v = torch.softmax(raw[..., 4:4 + C], -1) if softmax else raw[..., 4:4 + C].abs()
        s["semantic_map"] = (aw[..., None] * v).sum(1)
        s["fixed_semantic_map"] = aw.sum(1)[:, None].expand(R, C)
    if K > 0:
        s["instance_map"] = (aw[..., None] * raw[..., 4 + C:].abs()).sum(1)
        s["fixed_instance_map"] = aw.sum(1)[:, None].expand(R, K)
    w_max = w.max(1).values
    worst = {}
    for k, sm in s.items():
        if k not in got or k not in ref:
            continue
        per_ray = sm.reshape(R, -1).max(1).values
        if k.startswith("fixed_"):
            per_ray = torch.maximum(per_ray, w_max)
        r = ref[k].detach().reshape(R, -1)
        err = (got[k].detach().double().to(r.device).reshape(R, -1) - r).abs()
        bound = STAGE_REL * per_ray[:, None] + 2.0 ** -24 * r.abs()
        assert bool((err[bound == 0] == 0).all()), f"{k}: nonzero error where the float64 value is exactly 0"
        pos = bound > 0
        worst[k] = float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0
    err = (got["weights"].detach().double().to(w.device) - w).abs()
    bound = STAGE_REL * w_max[:, None].expand_as(err)
    assert bool((err[bound == 0] == 0).all()), "weights: nonzero error where the float64 ray is empty"
    worst["weights"] = float((err[bound > 0] / bound[bound > 0]).max()) if bool((bound > 0).any()) else 0.0
    return worst


def cos_norm(a, b):
    """The criterion these element-wise checks replaced: (cosine, norm ratio) of two gradients."""
    a, b = a.detach().double().reshape(-1), b.detach().double().to(a.device).reshape(-1)
    na, nb = float(a.norm()), float(b.norm())
    if na == 0.0 or nb == 0.0:
        return (1.0 if na == nb else 0.0), (1.0 if na == nb else float("inf"))
    return float((a * b).sum()) / (na * nb), na / nb


def old_criterion_accepts(got, ref):
    """True when every gradient passes cosine >= 0.999 and norm within 1 % (zero references exactly zero)."""
    for name, r in ref.items():
        c, q = cos_norm(got[name], r)
        if not (c >= 0.999 and abs(q - 1.0) < 1e-2):
            return False
    return True
