"""CPU PyTorch oracle for the PanopticNeRF per-ray render path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
legs may import this module.  The product package (``panopticnerf_b200``) never does.

PARITY UNPINNED.  The mounted reference (/root/reference) is the repository's landing branch only
(README.md:7 and README.md:13 point at the un-mounted code branches ``panopticnerf360`` and
``panopticnerf``), so no reference file:line exists for this path and the reference has no tests or
golden vectors.  This file therefore restates the *specification* in SURVEY.md section 8(a) rows
a1-a10 (nerf-pytorch conventions the reference is recalled to inherit).  Every function names the
row it follows.  Parity claims made against this oracle are "vs in-repo oracle".

All arithmetic is fp32 on CPU, written so that the bit-exact quantities (hit masks, box ids,
stratified z, sample_pdf indices) have a fully specified operation order:
  * no fused multiply-add anywhere (PyTorch CPU elementwise kernels never contract a*b+c),
  * true division,
  * torch.minimum/maximum (NaN-propagating),
  * running sums via torch.cumsum (sequential, double accumulator, rounded to fp32 per element).
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------
# a7  Embedder: gamma(p) = [p, sin(2^0 p), cos(2^0 p), ..., sin(2^(L-1) p), cos(2^(L-1) p)]
# --------------------------------------------------------------------------------------------
def embed(x: torch.Tensor, L: int) -> torch.Tensor:
    """SURVEY 8(a) a7. include-input, log-sampled bands, order [x | sin f0 | cos f0 | sin f1 | ...]."""
    out = [x]
    for k in range(L):
        f = float(2.0 ** k)
        out.append(torch.sin(x * f))
        out.append(torch.cos(x * f))
    return torch.cat(out, -1)


def embed_dim(L: int) -> int:
    return 3 + 6 * L


# --------------------------------------------------------------------------------------------
# a1/a8  Network
# --------------------------------------------------------------------------------------------
class Network(nn.Module):
    """SURVEY 8(a) a8.  NeRF MLP (D x W, ReLU, skip after layer D//2) + sigma / feature / view
    branch / rgb + optional semantic (W -> W/2 -> C) and instance (W -> W/2 -> K) heads.
    forward(pts[...,3], viewdirs[...,3]) -> raw[..., 4 + C + K] = [rgb_raw(3), sigma_raw(1), sem, inst].
    """

    def __init__(self, cfg):
        super().__init__()
        self.D, self.W = int(cfg.D), int(cfg.W)
        self.Lx, self.Ld = int(cfg.xyz_res), int(cfg.view_res)
        self.C, self.K = int(getattr(cfg, "num_classes", 0)), int(getattr(cfg, "num_instances", 0))
        self.skip = self.D // 2
        Ex, Ed, W = embed_dim(self.Lx), embed_dim(self.Ld), self.W
        layers = [nn.Linear(Ex, W)]
        for i in range(1, self.D):
            layers.append(nn.Linear(W + Ex if i == self.skip + 1 else W, W))
        self.pts_linears = nn.ModuleList(layers)
        self.alpha_linear = nn.Linear(W, 1)
        self.feature_linear = nn.Linear(W, W)
        self.views_linears = nn.ModuleList([nn.Linear(W + Ed, W // 2)])
        self.rgb_linear = nn.Linear(W // 2, 3)
        if self.C > 0:
            self.semantic_linears = nn.ModuleList([nn.Linear(W, W // 2), nn.Linear(W // 2, self.C)])
        if self.K > 0:
            self.instance_linears = nn.ModuleList([nn.Linear(W, W // 2), nn.Linear(W // 2, self.K)])

    def forward(self, pts: torch.Tensor, viewdirs: torch.Tensor) -> torch.Tensor:
        ex = embed(pts, self.Lx)
        ed = embed(viewdirs, self.Ld)
        h = ex
        for i, lin in enumerate(self.pts_linears):
            h = F.relu(lin(h))
            if i == self.skip:
                h = torch.cat([ex, h], -1)
        sigma = self.alpha_linear(h)
        feat = self.feature_linear(h)
        g = F.relu(self.views_linears[0](torch.cat([feat, ed], -1)))
        rgb = self.rgb_linear(g)
        outs = [rgb, sigma]
        if self.C > 0:
            outs.append(self.semantic_linears[1](F.relu(self.semantic_linears[0](h))))
        if self.K > 0:
            outs.append(self.instance_linears[1](F.relu(self.instance_linears[0](h))))
        return torch.cat(outs, -1)


def make_network(cfg) -> Network:
    """SURVEY 8(a) a1."""
    return Network(cfg)


# --------------------------------------------------------------------------------------------
# a5  ray / bounding-primitive intersection
# --------------------------------------------------------------------------------------------
def _dot3(a0, a1, a2, b0, b1, b2):
    # fixed association order ((a0*b0 + a1*b1) + a2*b2); every op is a separately rounded fp32 op
    return (a0 * b0 + a1 * b1) + a2 * b2


def slab_test(o: torch.Tensor, d: torch.Tensor, center: torch.Tensor, half: torch.Tensor,
              rot: torch.Tensor):
    """SURVEY 8(a) a5.  o,d [R,3]; center,half [B,3]; rot [B,3,3] (columns = box axes, box->world).
    Returns tmin, tmax [R,B] and hit [R,B] with hit = tmax > max(tmin, 0)."""
    oc = o[:, None, :] - center[None, :, :]                      # [R,B,3]
    dd = d[:, None, :].expand(-1, center.shape[0], -1)
    tmin = None
    tmax = None
    for j in range(3):
        ax = rot[None, :, :, j]                                   # box axis j in world coords [1,B,3]
        oj = _dot3(oc[..., 0], oc[..., 1], oc[..., 2], ax[..., 0], ax[..., 1], ax[..., 2])
        dj = _dot3(dd[..., 0], dd[..., 1], dd[..., 2], ax[..., 0], ax[..., 1], ax[..., 2])
        hj = half[None, :, j]
        t0 = (-hj - oj) / dj
        t1 = (hj - oj) / dj
        lo = torch.minimum(t0, t1)
        hi = torch.maximum(t0, t1)
        tmin = lo if tmin is None else torch.maximum(tmin, lo)
        tmax = hi if tmax is None else torch.minimum(tmax, hi)
    hit = tmax > torch.maximum(tmin, torch.zeros_like(tmin))
    return tmin, tmax, hit


def intersect(o, d, center, half, rot, max_hits: int):
    """SURVEY 8(a) a5.  Per ray: hit_mask (any box), and the ``max_hits`` nearest hit boxes sorted by
    tmin (ties -> lower box index): box_id int32 (-1 pad), t_in = max(tmin, 0), t_out = tmax (0 pad)."""
    R, B = o.shape[0], center.shape[0]
    M = max_hits
    if B == 0:
        return (torch.zeros(R, dtype=torch.bool), torch.full((R, M), -1, dtype=torch.int32),
                torch.zeros(R, M), torch.zeros(R, M))
    tmin, tmax, hit = slab_test(o, d, center, half, rot)
    key = torch.where(hit, tmin, torch.full_like(tmin, float("inf")))
    order = torch.sort(key, dim=1, stable=True).indices[:, :M]    # [R,min(M,B)]
    h = torch.gather(hit, 1, order)
    box_id = torch.where(h, order.to(torch.int32), torch.full_like(order, -1, dtype=torch.int32))
    t_in = torch.where(h, torch.maximum(torch.gather(tmin, 1, order), torch.zeros(())), torch.zeros(()))
    t_out = torch.where(h, torch.gather(tmax, 1, order), torch.zeros(()))
    if order.shape[1] < M:
        pad = M - order.shape[1]
        box_id = F.pad(box_id, (0, pad), value=-1)
        t_in = F.pad(t_in, (0, pad))
        t_out = F.pad(t_out, (0, pad))
    return hit.any(1), box_id.contiguous(), t_in.contiguous(), t_out.contiguous()


def scene_near_far(o, d, aabb, near_min: float, far_default: float):
    """Global near/far from the scene AABB (a5, 'AABB is the special case R=I').
    near = max(tmin, near_min), far = tmax when the ray hits; (near_min, far_default) otherwise."""
    lo, hi = aabb[0], aabb[1]
    center = ((lo + hi) * 0.5)[None]
    half = ((hi - lo) * 0.5)[None]
    rot = torch.eye(3)[None]
    tmin, tmax, hit = slab_test(o, d, center, half, rot)
    tmin, tmax, hit = tmin[:, 0], tmax[:, 0], hit[:, 0]
    near = torch.where(hit, torch.maximum(tmin, torch.full_like(tmin, near_min)),
                       torch.full_like(tmin, near_min))
    far = torch.where(hit, tmax, torch.full_like(tmax, far_default))
    return near, far


# --------------------------------------------------------------------------------------------
# a6  stratified sampling (+ per-sample primitive id)
# --------------------------------------------------------------------------------------------
def stratified_z(near, far, t_vals, perturb: float = 0.0, u: Optional[torch.Tensor] = None):
    """SURVEY 8(a) a6.  z = near*(1-t) + far*t ; optional jitter with externally supplied u."""
    z = near[:, None] * (1.0 - t_vals)[None, :] + far[:, None] * t_vals[None, :]
    if perturb > 0.0:
        mids = 0.5 * (z[:, 1:] + z[:, :-1])
        upper = torch.cat([mids, z[:, -1:]], -1)
        lower = torch.cat([z[:, :1], mids], -1)
        if u is None:
            u = torch.rand(z.shape)
        z = lower + (upper - lower) * u
    return z


def interval_z(near, far, t_vals, box_id, t_in, t_out, perturb: float = 0.0, u: Optional[torch.Tensor] = None):
    """SURVEY 8(a) a6, interval mode: "samples are placed inside the M hit intervals".  The reference's rule for
    dividing the N samples between the intervals is not in the mount (8(c) question 4); the rule restated here is
    the one chosen for this build (DESIGN.md, 'chosen, unverified'), in the same fp32 operation order as the kernel:
      1. valid intervals are clipped to [near, far] and kept when their length is positive;
      2. L = sum of kept lengths (interval order); n_m = min(floor(N*len_m/L), samples still unassigned) in
         interval order; the remainder goes one sample at a time to the kept intervals, nearest first (cyclic);
      3. sample j of interval m: a + (b-a)*((j+c)/n_m), c = 0.5 or the jitter u of that allocation slot;
      4. the N depths are sorted ascending.
    Rays without a kept interval use the uniform rule of stratified_z."""
    R, M = box_id.shape
    N = t_vals.shape[0]
    z_uniform = stratified_z(near, far, t_vals, perturb, u)
    valid = box_id >= 0
    a = torch.maximum(t_in, near[:, None])
    b = torch.minimum(t_out, far[:, None])
    ln = b - a
    keep = valid & (ln > 0)
    ln = torch.where(keep, ln, torch.zeros_like(ln))
    L = torch.zeros(R)
    seen = torch.zeros(R, dtype=torch.bool)
    for m in range(M):                       # sequential fp32 sum over the kept intervals, first one copied
        L = torch.where(keep[:, m], torch.where(seen, L + ln[:, m], ln[:, m]), L)
        seen = seen | keep[:, m]
    n = torch.zeros(R, M, dtype=torch.int64)
    left = torch.full((R,), N, dtype=torch.int64)
    Ls = torch.where(seen, L, torch.ones_like(L))
    for m in range(M):
        q = torch.floor((float(N) * ln[:, m]) / Ls).to(torch.int64)
        q = torch.clamp(torch.minimum(q, left), min=0)
        q = torch.where(keep[:, m], q, torch.zeros_like(q))
        n[:, m] = q
        left = left - q
    while bool(((left > 0) & seen).any()):
        for m in range(M):
            give = keep[:, m] & (left > 0)
            n[:, m] += give.to(torch.int64)
            left = left - give.to(torch.int64)
    first = torch.cumsum(n, 1) - n                                   # slot of each interval's first sample
    k = torch.arange(N)[None, :].expand(R, N)
    c = u if (perturb > 0.0 and u is not None) else torch.full((R, N), 0.5)
    z = torch.zeros(R, N)
    for m in range(M):
        j = k - first[:, m:m + 1]
        inside = (j >= 0) & (j < n[:, m:m + 1])
        nm = torch.clamp(n[:, m:m + 1], min=1).to(torch.float32)
        t = (j.to(torch.float32) + c) / nm
        zm = a[:, m:m + 1] + (b[:, m:m + 1] - a[:, m:m + 1]) * t
        z = torch.where(inside, zm, z)
    z = torch.sort(z, -1).values
    return torch.where(seen[:, None], z, z_uniform)


def tag_samples(z, box_id, t_in, t_out):
    """a6: each sample carries the id of the first (nearest) hit interval containing it, else -1."""
    R, N = z.shape
    sid = torch.full((R, N), -1, dtype=torch.int32)
    for m in reversed(range(box_id.shape[1])):
        inside = (box_id[:, m:m + 1] >= 0) & (z >= t_in[:, m:m + 1]) & (z <= t_out[:, m:m + 1])
        sid = torch.where(inside, box_id[:, m:m + 1].expand(-1, N), sid)
    return sid


# --------------------------------------------------------------------------------------------
# a9  raw2outputs
# --------------------------------------------------------------------------------------------
def raw2outputs(raw, z_vals, rays_d, raw_noise_std: float = 0.0, white_bkgd: bool = False,
                num_classes: int = 0, num_instances: int = 0, sem_activation: str = "none",
                sample_box: Optional[torch.Tensor] = None, box_sem: Optional[torch.Tensor] = None,
                box_inst: Optional[torch.Tensor] = None, mask_outside: bool = False,
                noise: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """SURVEY 8(a) a9.  raw [R,N,4+C+K], z_vals [R,N], rays_d [R,3]."""
    C, K = num_classes, num_instances
    dists = z_vals[:, 1:] - z_vals[:, :-1]
    dists = torch.cat([dists, torch.full_like(z_vals[:, :1], 1e10)], -1)   # (also right for N == 1)
    dists = dists * torch.norm(rays_d[:, None, :], dim=-1)
    rgb = torch.sigmoid(raw[..., :3])
    sig = raw[..., 3]
    if raw_noise_std > 0.0:
        sig = sig + (noise if noise is not None else torch.randn(sig.shape)) * raw_noise_std
    sig = F.relu(sig)
    if mask_outside and sample_box is not None:
        sig = torch.where(sample_box >= 0, sig, torch.zeros_like(sig))
    alpha = 1.0 - torch.exp(-sig * dists)
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    weights = alpha * trans
    rgb_map = torch.sum(weights[..., None] * rgb, -2)
    depth_map = torch.sum(weights * z_vals, -1)
    acc_map = torch.sum(weights, -1)
    disp_map = 1.0 / torch.maximum(torch.full_like(depth_map, 1e-10), depth_map / acc_map)
    if white_bkgd:
        rgb_map = rgb_map + (1.0 - acc_map[..., None])
    out = {"rgb_map": rgb_map, "depth_map": depth_map, "acc_map": acc_map, "disp_map": disp_map,
           "weights": weights}
    if C > 0:
        s = raw[..., 4:4 + C]
        if sem_activation == "softmax":
            s = torch.softmax(s, -1)
        out["semantic_map"] = torch.sum(weights[..., None] * s, -2)
    if K > 0:
        out["instance_map"] = torch.sum(weights[..., None] * raw[..., 4 + C:4 + C + K], -2)
    if sample_box is not None and box_sem is not None and C > 0:
        out["fixed_semantic_map"] = _composite_onehot(weights, sample_box, box_sem, C)
    if sample_box is not None and box_inst is not None and K > 0:
        out["fixed_instance_map"] = _composite_onehot(weights, sample_box, box_inst, K)
    return out


def raw2outputs_backward(raw, z_vals, rays_d, grads: Dict[str, torch.Tensor], white_bkgd: bool = False,
                         num_classes: int = 0, num_instances: int = 0,
                         sample_box: Optional[torch.Tensor] = None, box_sem: Optional[torch.Tensor] = None,
                         box_inst: Optional[torch.Tensor] = None, mask_outside: bool = False) -> torch.Tensor:
    """Closed form of d(loss)/d(raw) for `raw2outputs` (sem_activation "none", no noise), the algorithm
    `pnr_composite_backward` implements.  With t_i = 1 - alpha_i + 1e-10, T_i = prod_{j<i} t_j, w_i = alpha_i T_i,
    G_i = dL/dw_i:   dL/dalpha_i = G_i T_i - (sum_{j>i} G_j w_j) / t_i.
    tests/test_cpu_backward.py pins it against autograd through `raw2outputs`."""
    C, K = num_classes, num_instances
    R, N = z_vals.shape
    zero = torch.zeros((), dtype=raw.dtype)
    g = lambda k, shape: grads[k] if k in grads and grads[k] is not None else torch.zeros(shape, dtype=raw.dtype)
    dists = torch.cat([z_vals[:, 1:] - z_vals[:, :-1], torch.full_like(z_vals[:, :1], 1e10)], -1)
    dists = dists * torch.norm(rays_d[:, None, :], dim=-1)
    live = raw[..., 3] > 0
    if mask_outside and sample_box is not None:
        live = live & (sample_box >= 0)
    sig = torch.where(live, raw[..., 3], torch.zeros_like(raw[..., 3]))
    e = torch.exp(-sig * dists)
    alpha = 1.0 - e
    t = 1.0 - alpha + 1e-10
    T = torch.cumprod(torch.cat([torch.ones_like(t[:, :1]), t], -1), -1)[:, :-1]
    w = alpha * T
    c = torch.sigmoid(raw[..., :3])
    g_rgb = g("rgb_map", (R, 3))
    g_acc = g("acc_map", (R,)) - (g_rgb.sum(-1) if white_bkgd else zero)
    G = (c * g_rgb[:, None]).sum(-1) + g("depth_map", (R,))[:, None] * z_vals + g_acc[:, None] + g("weights", (R, N))
    d_raw = torch.zeros_like(raw)
    d_raw[..., :3] = w[..., None] * g_rgb[:, None] * c * (1.0 - c)
    if C > 0:
        gs = g("semantic_map", (R, C))
        G = G + (raw[..., 4:4 + C] * gs[:, None]).sum(-1)
        d_raw[..., 4:4 + C] = w[..., None] * gs[:, None]
    if K > 0:
        gi = g("instance_map", (R, K))
        G = G + (raw[..., 4 + C:4 + C + K] * gi[:, None]).sum(-1)
        d_raw[..., 4 + C:4 + C + K] = w[..., None] * gi[:, None]
    for key, table, n in (("fixed_semantic_map", box_sem, C), ("fixed_instance_map", box_inst, K)):
        if sample_box is not None and table is not None and n > 0 and grads.get(key) is not None:
            ids = _box_ids(sample_box, table)
            ok = (ids >= 0) & (ids < n)
            G = G + torch.where(ok, torch.gather(grads[key], 1, ids.clamp(0, n - 1)), torch.zeros_like(G))
    Gw = G * w
    # strictly later samples, summed without subtracting Gw_i (which cancels behind a surface, where S / t is large)
    S = torch.cat([torch.flip(torch.cumsum(torch.flip(Gw[:, 1:], [-1]), -1), [-1]), torch.zeros_like(Gw[:, :1])], -1)
    d_raw[..., 3] = (G * T - S / t) * torch.where(live, dists * e, torch.zeros_like(e))
    return d_raw


def _box_ids(sample_box, table):
    """table[sample_box_i] per sample, -1 where the sample is in no box: sample_box < 0 or >= len(table)."""
    B = table.shape[0]
    inside = (sample_box >= 0) & (sample_box < B)
    idx = sample_box.clamp(0, max(B - 1, 0)).to(torch.int64)
    looked = table.to(torch.int64)[idx] if B > 0 else torch.zeros_like(idx)
    return torch.where(inside, looked, torch.full_like(idx, -1))


def _composite_onehot(weights, sample_box, table, n):
    """sum_i w_i * onehot(table[sample_box_i]) ; samples in no box (sample_box < 0 or >= len(table)) or with an id
    outside [0,n) add nothing."""
    ids = _box_ids(sample_box, table)
    valid = (ids >= 0) & (ids < n)
    out = torch.zeros(weights.shape[0], n + 1, dtype=weights.dtype)
    out.scatter_add_(1, torch.where(valid, ids, torch.full_like(ids, n)), weights)
    return out[:, :n].contiguous()


# --------------------------------------------------------------------------------------------
# a10  sample_pdf
# --------------------------------------------------------------------------------------------
def sample_pdf(bins, weights, N_importance: int, det: bool = True, u: Optional[torch.Tensor] = None,
               pdf_norm: str = "cumsum"):
    """SURVEY 8(a) a10.  bins [R,Nb] (= mid points), weights [R,Nb-1] (= coarse weights[1:-1]).
    Returns z_f [R,Ni] and the searchsorted indices idx [R,Ni] (int64).
    pdf_norm: how the pdf is normalised.  "cumsum" (default; what the CUDA kernel reproduces bit for bit) divides by
    the last element of the running sum, so the operation order is fully specified.  "sum" divides by
    torch.sum(w, -1) as nerf-pytorch does: torch's blocked fp32 reduction differs from the running sum in the last
    ulp, which can move a searchsorted index when u falls within an ulp of a cdf entry
    (tests/test_cpu_oracle.py::test_sample_pdf_sum_variant counts how often).  Kept so that the variant the real
    reference uses can be switched on the day its source is mounted (VERDICT r1, weak item 1)."""
    w = weights + 1e-5
    if pdf_norm == "sum":
        pdf = w / torch.sum(w, -1, keepdim=True)
    else:
        csum = torch.cumsum(w, -1)
        pdf = w / csum[:, -1:]
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)       # [R,Nb]
    if u is None:
        if det:
            u = torch.linspace(0.0, 1.0, N_importance)[None].expand(cdf.shape[0], -1)
        else:
            u = torch.rand(cdf.shape[0], N_importance)
    u = u.contiguous()
    idx = torch.searchsorted(cdf.contiguous(), u, right=True)
    below = torch.clamp(idx - 1, min=0)
    above = torch.clamp(idx, max=cdf.shape[-1] - 1)
    cdf_b, cdf_a = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bin_b, bin_a = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = cdf_a - cdf_b
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_b) / denom
    z_f = bin_b + t * (bin_a - bin_b)
    return z_f, idx


def merge_sorted(z, z_f):
    """a10 tail: z_all = sort(cat(z, z_f))."""
    return torch.sort(torch.cat([z, z_f], -1), -1).values


# --------------------------------------------------------------------------------------------
# a3/a4  Renderer
# --------------------------------------------------------------------------------------------
class Renderer:
    """SURVEY 8(a) a2-a4.  Renderer(net).render(batch) -> dict of per-ray maps."""

    def __init__(self, cfg, net: Network, net_fine: Optional[Network] = None):
        self.cfg, self.net = cfg, net
        self.net_fine = net_fine if net_fine is not None else net

    # -- a4
    def batchify_rays(self, rays, near, far, batch, chunk: Optional[int] = None):
        chunk = int(chunk or getattr(self.cfg, "chunk", 32768))
        outs = []
        for i in range(0, rays.shape[0], chunk):
            sl = slice(i, i + chunk)
            outs.append(self.render_rays(rays[sl], near[sl], far[sl], batch, sl))
        return {k: torch.cat([o[k] for o in outs], 0) for k in outs[0]}

    def _query(self, net, o, d, z):
        pts = o[:, None, :] + d[:, None, :] * z[:, :, None]
        vd = d / torch.norm(d, dim=-1, keepdim=True)
        vd = vd[:, None, :].expand(pts.shape)
        return net(pts, vd)

    def render_rays(self, rays, near, far, batch, sl):
        cfg = self.cfg
        o, d = rays[:, :3], rays[:, 3:6]
        N = int(cfg.N_samples)
        Ni = int(getattr(cfg, "N_importance", 0))
        C, K = int(getattr(cfg, "num_classes", 0)), int(getattr(cfg, "num_instances", 0))
        M = int(getattr(cfg, "max_hits", 4))
        perturb = float(batch.get("perturb", getattr(cfg, "perturb", 0.0)))
        out = {}
        has_boxes = "box_center" in batch and batch["box_center"].shape[0] > 0
        if has_boxes:
            hit, box_id, t_in, t_out = intersect(o, d, batch["box_center"], batch["box_half"],
                                                 batch["box_rot"], M)
            out.update(hit_mask=hit, box_id=box_id, t_in=t_in, t_out=t_out)
            if bool(getattr(cfg, "bound_by_primitives", False)):
                first = t_in[:, 0]
                last = torch.where(box_id >= 0, t_out, torch.zeros_like(t_out)).max(1).values
                near = torch.where(hit, torch.maximum(near, first), near)
                far = torch.where(hit, torch.minimum(far, last), far)
        t_vals = torch.linspace(0.0, 1.0, N)
        u = batch["u"][sl] if "u" in batch else None
        if has_boxes and str(getattr(cfg, "sample_mode", "uniform")) == "intervals":
            z = interval_z(near, far, t_vals, box_id, t_in, t_out, perturb, u)
        else:
            z = stratified_z(near, far, t_vals, perturb, u)
        kw = dict(raw_noise_std=0.0, white_bkgd=bool(getattr(cfg, "white_bkgd", False)),
                  num_classes=C, num_instances=K,
                  sem_activation=str(getattr(cfg, "sem_activation", "none")),
                  mask_outside=bool(getattr(cfg, "mask_outside", False)))
        if has_boxes:
            kw.update(box_sem=batch.get("box_sem"), box_inst=batch.get("box_inst"))
        sb = tag_samples(z, box_id, t_in, t_out) if has_boxes else None
        raw = self._query(self.net, o, d, z)
        res = raw2outputs(raw, z, d, sample_box=sb, **kw)
        if Ni > 0:
            for k, v in res.items():
                out[k + "_0"] = v
            out["z_vals_0"] = z
            zm = 0.5 * (z[:, 1:] + z[:, :-1])
            u_f = batch["u_fine"][sl] if "u_fine" in batch else None
            z_f, _ = sample_pdf(zm, res["weights"][:, 1:-1], Ni, det=(perturb == 0.0), u=u_f)
            z = merge_sorted(z, z_f)
            sb = tag_samples(z, box_id, t_in, t_out) if has_boxes else None
            raw = self._query(self.net_fine, o, d, z)
            res = raw2outputs(raw, z, d, sample_box=sb, **kw)
        out.update(res)
        out["z_vals"] = z
        if sb is not None:
            out["sample_box"] = sb
        if bool(getattr(cfg, "return_raw", False)):
            out["raw"] = raw
        return out

    # -- a3
    @torch.no_grad()
    def render(self, batch: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        cfg = self.cfg
        rays = batch["rays"]
        o, d = rays[:, :3], rays[:, 3:6]
        if "near" in batch and "far" in batch:
            near, far = batch["near"], batch["far"]
        elif "scene_aabb" in batch:
            near, far = scene_near_far(o, d, batch["scene_aabb"], float(cfg.near), float(cfg.far))
        else:
            near = torch.full((rays.shape[0],), float(cfg.near))
            far = torch.full((rays.shape[0],), float(cfg.far))
        out = self.batchify_rays(rays, near, far, batch)
        out["near"], out["far"] = near, far
        return out


def make_renderer(cfg, net, net_fine=None) -> Renderer:
    """SURVEY 8(a) a2."""
    return Renderer(cfg, net, net_fine)


def _sqrt_rn(x: torch.Tensor) -> torch.Tensor:
    """Correctly rounded fp32 square root (torch.sqrt on CPU goes through a vector math library that is not: about
    0.5 % of its results are one ulp off; numpy's float32 sqrt is the hardware instruction)."""
    return torch.from_numpy(np.sqrt(x.detach().to(torch.float32).contiguous().numpy()))


def generate_rays(H: int, W: int, intr, c2w: torch.Tensor, camera: str = "pinhole", row0: int = 0,
                  rows: Optional[int] = None) -> torch.Tensor:
    """SURVEY 8(f) rank 3 (the step before the path; reference: ray generation in the KITTI-360 dataset
    loader, not in the mount).  rays [rows*W, 6] = origin || unnormalised direction for a pinhole or an
    equirectangular camera with camera-to-world [R|t] (3x4).  Elementwise fp32, fixed association order."""
    rows = H - row0 if rows is None else rows
    fx, fy, cx, cy = [float(x) for x in intr[:4]]
    v, u = torch.meshgrid(torch.arange(row0, row0 + rows, dtype=torch.float32),
                          torch.arange(W, dtype=torch.float32), indexing="ij")
    if camera == "pinhole":
        x, y, z = (u - cx) / fx, (v - cy) / fy, torch.ones_like(u)
    elif camera == "fisheye":
        # KITTI-360 fisheye, unified (MEI) model; intr = (gamma1, gamma2, u0, v0, xi, k1, k2).  Published model
        # (kitti360scripts CameraFisheye.cam2image is the projection); the inverse below is this repo's: radial
        # undistortion by 8 Newton steps from ro = rd, then the lift to the unit sphere.  Every op fp32, in this order.
        xi, k1, k2 = [torch.tensor(float(t), dtype=torch.float32) for t in intr[4:7]]
        mx, my = (u - cx) / fx, (v - cy) / fy
        rd = _sqrt_rn(mx * mx + my * my)
        k1x3, k2x5 = 3.0 * k1, 5.0 * k2
        ro = rd
        for _ in range(8):
            ro2 = ro * ro
            f = ro * (1.0 + ro2 * (k1 + k2 * ro2)) - rd
            fp = 1.0 + ro2 * (k1x3 + k2x5 * ro2)
            ro = ro - f / fp
        scale = torch.where(rd > 0, ro / rd, torch.ones_like(rd))
        px, py = mx * scale, my * scale
        r2 = px * px + py * py
        # (xi > 1: pixels beyond the mirror's field of view have a negative radicand; it is clamped, the caller masks them)
        fac = (xi + _sqrt_rn(torch.clamp_min(1.0 + (1.0 - xi * xi) * r2, 0.0))) / (1.0 + r2)
        x, y, z = fac * px, fac * py, fac - xi
    else:
        lon = (u / float(W) - 0.5) * 6.2831853071795864769
        lat = (0.5 - v / float(H)) * 3.14159265358979323846
        x, y, z = torch.cos(lat) * torch.sin(lon), -torch.sin(lat), torch.cos(lat) * torch.cos(lon)
    c = c2w.to(torch.float32)
    d = [(c[i, 0] * x + c[i, 1] * y) + c[i, 2] * z for i in range(3)]
    o = [torch.full_like(x, float(c[i, 3])) for i in range(3)]
    return torch.stack(o + d, -1).reshape(-1, 6).contiguous()


def mlp_flops_per_sample(cfg) -> int:
    """Algorithmic FLOPs (2 x MAC, true layer shapes) per SURVEY 8(d) / BASELINE.md section 3."""
    D, W = int(cfg.D), int(cfg.W)
    Ex, Ed = embed_dim(int(cfg.xyz_res)), embed_dim(int(cfg.view_res))
    C, K = int(getattr(cfg, "num_classes", 0)), int(getattr(cfg, "num_instances", 0))
    mac = Ex * W + (D - 2) * W * W + (W + Ex) * W + W + W * W + (W + Ed) * (W // 2) + (W // 2) * 3
    if C > 0:
        mac += W * (W // 2) + (W // 2) * C
    if K > 0:
        mac += W * (W // 2) + (W // 2) * K
    return 2 * mac
