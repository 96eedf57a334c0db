"""The sampling, compositing, loss, label and encoder kernels at the limits they accept, through the C ABI.

Two kinds of check:
- Kernels with a bit-exact contract (intersect, stratified / interval sampling, tags, sample_pdf, label tiles, panoptic
  fusion, the hash-grid forward) are held to the fp32 oracle bit for bit at the sizes where their staging, sorting and
  lane striding change: box chunks of 512, 512-wide sorts, channel groups of 32, C and K up to 32767.
- Floating-point kernels (compositing forward and backward, losses, positional encoding, hash-grid backward) are
  compared with the oracle run in float64 on the same fp32 inputs, ray by ray: every ray is held to a bound set by its
  own magnitudes, not by the RMS of the whole tensor, so an error on a few rays or a few channels cannot hide.
Each float64 comparison prints the largest error it measured over its bound (a ratio; 1 is the bound).
"""
import ctypes as C
import math

import pytest
import torch

from oracle import reference_losses as OL
from oracle import reference_panoptic as OP
from oracle import reference_renderer as O
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.networks.encoding import HashGrid
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from panopticnerf_b200.lib.visualizers import fuse_panoptic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64


def _report(what, ratio):
    print(f"{what}: largest error / bound = {ratio:.3e}")
    assert ratio <= 1.0, f"{what}: error {ratio:.3e} x its bound"


def _ratio(err, bound):
    """max of err / bound, where a zero bound demands an exact zero error."""
    err, bound = err.double(), bound.double()
    assert bool((err[bound == 0] == 0).all()), "nonzero error where the float64 value is exactly 0"
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


# ------------------------------------------------------------------------------------------------ intersect
def _rays_and_boxes(R, B, seed):
    """Rays from near the origin into +z and B oriented boxes in front of them.  A set of index positions, including both ends of each 512-box chunk, holds the same large box across every ray's path, nearer than any
    other box: duplicates with equal t_in, which must come out in box-index order, and more hits per ray than M."""
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(R, 3, generator=g) * 0.1
    d = torch.cat([(torch.rand(R, 2, generator=g) - 0.5), torch.ones(R, 1)], -1)
    center = torch.cat([(torch.rand(B, 2, generator=g) - 0.5) * 30, 12 + torch.rand(B, 1, generator=g) * 48], -1)
    half = 0.5 + 4.0 * torch.rand(B, 3, generator=g)
    rot = torch.linalg.qr(torch.randn(B, 3, 3, generator=g)).Q.contiguous()
    wall = [i for i in (0, 1, 255, 510, 511, 512, 513, 1022, 1023, 1024, B - 2, B - 1) if 0 <= i < B]
    center[wall] = torch.tensor([0.0, 0.0, 3.0])
    half[wall] = torch.tensor([8.0, 8.0, 0.5])
    rot[wall] = torch.eye(3)
    return torch.cat([o, d], -1), center, half, rot


@pytest.mark.parametrize("B", [511, 512, 513, 1024, 1025])
def test_intersect_across_box_chunks(B):
    rays, c, h, rot = _rays_and_boxes(2000, B, B)
    M = 8
    ref = O.intersect(rays[:, :3], rays[:, 3:], c, h, rot, M)
    got = P.intersect(rays.to(DEV), c.to(DEV), h.to(DEV), rot.to(DEV), M)
    for a, b, name in zip(got, ref, ("hit", "box_id", "t_in", "t_out")):
        assert torch.equal(a.cpu(), b), name
    hits = O.slab_test(rays[:, :3], rays[:, 3:], c, h, rot)[2].sum(1)
    assert int((hits > M).sum()) > 100                                 # lists overflow M: the selection is exercised
    assert bool((ref[1] == min(B, 512) - 1).any(1).all())               # every ray keeps the last box of chunk 0
    assert bool(((ref[1][:, 1:] < 0) | (ref[2][:, 1:] >= ref[2][:, :-1])).all())     # t_in ascending up to the padding


# ------------------------------------------------------------------------------------------------ sampling
def _intervals(R, M, near, far, seed):
    """Hit tables with overlapping, zero-length and wholly-outside intervals, and empty slots."""
    g = torch.Generator().manual_seed(seed)
    t_in = near[:, None] + (far - near)[:, None] * (torch.rand(R, M, generator=g) * 1.4 - 0.2)
    t_out = t_in + torch.rand(R, M, generator=g) * (far - near)[:, None] * 0.3
    zero = torch.rand(R, M, generator=g) < 0.15
    t_out = torch.where(zero, t_in, t_out)                                        # zero length
    out = torch.rand(R, M, generator=g) < 0.1
    t_in = torch.where(out, far[:, None] + 1.0, t_in)                             # wholly beyond far
    t_out = torch.where(out, far[:, None] + 5.0, t_out)
    t_in[:, 1] = t_in[:, 0]                                                       # overlapping / duplicate
    t_out[:, 1] = torch.maximum(t_out[:, 0], t_out[:, 1])
    box_id = torch.randint(0, 50, (R, M), generator=g, dtype=torch.int32)
    box_id = torch.where(torch.rand(R, M, generator=g) < 0.2, torch.full_like(box_id, -1), box_id)
    box_id[: R // 16] = -1                                                        # no interval: uniform fallback
    return box_id, t_in.contiguous(), t_out.contiguous()


@pytest.mark.parametrize("N,perturb", [(257, 0.0), (257, 1.0), (1000, 0.0), (1000, 1.0)])
def test_stratified_and_tags_past_256(N, perturb):
    R, M = 700, 8
    g = torch.Generator().manual_seed(N)
    near = 0.5 + torch.rand(R, generator=g)
    far = near + 1 + torch.rand(R, generator=g) * 60
    box_id, t_in, t_out = _intervals(R, M, near, far, N)
    t_vals = torch.linspace(0.0, 1.0, N)
    u = torch.rand(R, N, generator=g)
    z = O.stratified_z(near, far, t_vals, perturb, u)
    sb = O.tag_samples(z, box_id, t_in, t_out)
    gz, gsb = P.stratified_z(near.to(DEV), far.to(DEV), t_vals.to(DEV), perturb, u.to(DEV), box_id.to(DEV),
                             t_in.to(DEV), t_out.to(DEV), want_tags=True)
    assert torch.equal(gz.cpu(), z) and torch.equal(gsb.cpu(), sb)
    assert torch.equal(P.tag_samples(gz, box_id.to(DEV), t_in.to(DEV), t_out.to(DEV)).cpu(), sb)
    assert int((sb >= 0).sum()) > R


@pytest.mark.parametrize("N", [256, 255, 129])
@pytest.mark.parametrize("perturb", [0.0, 1.0])
def test_intervals_at_the_largest_sort(N, perturb):
    R, M = 1000, 8
    g = torch.Generator().manual_seed(N + int(perturb))
    near = 0.5 + torch.rand(R, generator=g)
    far = near + 1 + torch.rand(R, generator=g) * 60
    box_id, t_in, t_out = _intervals(R, M, near, far, N)
    t_vals = torch.linspace(0.0, 1.0, N)
    u = torch.rand(R, N, generator=g)
    z = O.interval_z(near, far, t_vals, box_id, t_in, t_out, perturb, u)
    sb = O.tag_samples(z, box_id, t_in, t_out)
    gz, gsb = P.interval_z(near.to(DEV), far.to(DEV), t_vals.to(DEV), box_id.to(DEV), t_in.to(DEV), t_out.to(DEV),
                           perturb, u.to(DEV))
    assert torch.equal(gz.cpu(), z), int((gz.cpu() != z).sum())
    assert torch.equal(gsb.cpu(), sb)
    assert bool((z[:, 1:] >= z[:, :-1]).all()) and int((sb >= 0).sum()) > R * N // 2


@pytest.mark.parametrize("N,Ni", [(3, 253), (3, 254), (3, 508), (3, 509), (255, 1), (255, 2), (255, 256), (256, 1),
                                  (256, 255), (256, 256)])
@pytest.mark.parametrize("det", [True, False])
def test_sample_pdf_at_the_largest_merge(N, Ni, det):
    """Coarse depths with runs of equal values (zero-length bins), so fine depths land exactly on coarse ones: ties for
    the rank merge (deterministic u) and for the bitonic sort (jittered u), padded from N + Ni to 512."""
    R = 600
    g = torch.Generator().manual_seed(N * 1000 + Ni)
    z = torch.sort(torch.randint(0, max(N // 3, 2), (R, N), generator=g).float() * 0.25 + 1.0, -1).values
    w = torch.rand(R, N, generator=g) ** 3
    w[: R // 5] *= (torch.rand(R // 5, N, generator=g) > 0.7)
    w[R // 5: R // 5 + 20] = 0.0
    w = w / (w.sum(-1, keepdim=True) + 1e-3)
    u = None if det else torch.rand(R, Ni, generator=g)
    zm = 0.5 * (z[:, 1:] + z[:, :-1])
    z_f, idx = O.sample_pdf(zm, w[:, 1:-1], Ni, det=det, u=u)
    z_all = O.merge_sorted(z, z_f)
    gz_f, gz_all, gidx = P.sample_pdf(z.to(DEV), w.to(DEV), Ni, det=det, u=None if u is None else u.to(DEV),
                                      want_idx=True)
    assert torch.equal(gidx.cpu(), idx)
    assert torch.equal(gz_f.cpu(), z_f)
    assert torch.equal(gz_all.cpu(), z_all)
    assert int((z_f[:, :, None] == z[:, None, :]).any(-1).sum()) > 0 or N == 3     # fine depths equal to coarse ones


# ------------------------------------------------------------------------------------------------ compositing
def _composite_case(R, N, C, K, seed, B=20, big_on_surface=True):
    """Rays in four regimes (a quarter each): mid-range densities; surface-like (empty space, then densities from 1 to
    1000 so alpha rounds to 1 in fp32); all empty; and duplicated depths (zero-length deltas).  Some rays carry
    logits of +-1e4.  Sample boxes run from -3 to B + 2 and the id tables hold ids from -2 to C + 2 / K + 2: boxes
    outside the table and ids outside [0, C) must add nothing."""
    g = torch.Generator().manual_seed(seed)
    raw = torch.randn(R, N, 4 + C + K, generator=g)
    q = R // 4
    sig = raw[..., 3] * 0.3 + 0.05
    surf = torch.randint(0, N, (q, 1), generator=g)
    dens = torch.exp(torch.rand(q, N, generator=g) * math.log(1000.0))
    sig[q:2 * q] = torch.where(torch.arange(N)[None] < surf, torch.full_like(dens, -1.0), dens)
    sig[2 * q:3 * q] = -torch.rand(q, N, generator=g)
    raw[..., 3] = sig
    if C + K > 0:
        big = torch.rand(R, generator=g) < 0.25
        if not big_on_surface:
            big[q:2 * q] = False
        raw[big, :, 4:] = torch.sign(raw[big, :, 4:]) * (1e4 * torch.rand(int(big.sum()), N, C + K, generator=g))
    z = torch.sort(torch.rand(R, N, generator=g) * 40 + 0.05, -1).values
    z[3 * q:] = torch.sort(torch.randint(0, 12, (R - 3 * q, N), generator=g).float() * 3.0 + 0.5, -1).values
    d = torch.randn(R, 3, generator=g) * (0.5 + torch.rand(R, 1, generator=g))
    sb = torch.randint(-3, B + 3, (R, N), generator=g, dtype=torch.int32)
    bs = torch.randint(-2, max(C, 1) + 3, (B,), generator=g, dtype=torch.int32)
    bi = torch.randint(-2, max(K, 1) + 3, (B,), generator=g, dtype=torch.int32)
    return raw, z, d, sb, bs, bi


def _abs_sums(raw, z, w, C, K, sb, bs, bi, softmax):
    """sum_i |w_i v_i| of every map, per ray and channel, in float64 (v_i = what sample i contributes)."""
    aw = w.abs()
    s = {"rgb_map": (aw[..., None] * torch.sigmoid(raw[..., :3])).sum(1), "depth_map": (aw * z.abs()).sum(1),
         "acc_map": aw.sum(1)}
    if C > 0:
        v = torch.softmax(raw[..., 4:4 + C], -1) if softmax else raw[..., 4:4 + C].abs()
        s["semantic_map"] = (aw[..., None] * v).sum(1)
        s["fixed_semantic_map"] = O._composite_onehot(aw, sb, bs, C)
    if K > 0:
        s["instance_map"] = (aw[..., None] * raw[..., 4 + C:].abs()).sum(1)
        s["fixed_instance_map"] = O._composite_onehot(aw, sb, bi, K)
    return s


@pytest.mark.parametrize("N,C,K,flags", [
    (1, 1, 1, {}), (31, 32, 33, {"sem_activation": "softmax"}), (32, 33, 32, {"white_bkgd": True}),
    (33, 96, 97, {"mask_outside": True}), (225, 97, 96, {"sem_activation": "softmax", "white_bkgd": True}),
    (256, 128, 128, {}), (256, 128, 128, {"sem_activation": "softmax", "mask_outside": True}), (256, 0, 0, {}),
    (33, 128, 1, {}), (225, 1, 128, {"mask_outside": True})])
def test_composite_per_ray_against_float64(N, C, K, flags):
    """Each map element within 1e-4 x sum_i |w_i v_i| of its ray (the largest over the map's channels, float64), plus
    half an ulp of the stored value; weights within 1e-4 of the ray's largest weight; disp within 2e-4 relative (it
    is depth / acc, each within 1e-4).  A fixed map can take all its weight from samples behind a near-opaque one,
    where fp32 keeps t = 1 - alpha + 1e-10 only to an ulp of 1 (float64 keeps exp(-sigma delta)); those weights are
    ~1e-10 of the ray's largest, so the fixed maps' sum is floored at the ray's largest weight, the scale the weights
    themselves are held to."""
    R = 256
    raw, z, d, sb, bs, bi = _composite_case(R, N, C, K, seed=N * 7 + C + 3 * K)
    kw = dict(num_classes=C, num_instances=K, sample_box=sb, box_sem=bs, box_inst=bi, **flags)
    ref = O.raw2outputs(raw.to(F64), z.to(F64), d.to(F64), **kw)
    got = P.raw2outputs(raw.to(DEV), z.to(DEV), d.to(DEV), **{k: (v.to(DEV) if torch.is_tensor(v) else v)
                                                              for k, v in kw.items()})
    assert set(got) == set(ref)
    w64 = ref["weights"]
    S = _abs_sums(raw.to(F64), z.to(F64), w64, C, K, sb, bs, bi, flags.get("sem_activation") == "softmax")
    if flags.get("white_bkgd"):
        S["rgb_map"] = S["rgb_map"] + S["acc_map"][:, None]
    w_max = w64.max(1).values
    worst = 0.0
    for k, s in S.items():
        per_ray = s.reshape(R, -1).max(1).values
        if k.startswith("fixed_"):
            per_ray = torch.maximum(per_ray, w_max)
        err = (got[k].cpu().double() - ref[k]).abs().reshape(R, -1)
        bound = 1e-4 * per_ray[:, None] + 2.0 ** -24 * ref[k].abs().reshape(R, -1)
        worst = max(worst, _ratio(err, bound))
    err = (got["weights"].cpu().double() - w64).abs()
    worst = max(worst, _ratio(err, 1e-4 * w_max[:, None].expand_as(err)))
    dg, dr = got["disp_map"].cpu().double(), ref["disp_map"]
    assert torch.equal(torch.isnan(dg), torch.isnan(dr))
    ok = ~torch.isnan(dr)
    worst = max(worst, _ratio((dg - dr)[ok].abs(), 2e-4 * dr[ok].abs()))
    _report(f"composite N={N} C={C} K={K} {flags}", worst)
    assert float(w64[R // 2: 3 * R // 4].max()) == 0.0                 # the all-empty quarter
    assert bool((got["weights"][R // 2: 3 * R // 4] == 0).all())


@pytest.mark.parametrize("N,C,K,flags", [
    (1, 1, 1, {}), (31, 32, 33, {"white_bkgd": True}), (32, 33, 32, {"mask_outside": True}), (33, 97, 96, {}),
    (225, 96, 97, {"white_bkgd": True, "mask_outside": True}), (256, 128, 128, {}),
    (256, 128, 128, {"mask_outside": True}), (256, 0, 0, {})])
def test_composite_backward_per_ray_against_float64(N, C, K, flags):
    """d(loss)/d(raw) against float64 autograd through the oracle's forward, with upstream gradients on every map.
    Per ray and channel group (rgb, sigma, semantic, instance): within 1e-4 of the ray's largest |ref| in that group,
    floored at 1e-6 of the group's RMS for rays whose gradient is ~0.  Logits of 1e4 go on every regime but the
    surface-like one: behind a surface whose alpha rounds to 1 in fp32, t = 1 - alpha + 1e-10 and so the transmittance
    are known only to an ulp of 1, and dL/dsigma there is G_i T_i with G_i ~ 1e5 - an fp32 limit of the forward's
    transmittance, which the backward recomputes bit for bit, not of the backward."""
    R = 128
    raw, z, d, sb, bs, bi = _composite_case(R, N, C, K, seed=N * 5 + C + 7 * K, big_on_surface=False)
    kw = dict(num_classes=C, num_instances=K, sample_box=sb, box_sem=bs, box_inst=bi, **flags)
    g = torch.Generator().manual_seed(N + C + K)
    x = raw.to(F64).requires_grad_(True)
    out = O.raw2outputs(x, z.to(F64), d.to(F64), **kw)
    ups = {k: torch.randn(v.shape, generator=g, dtype=F64) for k, v in out.items() if k != "disp_map"}
    (ref,) = torch.autograd.grad(sum((out[k] * u).sum() for k, u in ups.items()), x)
    got = P.raw2outputs_backward(raw.to(DEV), z.to(DEV), d.to(DEV), {k: u.float().to(DEV) for k, u in ups.items()},
                                 **{k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}).cpu().double()
    assert torch.isfinite(ref).all() and torch.isfinite(got).all()
    worst = 0.0
    for name, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4)), ("sem", slice(4, 4 + C)), ("inst", slice(4 + C, 4 + C + K))):
        r, a = ref[..., sl], got[..., sl]
        if r.numel() == 0:
            continue
        floor = 1e-6 * float(r.pow(2).mean().sqrt())
        per_ray = r.abs().reshape(R, -1).max(1).values.clamp(min=floor)
        e = _ratio((a - r).abs().reshape(R, -1), 1e-4 * per_ray[:, None].expand(R, a[0].numel()))
        print(f"  {name}: {e:.3e}")
        worst = max(worst, e)
    _report(f"composite backward N={N} C={C} K={K} {flags}", worst)


# ------------------------------------------------------------------------------------------------ losses
def _losses_direct(rgb, depth, sem, fix, rgb_gt, depth_gt, label, conf, nc, prob, eps, w=(1.0, 0.1, 0.5, 2.0)):
    """pnr_losses on the device: per-ray terms [R,4] and the map gradients."""
    R = rgb.shape[0]
    t = {k: v.to(DEV).contiguous() for k, v in dict(rgb=rgb, depth=depth, sem=sem, fix=fix, rgb_gt=rgb_gt,
                                                     depth_gt=depth_gt, conf=conf).items()}
    lab = label.to(DEV, torch.int32).contiguous()
    n_sem = max(int(((label >= 0) & (label < nc)).sum()), 1)
    n_depth = max(int((depth_gt > 0).sum()), 1)
    a = _capi.PnrLossArgs()
    a.R, a.C, a.sem_is_prob = R, nc, int(prob)
    a.rgb_map, a.rgb_gt, a.depth_map, a.depth_gt = (_capi.ptr(t[k]) for k in ("rgb", "rgb_gt", "depth", "depth_gt"))
    a.semantic_map, a.fixed_semantic_map, a.label, a.label_weight = _capi.ptr(t["sem"]), _capi.ptr(t["fix"]), _capi.ptr(lab), _capi.ptr(t["conf"])
    a.w_rgb, a.w_depth, a.w_sem, a.w_fix = w
    a.inv_n_rgb, a.inv_n_depth, a.inv_n_sem, a.eps = 1.0 / (3 * R), 1.0 / n_depth, 1.0 / n_sem, eps
    per_ray = torch.empty(R, 4, device=DEV)
    grads = {k: torch.empty_like(t[k]) for k in ("rgb", "depth", "sem", "fix")}
    a.per_ray = _capi.ptr(per_ray)
    a.d_rgb_map, a.d_depth_map = _capi.ptr(grads["rgb"]), _capi.ptr(grads["depth"])
    a.d_semantic_map, a.d_fixed_semantic_map = _capi.ptr(grads["sem"]), _capi.ptr(grads["fix"])
    _capi.check(_capi.lib().pnr_losses(C.byref(a), _capi.stream_ptr()), "pnr_losses")
    return per_ray.cpu(), {k: v.cpu() for k, v in grads.items()}, n_sem, n_depth


def _loss_case(R, C, prob, eps, seed):
    g = torch.Generator().manual_seed(seed)
    rgb, gt = torch.rand(R, 3, generator=g), torch.rand(R, 3, generator=g)
    depth = torch.rand(R, generator=g) * 50 + 1
    depth_gt = torch.where(torch.rand(R, generator=g) > 0.3, depth + torch.randn(R, generator=g), torch.zeros(R))
    if prob:
        sem = torch.rand(R, C, generator=g)
        sem = sem / sem.sum(1, keepdim=True)
    else:
        sem = torch.randn(R, C, generator=g) * 3
        big = torch.rand(R, generator=g) < 0.4
        sem[big] = torch.sign(sem[big]) * 1e4 * torch.rand(int(big.sum()), C, generator=g)     # logits up to +-1e4
        sem[big.nonzero()[::2, 0], 0] = sem[big].abs().max(1).values[::2]                      # near-tied maxima
    fix = torch.rand(R, C, generator=g) * (torch.rand(R, C, generator=g) > 0.5)
    label = torch.randint(-1, C + 1, (R,), generator=g)                                          # -1 and C: ignored
    conf = torch.rand(R, generator=g)
    conf[::9] = 0.0
    lab = label.clamp(0, C - 1)
    # probabilities exactly at 0, eps and 2 eps on the labelled channel (and a tiny sum elsewhere)
    for m, p in enumerate((0.0, eps, 2 * eps)):
        rows = torch.arange(m, R, 7)
        fix[rows, lab[rows]] = p
        if prob:
            sem[rows, lab[rows]] = p
    return rgb, depth, sem, fix, gt, depth_gt, label, conf


@pytest.mark.parametrize("C", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("prob", [False, True])
def test_losses_per_ray_against_float64(C, prob):
    """Per-ray terms within 1e-4 of their float64 value (plus 2^-23 x the largest input magnitude the term subtracts:
    logits of 1e4 make lse - s_label an fp32 difference of numbers ~1e4); map gradients per ray within 1e-4 of the
    ray's largest |ref|.  p == eps passes the gradient of max(p, eps), p == 0 does not, as torch.clamp_min."""
    R, eps = 2000, 2.0 ** -20                                          # eps exact in fp32: p == eps on both sides
    rgb, depth, sem, fix, gt, depth_gt, label, conf = _loss_case(R, C, prob, eps, seed=C * 2 + int(prob))
    per_ray, grads, n_sem, n_depth = _losses_direct(rgb, depth, sem, fix, gt, depth_gt, label, conf, C, prob, eps)
    maps = [t.to(F64).requires_grad_(True) for t in (rgb, depth, sem, fix)]
    w = (1.0, 0.1, 0.5, 2.0)
    total, _ = OL.losses(maps[0], None, maps[1], maps[2], maps[3], gt.to(F64), depth_gt.to(F64), label, conf.to(F64),
                         w, prob, eps)
    total.backward()
    # per-ray terms in float64
    has = (label >= 0) & (label < C)
    lab = label.clamp(0, C - 1)
    s64, f64 = sem.to(F64), fix.to(F64)
    if prob:
        l_sem = -torch.log(s64.gather(1, lab[:, None])[:, 0].clamp_min(eps))
        sem_scale = torch.zeros(R, dtype=F64)
    else:
        l_sem = torch.logsumexp(s64, 1) - s64.gather(1, lab[:, None])[:, 0]
        sem_scale = s64.abs().max(1).values
    ref = torch.stack([((rgb.to(F64) - gt.to(F64)) ** 2).sum(1),
                       torch.where(depth_gt > 0, (depth.to(F64) - depth_gt.to(F64)).abs(), torch.zeros(R, dtype=F64)),
                       torch.where(has, l_sem * conf.to(F64), torch.zeros(R, dtype=F64)),
                       torch.where(has, -torch.log(f64.gather(1, lab[:, None])[:, 0].clamp_min(eps)) * conf.to(F64),
                                   torch.zeros(R, dtype=F64))], 1)
    slack = torch.zeros(R, 4, dtype=F64)
    slack[:, 1] = 2.0 ** -23 * torch.maximum(depth.abs(), depth_gt.abs()).to(F64)
    slack[:, 2] = torch.where(has, 2.0 ** -23 * sem_scale * conf.to(F64), torch.zeros(R, dtype=F64))
    worst = _ratio((per_ray.double() - ref).abs(), 1e-4 * ref.abs() + slack)
    for name, m, i in (("rgb", maps[0], "rgb"), ("depth", maps[1], "depth"), ("sem", maps[2], "sem"), ("fix", maps[3], "fix")):
        r, a = m.grad.reshape(R, -1), grads[i].double().reshape(R, -1)
        floor = 1e-6 * float(r.pow(2).mean().sqrt())
        per = r.abs().max(1).values.clamp(min=floor)
        worst = max(worst, _ratio((a - r).abs(), 1e-4 * per[:, None].expand_as(r)))
    _report(f"losses C={C} prob={prob}", worst)
    # the eps edge, exactly: p == eps -> -w / (n eps) * conf, p == 0 -> 0
    rows_eps, rows_zero = torch.arange(1, R, 7), torch.arange(0, R, 7)
    for rows, live in ((rows_eps, True), (rows_zero, False)):
        rows = rows[has[rows] & (conf[rows] > 0)]
        gfix = grads["fix"][rows, lab[rows]]
        assert bool((gfix != 0).all()) if live else bool((gfix == 0).all())
    assert bool((grads["sem"][~has] == 0).all()) and bool((grads["fix"][conf == 0] == 0).all())


# ------------------------------------------------------------------------------------------------ labels and fusion
@pytest.mark.parametrize("C,K", [(129, 1000), (1000, 129), (32767, 129), (129, 32767)])
def test_label_tiles_and_fusion_at_wide_maps(C, K):
    R = 96 if max(C, K) > 1000 else 700
    g = torch.Generator().manual_seed(C + K)
    sem = torch.randn(R, C, generator=g)
    inst = torch.randn(R, K, generator=g)
    sem[::5] = sem[::5].round(decimals=0)                                  # ties: the lowest index wins
    inst[::3] = inst[::3].round(decimals=0)
    sem[3, C - 1] = sem[3].max() + 1                                       # maximum in the last channel
    sem[4, :] = float("nan")                                               # all NaN: label 0
    sem[6, : C // 2] = float("nan")
    inst[7, K - 1] = float("nan")
    rgb, depth = torch.rand(R, 3, generator=g) * 1.2 - 0.1, torch.rand(R, generator=g) * 50
    rgb_g, dep_g, sem_g, inst_g = rgb.to(DEV), depth.to(DEV), sem.to(DEV), inst.to(DEV)
    rgb8 = torch.empty(R, 3, dtype=torch.uint8, device=DEV)
    dep = torch.empty(R, device=DEV)
    sl = torch.empty(R, dtype=torch.int16, device=DEV)
    il = torch.empty(R, dtype=torch.int16, device=DEV)
    _capi.check(_capi.lib().pnr_label_tiles(rgb_g.data_ptr(), dep_g.data_ptr(), sem_g.data_ptr(), inst_g.data_ptr(),
                                            R, C, K, rgb8.data_ptr(), dep.data_ptr(), sl.data_ptr(), il.data_ptr(),
                                            _capi.stream_ptr()), "pnr_label_tiles")
    assert torch.equal(sl.cpu(), OP._argmax_first(sem).to(torch.int16))
    assert torch.equal(il.cpu(), OP._argmax_first(inst).to(torch.int16))
    assert int(sl[3]) == C - 1 and int(sl[4]) == 0
    assert torch.equal(rgb8.cpu().float(), torch.round(rgb.clamp(0, 1) * 255)) and torch.equal(dep.cpu(), depth)
    is_thing = (torch.rand(C, generator=g) > 0.5).to(torch.uint8)
    inst_class = torch.randint(0, C, (K,), generator=g)
    inst_class[: K // 2] = OP._argmax_first(sem)[torch.arange(K // 2) % R].clamp(min=0)   # many rays have slots
    is_thing[inst_class[: K // 2]] = 1
    inst_id = inst_class * 1000 + torch.arange(K) + 1
    class_id = torch.randperm(C, generator=g) + 3
    pal = torch.randint(0, 256, (C, 3), generator=g, dtype=torch.uint8)
    got = fuse_panoptic({"semantic_map": sem_g, "instance_map": inst_g}, is_thing, inst_class, inst_id, class_id, pal)
    pan, s, k, col = OP.panoptic_fuse(sem, inst, is_thing, inst_class, inst_id, class_id, pal)
    assert torch.equal(got["semantic"].cpu(), s) and torch.equal(got["instance_slot"].cpu(), k)
    assert torch.equal(got["panoptic"].cpu(), pan) and torch.equal(got["color"].cpu(), col)
    assert int((k >= 0).sum()) > 0


# ------------------------------------------------------------------------------------------------ encoders
@pytest.mark.parametrize("n", [1, 127, 129, 1000 + 37])
def test_encode_at_16_bands_against_float64(n):
    """gamma(x) at L = 16 (the largest: a 50 KB shared tile per 128 samples) against sin / cos in float64 of the same
    fp32 x: within 2 ulps of 1 (the power-of-two scaling is exact, sincosf is accurate over the full range)."""
    L = 16
    g = torch.Generator().manual_seed(n)
    x = (torch.rand(n, 3, generator=g) - 0.5) * 128.0
    x[0] = torch.tensor([0.0, math.pi / 2, -64.0])
    got = P.embed(x.to(DEV), L).cpu().double()
    ref = O.embed(x.to(F64), L)
    assert got.shape == (n, 3 + 6 * L)
    assert torch.equal(got[:, :3], x.double())
    _report(f"encode L=16 n={n}", float((got - ref).abs().max()) / 2.0 ** -22)


# (L, F, T_log2, base, scale): level resolutions with (res+1)^3 == 2^T exactly (dense, the last such level), T = 2^4,
# and L = 32
HASH_CASES = [(4, 2, 12, 3.0, 2.0),        # res 3, 6, 12, 24: 13^3 = 2197 <= 4096 dense, 25^3 hashed
              (3, 4, 12, 15.0, 1.0),       # res 15: 16^3 == 2^12, dense at equality
              (2, 8, 9, 7.0, 1.2),         # res 7, 8: 8^3 == 2^9 dense, 9^3 hashed
              (3, 1, 4, 1.0, 2.0),         # T = 16: res 1 dense (8 <= 16), res 2 and 4 hashed
              (32, 2, 10, 2.0, 1.25)]      # L = 32


def _hash_points(n, seed, res_list):
    """Points in [-1, 1]^3 (aabb), a share of them outside and a share exactly on cell faces of every level."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, generator=g) * 2.4 - 1.2
    faces = n // 4
    res = torch.tensor(res_list)[torch.randint(0, len(res_list), (faces,), generator=g)].float()
    k = torch.floor(torch.rand(faces, 3, generator=g) * (res[:, None] + 1))
    x[:faces] = (k / res[:, None]) * 2.0 - 1.0                # exact in fp32 for these resolutions (powers of two / small)
    x[faces] = torch.tensor([1.0, -1.0, 1.0])
    return x


@pytest.mark.parametrize("L,F,T_log2,base,scale", HASH_CASES)
def test_hashgrid_edges_forward_bit_exact_and_backward_against_float64(L, F, T_log2, base, scale):
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    res = OP.hashgrid_resolutions(L, base, scale)
    n = 3000
    x = _hash_points(n, L * 100 + T_log2, res)
    enc = HashGrid(L, F, T_log2, base, scale, aabb=aabb, seed=L + F)
    with torch.no_grad():
        enc.table.mul_(1e4)
    table = enc.table.detach().clone()
    ref = OP.hashgrid_encode(x, aabb, table, base, scale)
    encd = enc.to(DEV)
    got = encd(x.to(DEV))
    assert torch.equal(got.detach().cpu(), ref)
    # backward: float64 autograd through the oracle's gather (the trilinear weights are the fp32 ones the kernel uses)
    g = torch.Generator().manual_seed(T_log2)
    up = torch.randn(n, L * F, generator=g)
    t64 = table.to(F64).requires_grad_(True)
    (OP.hashgrid_encode(x, aabb, t64, base, scale) * up.to(F64)).sum().backward()
    t64a = table.to(F64).requires_grad_(True)
    (OP.hashgrid_encode(x, aabb, t64a, base, scale) * up.abs().to(F64)).sum().backward()   # sum_k w_k |g|: the scale
    (got * up.to(DEV)).sum().backward()
    gt_ = encd.table.grad.cpu().double()
    assert torch.equal(gt_ == 0, t64a.grad == 0)
    _report(f"hashgrid backward L={L} F={F} T=2^{T_log2}", _ratio((gt_ - t64.grad).abs(), 1e-4 * t64a.grad))
