"""The compositing epilogue of the fused MLP kernel and pnr_render_fused at the limits they accept.

- pnr_mlp_composite (compositing in the MLP kernel's epilogue, raw never written) is compared ray by ray with the
  float64 compositing of the kernel's own raw: pnr_mlp_forward on the same rays and depths.  The epilogue forms sigma,
  rgb and logits in the order of the kernel that writes raw, so this reference isolates the epilogue from the MLP's
  rounding and every precision is held to one bound, the one of test_gpu_stage_limits'
  test_composite_per_ray_against_float64.  The matrix crosses the epilogue's own structure: rays of 1 to 8 groups of
  32 samples over tiles of 64 (N = 32 .. 256, rays that start mid-tile, four tiles per ray), CTA ranges of whole rays
  that end mid-tile or are empty (R around multiples of the persistent grid, read from the device), the widest channel
  fold (5 + 128 + 128), logits of 1e4, and rays whose transmittance underflows inside a tile.
- pnr_render_fused is called through ctypes with the buffer sets, near / far sources, pass mixes and workspaces the
  Python Renderer never passes, and compared with the staged path on the same networks: integers, depths and weights
  bit for bit, the summed maps per ray against the float64 compositing of the staged raw of each pass.
Each float64 comparison prints its largest error over its bound (1 is the bound).
"""
import ctypes as C
import re

import pytest
import torch

from oracle import reference_renderer as O
from oracle_hashgrid import hash_cfg
from panopticnerf_b200 import _capi, make_cfg, make_network, make_renderer, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from test_gpu_stage_limits import _abs_sums, _ratio, _report

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
I32 = torch.int32
KROWS = 64                                 # samples per tile of the fused MLP kernel (csrc/mlp_program.h kRows)
PAD = 3                                    # sentinel rows past R in every output
SENT = {torch.float32: -12345.0, torch.int32: -777, torch.uint8: 77}
SIGMA0 = 1000.0                            # sigma >= SIGMA0 everywhere: the depths decide each ray's regime
N_BOXES = 20                               # primitives of the epilogue cases; the render cases use 64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cta_split(R, N):
    """(grid, rays_per_cta) of a compositing launch: the persistent grid is min(tiles of 64 samples, SMs), and every
    CTA owns ceil(R / grid) whole rays; its tiles start at its first sample."""
    grid = min(-(-R * N // KROWS), _sms())
    return grid, -(-R // grid)


def _rays_for(spec, N):
    sms = _sms()
    if spec == "one":
        return 1
    if spec == "lt_grid":                  # fewer rays than CTAs: the last CTAs own nothing
        return sms // 2 + 3
    if spec == "large":                    # many tiles per CTA
        return 40 * sms
    if spec == "odd":                      # rays_per_cta x N an odd number of 32-sample groups: ranges end mid-tile
        rpc = next(r for r in (1, 3, 5, 7) if r * N % KROWS == 32 and r * N > KROWS)
        return rpc * sms
    k = 1                                  # k * grid - 1, k * grid, k * grid + 1 with the grid at its full size
    while -(-(k * sms - 1) * N // KROWS) < sms:
        k += 1
    return k * sms + {"k-1": -1, "k": 0, "k+1": 1}[spec]


def _sentinel(*shape, dtype=torch.float32):
    return torch.full(shape, SENT[dtype], dtype=dtype, device=DEV)


def _check_pads(bufs, R):
    for k, v in bufs.items():
        assert bool((v[R:] == SENT[v.dtype]).all()), f"{k}: a row past R was written"


def _bits_equal(a, b, what):
    a, b = a.cpu(), b.cpu()
    assert a.shape == b.shape, f"{what}: {tuple(a.shape)} vs {tuple(b.shape)}"
    if a.is_floating_point():
        assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{what}: NaN patterns differ"
        a, b = torch.nan_to_num(a), torch.nan_to_num(b)
    assert torch.equal(a, b.to(a.dtype)), f"{what} differs ({int((a != b.to(a.dtype)).sum())} elements)"


def _per_ray_ratio(got, raw, z, rays, Cn, Kn, sb, bs, bi, white, mask, softmax, suffix=""):
    """Largest error / bound of one pass's maps against the float64 compositing of `raw`, and the name of the map it
    was found in.  The bound model of test_composite_per_ray_against_float64: each map element within
    1e-4 x sum_i |w_i v_i| of its ray (the largest over the map's channels) plus half an ulp of the stored value, the
    fixed maps' sum floored at the ray's largest weight; weights within 1e-4 of the ray's largest.  Plus one term for
    nearly transparent samples (rendered scenes have them, with sigma x delta ~ 1e-6): fp32 alpha = 1 - expf(-x) is
    exact in its subtraction but expf is within 2 ulps of its value just below 1, so alpha is known only to 2^-23
    absolute.  Where 0 < x < 2^-6 that is more than 1.5e-5 of alpha, so weight i there carries 2^-22 T_i (twice that,
    T_i the float64 transmittance) and a map sum_i 2^-22 T_i |v_i| over those samples; elsewhere alpha is exactly 0
    (masked samples, zero-length deltas) or within 1.5e-5 of itself, inside the 1e-4 model.  disp = 1 / (depth / acc)
    within the sum of depth's and acc's relative bounds."""
    R = z.shape[0]
    raw64, z64, d64 = raw.cpu().double(), z.cpu().double(), rays[:, 3:].cpu().double()
    if sb is None:                          # no boxes: no fixed maps, the sums below see no box
        sb = torch.full(z.shape, -1, dtype=I32)
        bs = bi = torch.zeros(0, dtype=I32)
    sb, bs, bi = sb.cpu(), (bs.cpu() if bs is not None else None), (bi.cpu() if bi is not None else None)
    kw = dict(num_classes=Cn, num_instances=Kn, white_bkgd=white, mask_outside=mask, sample_box=sb, box_sem=bs,
              box_inst=bi, sem_activation="softmax" if softmax else "none")
    ref = O.raw2outputs(raw64, z64, d64, **kw)
    w64 = ref["weights"]
    sums = _abs_sums(raw64, z64, w64, Cn, Kn, sb, bs if bs is not None else torch.zeros(0, dtype=I32),
                     bi if bi is not None else torch.zeros(0, dtype=I32), softmax)
    dist = torch.cat([z64[:, 1:] - z64[:, :-1], torch.full_like(z64[:, :1], 1e10)], -1) * d64.norm(dim=-1)[:, None]
    sig = torch.relu(raw64[..., 3])
    if mask:
        sig = torch.where(sb >= 0, sig, torch.zeros_like(sig))
    x = sig * dist
    t = torch.cat([torch.ones_like(sig[:, :1]), torch.exp(-x) + 1e-10], -1)
    u = torch.where((x > 0) & (x < 2.0 ** -6), 2.0 ** -22 * torch.cumprod(t, -1)[:, :-1], torch.zeros_like(x))
    usums = _abs_sums(raw64, z64, u, Cn, Kn, sb, bs if bs is not None else torch.zeros(0, dtype=I32),
                      bi if bi is not None else torch.zeros(0, dtype=I32), softmax)
    if white:
        sums["rgb_map"] = sums["rgb_map"] + sums["acc_map"][:, None]
        usums["rgb_map"] = usums["rgb_map"] + usums["acc_map"][:, None]
    w_max = w64.max(1).values
    worst, where = 0.0, ""
    bounds = {}
    for k, s in sums.items():
        per_ray = s.reshape(R, -1).max(1).values
        if k.startswith("fixed_"):
            per_ray = torch.maximum(per_ray, w_max)
        bounds[k] = (1e-4 * per_ray + usums[k].reshape(R, -1).max(1).values)[:, None] \
            + 2.0 ** -24 * ref[k].abs().reshape(R, -1)
        if k + suffix in got:
            err = (got[k + suffix].cpu().double() - ref[k]).abs().reshape(R, -1)
            worst, where = max((worst, where), (_ratio(err, bounds[k]), k))
    if "weights" + suffix in got:
        err = (got["weights" + suffix].cpu().double() - w64).abs()
        worst, where = max((worst, where), (_ratio(err, 1e-4 * w_max[:, None] + u), "weights"))
    if "disp_map" + suffix in got:
        dg, dr = got["disp_map" + suffix].cpu().double(), ref["disp_map"]
        assert torch.equal(torch.isnan(dg), torch.isnan(dr)), "disp_map: NaN patterns differ"
        ok = ~torch.isnan(dr)
        rel = bounds["depth_map"][:, 0] / ref["depth_map"].abs() + bounds["acc_map"][:, 0] / ref["acc_map"].abs()
        worst, where = max((worst, where), (_ratio((dg - dr)[ok].abs(), rel[ok] * dr[ok].abs()), "disp_map"))
    return worst, where


# ------------------------------------------------------------------------------------------------ the epilogue
def _epilogue_network(N, Cn, Kn, precision, grid, seed):
    """The initialised network with alpha_linear made positive and biased to SIGMA0 (sigma >= SIGMA0 wherever the trunk
    output is >= 0, i.e. everywhere)."""
    over = dict(N_samples=N, N_importance=0, num_classes=Cn, num_instances=Kn, precision=precision)
    cfg = (hash_cfg("cfg2", hash_levels=grid[0], hash_features=grid[1], hash_log2_size=14, **over) if grid
           else make_cfg("cfg2", **over))
    net = S.init_network_weights(make_network(cfg), seed=seed)
    with torch.no_grad():
        net.alpha_linear.weight.abs_()
        net.alpha_linear.bias.fill_(SIGMA0)
    return cfg, net.to(DEV)


def _epilogue_inputs(R, N, Cn, Kn, seed):
    """Rays in four regimes, interleaved (ray r is in regime r % 4, so neighbouring rays of a CTA differ):
    0 mid-range: depth steps of ~2 / (SIGMA0 N) per unit of |d|, an optical depth of ~2 over the ray;
    1 surface-like: samples before a random index are outside every box (masked under mask_outside), the rest are
      >= 0.03 / |d| apart, so sigma x delta >= 30, alpha rounds to 1 and the transmittance underflows;
    2 empty: every sample outside every box (all masked under mask_outside);
    3 zero-length deltas: depths repeated in runs.
    Sample boxes run from -3 to B + 2 and the id tables hold ids from -2 to C + 2 / K + 2."""
    g = torch.Generator().manual_seed(seed)
    reg = torch.arange(R) % 4
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1) * (0.5 + torch.rand(R, 1, generator=g))
    o = torch.randn(R, 3, generator=g)
    dn = d.norm(dim=-1, keepdim=True)
    near = 0.5 + 2 * torch.rand(R, 1, generator=g)
    z_mid = near + torch.cumsum(torch.rand(R, N, generator=g) * 4.0 / (SIGMA0 * N) / dn, -1)
    z_surf = near + torch.cumsum((0.03 + 0.03 * torch.rand(R, N, generator=g)) / dn, -1)
    z_dup = near + torch.sort(torch.randint(0, max(N // 3, 2), (R, N), generator=g).float(), -1).values \
        * (6.0 / (SIGMA0 * N)) / dn
    z = torch.where((reg == 1)[:, None], z_surf, torch.where((reg == 3)[:, None], z_dup, z_mid))
    sb = torch.randint(-3, N_BOXES + 3, (R, N), generator=g, dtype=I32)
    surf_at = torch.randint(0, max(N - 8, 1), (R, 1), generator=g)   # >= 8 samples behind the surface
    inside = torch.randint(0, N_BOXES + 3, (R, N), generator=g, dtype=I32)
    sb = torch.where((reg == 1)[:, None], torch.where(torch.arange(N)[None] < surf_at, torch.full_like(sb, -1), inside), sb)
    sb[reg == 2] = -1 - torch.randint(0, 3, (int((reg == 2).sum()), N), generator=g, dtype=I32)
    bs = torch.randint(-2, max(Cn, 1) + 3, (N_BOXES,), generator=g, dtype=I32)
    bi = torch.randint(-2, max(Kn, 1) + 3, (N_BOXES,), generator=g, dtype=I32)
    rays = torch.cat([o, d], -1).contiguous()
    return rays.to(DEV), z.contiguous().to(DEV), sb.to(DEV), bs.to(DEV), bi.to(DEV), reg


def _scale_logits(net, rays, z):
    """Scale the heads' output layers so that the largest |logit| on these samples is 1e4 (fp32 outputs of the kernel,
    not 16-bit operands: the range check stays clear)."""
    raw = net.forward_rays(rays, z)
    m = float(raw[..., 4:].abs().max())
    with torch.no_grad():
        for heads in (getattr(net, "semantic_linears", None), getattr(net, "instance_linears", None)):
            if heads is not None:
                heads[1].weight.mul_(1e4 / m)
                heads[1].bias.mul_(1e4 / m)


def _composite_direct(net, rays, z, white, mask, sb, bs, bi):
    """pnr_mlp_composite into outputs with PAD sentinel rows past R (which must stay untouched)."""
    R, N = z.shape
    Cn, Kn = net.C, net.K
    out = {"rgb_map": _sentinel(R + PAD, 3), "depth_map": _sentinel(R + PAD), "acc_map": _sentinel(R + PAD),
           "disp_map": _sentinel(R + PAD), "weights": _sentinel(R + PAD, N)}
    if Cn:
        out["semantic_map"], out["fixed_semantic_map"] = _sentinel(R + PAD, Cn), _sentinel(R + PAD, Cn)
    if Kn:
        out["instance_map"], out["fixed_instance_map"] = _sentinel(R + PAD, Kn), _sentinel(R + PAD, Kn)
    co = _capi.PnrCompositeOut(**{k: _capi.ptr(out[k]) if k in out else None for k, _ in _capi.PnrCompositeOut._fields_})
    ctx = net.pack(torch.device(DEV))
    _capi.check(_capi.lib().pnr_mlp_composite(ctx, _capi.ptr(rays), _capi.ptr(z), R, N, int(white), int(mask),
                                              _capi.ptr(sb), _capi.ptr(bs), _capi.ptr(bi), bs.shape[0], C.byref(co),
                                              _capi.stream_ptr()), "pnr_mlp_composite")
    _check_pads(out, R)
    return {k: v[:R] for k, v in out.items()}


# (N, C, K, precision, rays, flags, hash grid (levels, features))
EPILOGUE = [
    (32, 1, 0, "fp16x3", "k-1", "mask", None),
    (32, 0, 1, "bf16x3", "odd", "mask,white", None),
    (64, 45, 64, "fp16", "one", "mask", None),
    (64, 0, 1, "fp16x3", "large", "mask", None),
    (64, 3, 6, "fp16x3", "k", "mask", (5, 2)),
    (96, 45, 64, "fp16x3", "k+1", "mask", None),
    (96, 128, 1, "bf16x3", "odd", "mask", None),
    (128, 128, 128, "fp16x3", "k+1", "mask", None),
    (128, 45, 64, "fp16x3", "k-1", "white", None),
    (160, 128, 128, "fp16x3", "k", "mask,white", None),
    (224, 128, 1, "bf16x3", "lt_grid", "mask,white", None),
    (224, 45, 64, "fp16x3", "odd", "mask", None),
    (256, 128, 128, "fp16x3", "k-1", "mask,white", None),
    (256, 1, 0, "bf16x3", "one", "mask", None),
]


@pytest.mark.parametrize("N,Cn,Kn,precision,rays_spec,flags,grid", EPILOGUE,
                         ids=[f"N{c[0]}-C{c[1]}K{c[2]}-{c[3]}-R{c[4]}-{c[5]}" + ("-hash" if c[6] else "") for c in EPILOGUE])
def test_epilogue_per_ray_against_float64(N, Cn, Kn, precision, rays_spec, flags, grid):
    """pnr_mlp_composite per ray against the float64 compositing of pnr_mlp_forward's raw on the same samples; weights
    and both fixed maps equal to the two-kernel path (pnr_composite on that raw) bit for bit; rows past R untouched."""
    white, mask = "white" in flags, "mask" in flags
    R = _rays_for(rays_spec, N)
    grid_size, rpc = _cta_split(R, N)
    if rays_spec == "odd":
        assert grid_size == _sms() and rpc * N % KROWS == 32
    if rays_spec == "lt_grid":
        assert R < grid_size
    cfg, net = _epilogue_network(N, Cn, Kn, precision, grid, seed=N + Cn + Kn)
    rays, z, sb, bs, bi, reg = _epilogue_inputs(R, N, Cn, Kn, seed=R + N)
    if Cn + Kn:
        _scale_logits(net, rays, z)
    got = _composite_direct(net, rays, z, white, mask, sb, bs, bi)
    raw = net.forward_rays(rays, z)
    two = P.raw2outputs(raw, z, rays, white_bkgd=white, mask_outside=mask, num_classes=Cn, num_instances=Kn,
                        sample_box=sb, box_sem=bs, box_inst=bi)
    assert set(got) == set(two)
    for k in ("weights", "fixed_semantic_map", "fixed_instance_map"):
        if k in two:
            _bits_equal(got[k], two[k], k)
    worst, where = _per_ray_ratio(got, raw, z, rays, Cn, Kn, sb, bs, bi, white, mask, softmax=False)
    _report(f"epilogue N={N} C={Cn} K={Kn} {precision} R={R} (grid {grid_size}, {rpc} rays per CTA) {flags}"
            + (f" hash {grid}" if grid else "") + f" [{where}]", worst)
    assert net.range_status() == 0
    if Cn + Kn:
        assert float(raw[..., 4:].abs().max()) >= 5e3
    if R >= 4:
        assert float(got["weights"][reg == 0].sum()) > 0
        if mask:
            assert bool((got["weights"][reg == 2] == 0).all())
        surf = got["weights"][reg == 1]
        assert bool((surf.max(1).values > 0.999).all())                 # alpha rounds to 1 at the surface
        assert bool(((surf == 0).sum(1) > 0).all())                      # and the transmittance underflows behind it


# ------------------------------------------------------------------------------------------------ pnr_render_fused
BUFFERS = ("all", "none", "no_out0", "no_z", "no_hits")
NEAR_FAR = ("arrays", "aabb", "fill")
AABB = [float(v) for v in S.SCENE_AABB[0] + S.SCENE_AABB[1]]


def _render_inputs(cfg, R, M, perturb, stride0, near_far, seed):
    g = torch.Generator().manual_seed(seed)
    N, Ni = cfg.N_samples, cfg.N_importance
    batch = S.make_batch(cfg, row0=cfg.H // 3, rows=-(-R // cfg.W_img) + 1, seed=seed, num_boxes=64)
    rays = batch["rays"][torch.randperm(batch["rays"].shape[0], generator=g)[:R]].contiguous()
    bs = torch.randint(-2, max(cfg.num_classes, 1) + 3, (64,), generator=g, dtype=I32)
    bi = torch.randint(-2, max(cfg.num_instances, 1) + 3, (64,), generator=g, dtype=I32)
    inp = dict(rays=rays.to(DEV), box_center=batch["box_center"].to(DEV), box_half=batch["box_half"].to(DEV),
               box_rot=batch["box_rot"].to(DEV), box_sem=bs.to(DEV), box_inst=bi.to(DEV), M=M, perturb=perturb,
               t_vals=torch.linspace(0.0, 1.0, N).to(DEV), near_far=near_far)
    if near_far == "arrays":
        near, far = P.scene_near_far(inp["rays"], batch["scene_aabb"], cfg.near, cfg.far)
        inp["near"], inp["far"] = near, torch.minimum(far, torch.full_like(far, 45.0))
    if perturb > 0:
        inp["u"] = torch.rand(R, N, generator=g).to(DEV)
    if Ni:
        if stride0:
            row = torch.linspace(0.0, 1.0, Ni) if perturb == 0 else torch.sort(torch.rand(Ni, generator=g)).values
            inp["u_fine"], inp["u_fine_stride"] = row.to(DEV), 0
            inp["u_fine_rows"] = row[None].expand(R, Ni).contiguous().to(DEV)
        else:
            u = torch.rand(R, Ni, generator=g)
            u = u if perturb > 0 else torch.sort(u, -1).values
            inp["u_fine"] = inp["u_fine_rows"] = u.to(DEV)
            inp["u_fine_stride"] = Ni
    return inp


def _fused(ctx, ctx_fine, cfg, inp, buffers="all", R=None, ws_bytes=None, ws=None):
    """One pnr_render_fused call with the given buffer set; every output has PAD sentinel rows past R.
    Returns (rc, error text, outputs[:R])."""
    R = inp["rays"].shape[0] if R is None else R
    N, Ni = cfg.N_samples, cfg.N_importance
    Nt, Cn, Kn, M, Rp = N + Ni, cfg.num_classes, cfg.num_instances, inp["M"], R + PAD
    bufs = {}

    def maps(suffix, n):
        m = {"rgb_map": _sentinel(Rp, 3), "depth_map": _sentinel(Rp), "acc_map": _sentinel(Rp), "disp_map": _sentinel(Rp)}
        if buffers != "none":
            m["weights"] = _sentinel(Rp, n)
        if Cn:
            m["semantic_map"], m["fixed_semantic_map"] = _sentinel(Rp, Cn), _sentinel(Rp, Cn)
        if Kn:
            m["instance_map"], m["fixed_instance_map"] = _sentinel(Rp, Kn), _sentinel(Rp, Kn)
        bufs.update({k + suffix: v for k, v in m.items()})
        return _capi.PnrCompositeOut(**{k: _capi.ptr(m[k]) if k in m else None for k, _ in _capi.PnrCompositeOut._fields_})

    a = _capi.PnrRenderArgs()
    a.rays, a.R = _capi.ptr(inp["rays"]), R
    if inp["near_far"] == "arrays":
        a.near, a.far = _capi.ptr(inp["near"]), _capi.ptr(inp["far"])
    aabb = (C.c_float * 6)(*AABB)
    if inp["near_far"] == "aabb":
        a.aabb_host = C.cast(aabb, C.POINTER(C.c_float))
    a.near_min, a.far_default = cfg.near, cfg.far
    a.box_center, a.box_half, a.box_rot = (_capi.ptr(inp[k]) for k in ("box_center", "box_half", "box_rot"))
    a.box_sem, a.box_inst, a.M = _capi.ptr(inp["box_sem"]), _capi.ptr(inp["box_inst"]), M
    a.B = inp["box_center"].shape[0]
    a.N, a.Ni, a.t_vals = N, Ni, _capi.ptr(inp["t_vals"])
    a.u, a.perturb = _capi.ptr(inp.get("u")), inp["perturb"]
    if Ni:
        a.u_fine, a.u_fine_stride = _capi.ptr(inp["u_fine"]), inp["u_fine_stride"]
    a.sample_mode = _capi.SAMPLE_MODE[cfg.sample_mode]
    a.white_bkgd, a.sem_softmax = int(cfg.white_bkgd), int(cfg.sem_activation == "softmax")
    a.mask_outside, a.bound_by_primitives = int(cfg.mask_outside), int(cfg.bound_by_primitives)
    a.out = maps("", Nt)
    if Ni and buffers != "no_out0":
        a.out0 = maps("_0", N)
    if buffers not in ("none", "no_z"):
        bufs["z_vals"] = _sentinel(Rp, Nt)
        a.z_vals = _capi.ptr(bufs["z_vals"])
        if Ni:
            bufs["z_vals_0"] = _sentinel(Rp, N)
            a.z_vals0 = _capi.ptr(bufs["z_vals_0"])
    if buffers not in ("none", "no_hits"):
        bufs.update(hit_mask=_sentinel(Rp, dtype=torch.uint8), box_id=_sentinel(Rp, M, dtype=I32),
                    t_in=_sentinel(Rp, M), t_out=_sentinel(Rp, M))
        a.hit_mask, a.box_id, a.t_in, a.t_out = (_capi.ptr(bufs[k]) for k in ("hit_mask", "box_id", "t_in", "t_out"))
    if buffers != "none":
        bufs.update(sample_box=_sentinel(Rp, Nt, dtype=I32), near_out=_sentinel(Rp), far_out=_sentinel(Rp))
        a.sample_box, a.near_out, a.far_out = (_capi.ptr(bufs[k]) for k in ("sample_box", "near_out", "far_out"))
    if ws_bytes is None:
        ws_bytes = int(_capi.lib().pnr_workspace_bytes(ctx, R, N, Ni))
    if ws is None:
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws_bytes
    rc = _capi.lib().pnr_render_fused(ctx, ctx_fine, C.byref(a), _capi.stream_ptr())
    msg = _capi.lib().pnr_last_error().decode() if rc else ""
    torch.cuda.synchronize()
    _check_pads(bufs, R)
    return rc, msg, {k: v[:R] for k, v in bufs.items()}


def _with(cfg, **over):
    d = dict(vars(cfg))
    preset = d.pop("preset")
    return make_cfg(preset, **dict(d, **over))


def _staged(cfg, net, net_fine, inp):
    """The stage-by-stage Renderer on the same inputs (return_raw keeps the final pass's raw)."""
    scfg = _with(cfg, render_path="staged", return_raw=True, max_hits=inp["M"])
    batch = {k: inp[k] for k in ("rays", "box_center", "box_half", "box_rot", "box_sem", "box_inst")}
    batch["perturb"] = inp["perturb"]
    if inp["near_far"] == "arrays":
        batch["near"], batch["far"] = inp["near"], inp["far"]
    elif inp["near_far"] == "aabb":
        batch["scene_aabb"] = torch.tensor(S.SCENE_AABB)
    if "u" in inp:
        batch["u"] = inp["u"]
    if cfg.N_importance:
        batch["u_fine"] = inp["u_fine_rows"]
    return make_renderer(scfg, net, net_fine).render(batch)


def _compare_with_staged(cfg, net, net_fine, inp, got, what):
    ref = _staged(cfg, net, net_fine, inp)
    Cn, Kn, softmax = cfg.num_classes, cfg.num_instances, cfg.sem_activation == "softmax"
    exact = ["hit_mask", "box_id", "t_in", "t_out", "sample_box", "z_vals", "z_vals_0", "weights", "weights_0",
             "fixed_semantic_map", "fixed_instance_map", "fixed_semantic_map_0", "fixed_instance_map_0"]
    if softmax:                             # both passes take the two-kernel path: every map bit for bit
        exact += [k for k in got if k not in exact and k not in ("near_out", "far_out")]
    for k in exact:
        if k in got:
            _bits_equal(got[k], ref[k].to(got[k].dtype) if k == "hit_mask" else ref[k], f"{what} {k}")
    if "near_out" in got:
        near, far = ref["near"], ref["far"]
        if cfg.bound_by_primitives:
            near, far = P.bound_by_primitives(ref["hit_mask"], ref["box_id"], ref["t_in"], ref["t_out"], near, far)
        _bits_equal(got["near_out"], near, f"{what} near_out")
        _bits_equal(got["far_out"], far, f"{what} far_out")
    rays, bs, bi = inp["rays"], inp["box_sem"], inp["box_inst"]
    flags = dict(white=cfg.white_bkgd, mask=cfg.mask_outside, softmax=softmax)
    worst, where = _per_ray_ratio(got, ref["raw"], ref["z_vals"], rays, Cn, Kn, ref["sample_box"], bs, bi, **flags)
    if cfg.N_importance and "rgb_map_0" in got:
        z0 = ref["z_vals_0"]
        sb0 = P.tag_samples(z0, ref["box_id"], ref["t_in"], ref["t_out"])
        w0, where0 = _per_ray_ratio(got, net.forward_rays(rays, z0), z0, rays, Cn, Kn, sb0, bs, bi, suffix="_0", **flags)
        worst, where = max((worst, where), (w0, where0 + "_0"))
    assert net.range_status() == 0 and net_fine.range_status() == 0
    return worst, where


MIXES = [(64, 192), (64, 100), (48, 80), (48, 50), (3, 253), (256, 0), (32, 0)]
HEADS = {"heads": dict(num_classes=128, num_instances=128), "noheads": dict(),
         "softmax": dict(num_classes=128, num_instances=128, sem_activation="softmax")}
RENDER = [(N, Ni, h) for N, Ni in MIXES for h in HEADS]


def _variant(i):
    """The buffer set, near / far source, hits kept, sampler and flags of case i (cycled so that the pass mixes and head
    sets meet each of them)."""
    return dict(buffers=BUFFERS[i % 5], near_far=NEAR_FAR[i % 3], M=(8, 1)[i % 2], intervals=i % 4 == 1,
                perturb=float((i // 2) % 2), stride0=i % 3 == 2, white=i % 7 == 3, mask=i % 2 == 0)


def _render_cfg(N, Ni, heads, v, **over):
    return make_cfg("cfg2", D=4, W=128, N_samples=N, N_importance=Ni, white_bkgd=v["white"], mask_outside=v["mask"],
                    sample_mode="intervals" if v["intervals"] else "uniform", bound_by_primitives=v["intervals"],
                    max_hits=v["M"], **dict(HEADS[heads], **over))


@pytest.mark.parametrize("i", range(len(RENDER)), ids=[f"N{N}-Ni{Ni}-{h}" for N, Ni, h in RENDER])
def test_render_fused_against_staged_and_float64(i):
    """Every pass mix of N + Ni <= 256 (both passes one kernel, coarse only, fine only, neither, N = 3, single passes)
    with C = K = 128 heads, without heads and with softmax, each with another buffer set / near-far source / sampler;
    the default workspace pnr_workspace_bytes(ctx, R, N, Ni)."""
    N, Ni, heads = RENDER[i]
    v = _variant(i)
    cfg = _render_cfg(N, Ni, heads, v)
    net = S.init_network_weights(make_network(cfg), seed=i).to(DEV)
    inp = _render_inputs(cfg, 97, v["M"], v["perturb"], v["stride0"], v["near_far"], seed=i)
    rc, msg, got = _fused(net.pack(torch.device(DEV)), None, cfg, inp, v["buffers"])
    assert rc == 0, msg
    worst, where = _compare_with_staged(cfg, net, net, inp, got, f"case {i}")
    _report(f"render_fused N={N} Ni={Ni} {heads} {v} [{where}]", worst)


@pytest.mark.parametrize("fine_over", [dict(), dict(D=6, W=64, precision="bf16x3")], ids=["same-arch", "D6-W64-bf16x3"])
@pytest.mark.parametrize("mix", [(64, 192), (48, 80)], ids=["both-one-kernel", "fine-only"])
def test_render_fused_with_a_distinct_fine_network(mix, fine_over):
    """ctx_fine with other weights, or another depth / width / precision with the same heads, against the staged path
    with make_renderer(cfg, net, net_fine)."""
    v = dict(_variant(0), buffers="all", perturb=1.0, stride0=False)
    cfg = _render_cfg(*mix, "heads", v, num_classes=45, num_instances=64)
    net = S.init_network_weights(make_network(cfg), seed=1).to(DEV)
    fine_cfg = _with(cfg, **fine_over)
    net_fine = S.init_network_weights(make_network(fine_cfg), seed=2).to(DEV)
    inp = _render_inputs(cfg, 150, v["M"], v["perturb"], v["stride0"], "aabb", seed=5)
    rc, msg, got = _fused(net.pack(torch.device(DEV)), net_fine.pack(torch.device(DEV)), cfg, inp)
    assert rc == 0, msg
    worst, where = _compare_with_staged(cfg, net, net_fine, inp, got, "distinct fine")
    _report(f"render_fused distinct fine network {mix} {fine_over} [{where}]", worst)


@pytest.mark.parametrize("fine_heads", [(6, 5), (5, 7)])
def test_fine_network_with_other_heads_is_refused(fine_heads):
    """The maps are [R, C] / [R, K] of the coarse network: a fine network with another C or K (even with the same
    4 + C + K) is refused before any launch, with both pairs in the message, and nothing is written."""
    v = dict(_variant(0), buffers="all")
    cfg = _render_cfg(64, 64, "noheads", v, num_classes=5, num_instances=6)
    net = S.init_network_weights(make_network(cfg), seed=1).to(DEV)
    fine_cfg = _with(cfg, num_classes=fine_heads[0], num_instances=fine_heads[1])
    fine = S.init_network_weights(make_network(fine_cfg), seed=2).to(DEV)
    inp = _render_inputs(cfg, 50, v["M"], 0.0, False, "fill", seed=3)
    rc, msg, got = _fused(net.pack(torch.device(DEV)), fine.pack(torch.device(DEV)), cfg, inp)
    assert rc == -1, (rc, msg)
    assert f"(C={fine_heads[0]}, K={fine_heads[1]})" in msg and "(C=5, K=6)" in msg, msg
    for k, t in got.items():
        assert bool((t == SENT[t.dtype]).all()), f"{k} was written"


def test_render_fused_with_no_rays_writes_nothing():
    v = dict(_variant(0), buffers="all")
    cfg = _render_cfg(64, 192, "heads", v)
    net = S.init_network_weights(make_network(cfg), seed=1).to(DEV)
    inp = _render_inputs(cfg, 4, v["M"], 1.0, False, "arrays", seed=3)
    rc, msg, got = _fused(net.pack(torch.device(DEV)), None, cfg, inp, R=0, ws_bytes=1)
    assert rc == 0, msg
    assert all(t.shape[0] == 0 for t in got.values())       # and the PAD rows after them are intact (_fused checks)


@pytest.mark.parametrize("preset,over,chunk", [
    ("cfg3", {}, 65537), ("cfg3", {}, 262144), ("cfg3", dict(sem_activation="softmax"), 600000),
    ("cfg2", {}, 262144), ("cfg3", dict(N_samples=48, N_importance=80), 70000)],
    ids=["cfg3-65537", "cfg3-262144", "cfg3-softmax-600000", "cfg2-262144", "cfg3-N48-Ni80-70000"])
def test_renderer_gpu_chunk_workspace_is_rays_times_bytes_per_ray(preset, over, chunk):
    """Renderer with gpu_chunk rays per chunk past 2^16: the workspace is chunk x the bytes per ray of the layout
    pnr_workspace_bytes sizes (its exact slope where it is proportional to R), not chunk x pnr_workspace_bytes(1), which
    for a network with heads is a softmax ray with raw (cfg3: 91 KB against 2.9 KB).  It still holds the softmax rays
    pnr_workspace_bytes(2^16) holds, and renders (cfg3 N = 48: the coarse pass keeps raw, 21 KB per ray)."""
    cfg = make_cfg(preset, gpu_chunk=chunk, **over)
    net = S.init_network_weights(make_network(cfg), seed=1).to(DEV)
    ctx = net.pack(torch.device(DEV))
    N, Ni = cfg.N_samples, cfg.N_importance
    ws = lambda r: int(_capi.lib().pnr_workspace_bytes(ctx, r, N, Ni))
    # bytes per ray of the sized layout: at 2^13 rays it is proportional to R for these networks (past the softmax rays,
    # below the chunk size of cfg3 N = 48, 27 k rays)
    assert ws(1 << 14) == 2 * ws(1 << 13)
    per_ray = ws(1 << 13) >> 13
    want = make_renderer(cfg, net)._workspace(ctx, chunk, N, Ni, torch.device(DEV)).numel()
    print(f"{preset} {over} gpu_chunk={chunk}: workspace {want} B = {want / chunk:.1f} B per ray "
          f"(layout {per_ray} B per ray, pnr_workspace_bytes(1) = {ws(1)} B)")
    assert ws(1 << 16) <= want and chunk * per_ray <= want <= max(chunk * per_ray + 12 * 256, ws(1 << 16))
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, rows=2).items()}
    out = make_renderer(cfg, net).render(batch)
    assert bool(torch.isfinite(out["rgb_map"]).all())


def _cfg3(softmax, v):
    return make_cfg("cfg3", max_hits=v["M"], sem_activation="softmax" if softmax else "none",
                    mask_outside=v["mask"], white_bkgd=v["white"])


@pytest.mark.parametrize("softmax", [False, True], ids=["logits", "softmax"])
def test_default_workspace_renders_every_call(softmax):
    """pnr_workspace_bytes(ctx, R, N, Ni) must hold at least one ray of every call of R rays it may be handed.  The call
    with no optional buffer, M = 8 and primitives needs the most bytes per ray; a softmax call of a network with heads
    runs both passes on the two-kernel path, which needs raw (cfg3: 87 KB per ray).  Each size renders, equal bit for
    bit to the same call in one chunk."""
    v = dict(_variant(0), M=8, perturb=1.0, stride0=False)
    cfg = _cfg3(softmax, v)
    net = S.init_network_weights(make_network(cfg), seed=4).to(DEV)
    ctx = net.pack(torch.device(DEV))
    big = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    for R in (1, 7, 29, 30, 1000):
        ws = int(_capi.lib().pnr_workspace_bytes(ctx, R, cfg.N_samples, cfg.N_importance))
        print(f"cfg3 {'softmax' if softmax else 'logits'}: pnr_workspace_bytes(R={R}) = {ws} B")
        inp = _render_inputs(cfg, R, v["M"], v["perturb"], v["stride0"], "aabb", seed=R)
        rc, msg, got = _fused(ctx, None, cfg, inp, "none", ws_bytes=ws)
        assert rc == 0, f"R={R}: {msg}"
        rc, msg, one = _fused(ctx, None, cfg, inp, "none", ws_bytes=big.numel(), ws=big)
        assert rc == 0, msg
        for k in one:
            _bits_equal(got[k], one[k], f"R={R} {k}")
    assert net.range_status() == 0


@pytest.mark.parametrize("softmax", [False, True], ids=["logits", "softmax"])
def test_smallest_workspace_and_chunkings_are_bit_identical(softmax):
    """The smallest accepted workspace, found by bisection on the refusal (host-side, before any launch): one byte less
    is refused with PNR_ERR_ARG and "cannot hold one ray".  Rendering at that size (one ray per chunk) and at sizes of
    2, R - 1 and R rays per chunk gives the same outputs bit for bit, with jittered per-ray depths and fine samples."""
    v = dict(_variant(0), M=8, perturb=1.0, stride0=False)
    cfg = _cfg3(softmax, v)
    net = S.init_network_weights(make_network(cfg), seed=4).to(DEV)
    ctx = net.pack(torch.device(DEV))
    R, N, Ni = 29, cfg.N_samples, cfg.N_importance
    inp = _render_inputs(cfg, R, v["M"], v["perturb"], v["stride0"], "arrays", seed=6)
    hi = int(_capi.lib().pnr_workspace_bytes(ctx, 1, N, Ni))
    ws = torch.empty(max(hi, R * 100_000) + 8192, dtype=torch.uint8, device=DEV)
    lo = 1
    rc, msg, _ = _fused(ctx, None, cfg, inp, "none", R=1, ws_bytes=lo, ws=ws)
    assert rc == -1 and "cannot hold one ray" in msg, msg
    while hi - lo > 1:                      # lo refused, hi accepted
        mid = (lo + hi) // 2
        rc, msg, _ = _fused(ctx, None, cfg, inp, "none", R=1, ws_bytes=mid, ws=ws)
        assert rc in (0, -1) and (rc == 0 or "cannot hold one ray" in msg), msg
        lo, hi = (lo, mid) if rc == 0 else (mid, hi)
    rc, msg, _ = _fused(ctx, None, cfg, inp, "none", R=R, ws_bytes=hi - 1, ws=ws)
    assert rc == -1 and "cannot hold one ray" in msg, msg
    per_ray = int(re.search(r"\((\d+) bytes per ray\)", msg).group(1))
    print(f"cfg3 {'softmax' if softmax else 'logits'}, no optional buffer: smallest workspace {hi} B, {per_ray} B per ray")
    # k rays per chunk: chunk_bytes(k) <= k * per_ray + the alignment of <= 12 sub-buffers < (k + 1) * per_ray
    runs = {}
    for k in (1, 2, R - 1, R):
        size = hi if k == 1 else k * per_ray + 12 * 256
        rc, msg, runs[k] = _fused(ctx, None, cfg, inp, "none", ws_bytes=size, ws=ws)
        assert rc == 0, f"{k} rays per chunk: {msg}"
    for k in (2, R - 1, R):
        for name in runs[1]:
            _bits_equal(runs[k][name], runs[1][name], f"{k} rays per chunk: {name}")
    assert net.range_status() == 0
