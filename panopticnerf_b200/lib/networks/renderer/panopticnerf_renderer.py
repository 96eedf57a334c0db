"""Renderer / raw2outputs / sample_pdf — the volume-render loop of PanopticNeRF (SURVEY.md 8(a)
a3, a4, a5, a6, a9, a10; reference: the Renderer module under lib/networks/renderer/ and its
raw2outputs / sample_pdf helpers, not in the mount).

Same names, argument meaning and returned keys as the oracle restatement (oracle/reference_renderer.py),
but every stage is a libpnr CUDA kernel called through the C ABI; torch only owns the device buffers.
CPU tensors raise: there is no CPU path in the product.
"""
from __future__ import annotations

import ctypes as C
import functools
from typing import Dict, List, Optional

import torch

from panopticnerf_b200 import _capi

_F32, _I32 = torch.float32, torch.int32
MAX_SAMPLES_PER_RAY = 256      # pnr_composite: 32 lanes x 8 samples


def _f(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _capi.PnrError(f"{name}: expected a CUDA tensor, got {t.device} (panopticnerf_b200 is GPU-only)")
    return t.to(_F32).contiguous()


def _on_tensor_device(fn):
    """Run a stage wrapper with the device of its first tensor argument current: the stream handed to libpnr
    (torch's current stream) and the kernels it launches then belong to the device the buffers live on, whatever
    the caller's current device is (several GPUs driven from one process)."""
    @functools.wraps(fn)
    def wrapper(*args, **kw):
        t = next((a for a in args if torch.is_tensor(a)), None)
        if t is None or not t.is_cuda:
            return fn(*args, **kw)          # the wrapper's own checks raise the "GPU-only" error
        with torch.cuda.device(t.device):
            return fn(*args, **kw)
    return wrapper


# ------------------------------------------------------------------------------------------------
# what every compositing call (pnr_composite, pnr_composite_backward, pnr_mlp_composite, pnr_render_fused) shares
# ------------------------------------------------------------------------------------------------
def composite_map_keys(C: int, K: int, fixed_sem: bool, fixed_inst: bool) -> List[str]:
    """The maps a compositing call produces, in the order it returns them: rgb / depth / acc / disp / weights always,
    semantic_map if C > 0, instance_map if K > 0, and a fixed (bounding-box) map when it is wanted (per-sample
    primitive ids and that id table given) and its head exists."""
    keys = ["rgb_map", "depth_map", "acc_map", "disp_map", "weights"]
    if C > 0:
        keys.append("semantic_map")
    if K > 0:
        keys.append("instance_map")
    if fixed_sem and C > 0:
        keys.append("fixed_semantic_map")
    if fixed_inst and K > 0:
        keys.append("fixed_instance_map")
    return keys


def _map_shapes(R: int, n: int, C: int, K: int) -> Dict[str, tuple]:
    return {"rgb_map": (R, 3), "depth_map": (R,), "acc_map": (R,), "disp_map": (R,), "weights": (R, n),
            "semantic_map": (R, C), "instance_map": (R, K), "fixed_semantic_map": (R, C), "fixed_instance_map": (R, K)}


def empty_composite_maps(R: int, n: int, C: int, K: int, fixed_sem: bool, fixed_inst: bool,
                         device) -> Dict[str, torch.Tensor]:
    """Uninitialised float32 maps of `composite_map_keys` for R rays of n samples on `device`."""
    shapes = _map_shapes(R, n, C, K)
    return {k: torch.empty(shapes[k], dtype=_F32, device=device) for k in composite_map_keys(C, K, fixed_sem, fixed_inst)}


def primitive_tables(ref: torch.Tensor, sample_box, box_sem, box_inst):
    """(sample_box, box_sem, box_inst, B) as the compositing kernels take them: each table int32 and contiguous (None
    stays None) and B, the one bound of both id tables, which sample_box indexes (0 without sample_box).  The tables
    must live on ref's device and, with sample_box, the id tables must have the same length."""
    for name, t in (("sample_box", sample_box), ("box_sem", box_sem), ("box_inst", box_inst)):
        if t is not None and t.device != ref.device:
            raise _capi.PnrError(f"{name} is on {t.device}, expected {ref.device}")
    B = 0
    if sample_box is not None:
        sizes = {int(t.shape[0]) for t in (box_sem, box_inst) if t is not None}
        if len(sizes) > 1:
            raise ValueError(f"box_sem and box_inst must have one entry per primitive each, got lengths {sorted(sizes)}")
        B = sizes.pop() if sizes else 0
    sb, bs, bi = (t.to(_I32).contiguous() if t is not None else None for t in (sample_box, box_sem, box_inst))
    return sb, bs, bi, B


def _rays(rays_d: torch.Tensor) -> torch.Tensor:
    """rays [R,6] for the compositing kernels, which read only the directions: rays_d [R,3] gets zero origins."""
    return _f(torch.cat([torch.zeros_like(rays_d), rays_d], -1) if rays_d.shape[-1] == 3 else rays_d, "rays")


# ------------------------------------------------------------------------------------------------
# stage wrappers (one libpnr call each)
# ------------------------------------------------------------------------------------------------
@_on_tensor_device
def intersect(rays, box_center, box_half, box_rot, max_hits: int, mesh_tri_start=None, mesh_tris=None,
              ray_frame=None, frame_boxes=None, static_boxes=None):
    """a5 -> hit_mask [R] bool, box_id [R,M] i32, t_in, t_out [R,M].  With a mesh table (mesh_tri_start [B+1] int32,
    mesh_tris [T,3,3]) the primitives that own triangles are closed meshes culled by their box (DESIGN 3.2).  With a
    sequence table (ray_frame [R] int, frame_boxes [F,2] int, static_boxes S: kitti360.sequence_primitives) ray r meets
    the primitives [0, S) and its frame's block frame_boxes[ray_frame[r]] (include/pnr.h pnr_intersect_frames)."""
    rays = _f(rays, "rays")
    R, B, M = rays.shape[0], box_center.shape[0], int(max_hits)
    dev = rays.device
    hit = torch.empty(R, dtype=torch.uint8, device=dev)
    box_id = torch.empty(R, M, dtype=_I32, device=dev)
    t_in = torch.empty(R, M, dtype=_F32, device=dev)
    t_out = torch.empty(R, M, dtype=_F32, device=dev)
    bc, bh, br = _f(box_center, "box_center"), _f(box_half, "box_half"), _f(box_rot, "box_rot")
    mesh = mesh_tri_start is not None or mesh_tris is not None
    starts, tris = _mesh_table(mesh_tri_start, mesh_tris, B, dev) if mesh else (None, None)
    frames = _frame_table(ray_frame, frame_boxes, static_boxes, R, dev)
    if frames is not None:
        a = _capi.PnrIntersectFramesArgs(rays=_capi.ptr(rays), R=R, box_center=_capi.ptr(bc), box_half=_capi.ptr(bh),
                                         box_rot=_capi.ptr(br), B=B, M=M, mesh_tri_start=_capi.ptr(starts),
                                         mesh_tris=_capi.ptr(tris), T=tris.shape[0] if mesh else 0,
                                         frames=frames[0], hit_mask=_capi.ptr(hit), box_id=_capi.ptr(box_id),
                                         t_in=_capi.ptr(t_in), t_out=_capi.ptr(t_out))
        _capi.check(_capi.lib().pnr_intersect_frames(C.byref(a), _capi.stream_ptr()), "pnr_intersect_frames")
        return hit.bool(), box_id, t_in, t_out
    if not mesh:
        _capi.check(_capi.lib().pnr_intersect(_capi.ptr(rays), R, _capi.ptr(bc), _capi.ptr(bh), _capi.ptr(br), B, M,
                                              _capi.ptr(hit), _capi.ptr(box_id), _capi.ptr(t_in), _capi.ptr(t_out),
                                              _capi.stream_ptr()), "pnr_intersect")
        return hit.bool(), box_id, t_in, t_out
    _capi.check(_capi.lib().pnr_intersect_meshes(_capi.ptr(rays), R, _capi.ptr(bc), _capi.ptr(bh), _capi.ptr(br),
                                                 _capi.ptr(starts), _capi.ptr(tris), tris.shape[0], B, M,
                                                 _capi.ptr(hit), _capi.ptr(box_id), _capi.ptr(t_in), _capi.ptr(t_out),
                                                 _capi.stream_ptr()), "pnr_intersect_meshes")
    return hit.bool(), box_id, t_in, t_out


def _frame_table(ray_frame, frame_boxes, static_boxes, R: int, device):
    """(PnrFrameTable, tensors it points to) of a sequence table on `device`, or None without one; shapes checked (the
    library checks S against B and clamps the ranges)."""
    given = [x is not None for x in (ray_frame, frame_boxes, static_boxes)]
    if not any(given):
        return None
    if not all(given):
        raise ValueError("a sequence table needs ray_frame, frame_boxes and static_boxes together (ray_frame "
                         f"{'set' if given[0] else 'missing'}, frame_boxes {'set' if given[1] else 'missing'}, "
                         f"static_boxes {'set' if given[2] else 'missing'})")
    rf = ray_frame.to(device=device, dtype=_I32).contiguous()
    fb = frame_boxes.to(device=device, dtype=_I32).contiguous()
    if tuple(rf.shape) != (R,) or fb.dim() != 2 or fb.shape[1] != 2 or fb.shape[0] < 1:
        raise ValueError(f"sequence table: ray_frame {tuple(rf.shape)} (want ({R},)), frame_boxes {tuple(fb.shape)} "
                         "(want (F, 2), F >= 1)")
    t = _capi.PnrFrameTable(ray_frame=_capi.ptr(rf), frame_boxes=_capi.ptr(fb), F=fb.shape[0], S=int(static_boxes))
    return t, (rf, fb)


def _mesh_table(mesh_tri_start, mesh_tris, B: int, device):
    """(mesh_tri_start int32 [B+1], mesh_tris fp32 [T,3,3]) on `device`, shapes checked."""
    if mesh_tri_start is None or mesh_tris is None:
        raise ValueError("mesh_tri_start and mesh_tris come together")
    starts = mesh_tri_start.to(device=device, dtype=_I32).contiguous()
    tris = _f(mesh_tris.to(device), "mesh_tris")
    if tuple(starts.shape) != (B + 1,) or tris.dim() != 3 or tuple(tris.shape[1:]) != (3, 3):
        raise ValueError(f"mesh table: mesh_tri_start {tuple(starts.shape)} (want ({B + 1},)), mesh_tris "
                         f"{tuple(tris.shape)} (want (T, 3, 3))")
    return starts, tris


@_on_tensor_device
def scene_near_far(rays, aabb, near_min: float, far_default: float):
    rays = _f(rays, "rays")
    R = rays.shape[0]
    near = torch.empty(R, dtype=_F32, device=rays.device)
    far = torch.empty(R, dtype=_F32, device=rays.device)
    a = (C.c_float * 6)(*[float(x) for x in aabb.detach().to("cpu", _F32).reshape(-1).tolist()])
    _capi.check(_capi.lib().pnr_scene_near_far(_capi.ptr(rays), R, a, float(near_min), float(far_default),
                                               _capi.ptr(near), _capi.ptr(far), _capi.stream_ptr()),
                "pnr_scene_near_far")
    return near, far


@_on_tensor_device
def bound_by_primitives(hit, box_id, t_in, t_out, near, far):
    hit8 = hit.to(torch.uint8).contiguous()
    near, far = near.clone(), far.clone()
    _capi.check(_capi.lib().pnr_bound_by_primitives(_capi.ptr(hit8), _capi.ptr(box_id, _I32), _capi.ptr(t_in),
                                                    _capi.ptr(t_out), near.shape[0], box_id.shape[1],
                                                    _capi.ptr(near), _capi.ptr(far), _capi.stream_ptr()),
                "pnr_bound_by_primitives")
    return near, far


@_on_tensor_device
def stratified_z(near, far, t_vals, perturb: float = 0.0, u: Optional[torch.Tensor] = None,
                 box_id=None, t_in=None, t_out=None, want_tags: bool = False):
    """a6 -> z [R,N] (and sample_box [R,N] i32 when want_tags)."""
    near, far, t_vals = _f(near, "near"), _f(far, "far"), _f(t_vals, "t_vals")
    R, N = near.shape[0], t_vals.shape[0]
    if perturb > 0.0 and u is None:
        u = torch.rand(R, N, device=near.device, dtype=_F32)
    u = _f(u, "u") if (u is not None and perturb > 0.0) else None
    z = torch.empty(R, N, dtype=_F32, device=near.device)
    sb = torch.empty(R, N, dtype=_I32, device=near.device) if want_tags else None
    M = box_id.shape[1] if box_id is not None else 0
    _capi.check(_capi.lib().pnr_sample_stratified(
        _capi.ptr(near), _capi.ptr(far), _capi.ptr(t_vals), _capi.ptr(u), R, N, float(perturb),
        _capi.ptr(box_id, _I32) if box_id is not None else None, _capi.ptr(t_in), _capi.ptr(t_out), M,
        _capi.ptr(z), _capi.ptr(sb), _capi.stream_ptr()), "pnr_sample_stratified")
    return (z, sb) if want_tags else z


@_on_tensor_device
def interval_z(near, far, t_vals, box_id, t_in, t_out, perturb: float = 0.0, u: Optional[torch.Tensor] = None):
    """a6 interval mode -> (z [R,N] ascending, sample_box [R,N] i32): the N samples sit inside the ray's hit
    intervals (n_m ~ N * len_m / sum len, remainder to the nearest; rays without a hit use the uniform rule)."""
    near, far, t_vals = _f(near, "near"), _f(far, "far"), _f(t_vals, "t_vals")
    R, N = near.shape[0], t_vals.shape[0]
    if perturb > 0.0 and u is None:
        u = torch.rand(R, N, device=near.device, dtype=_F32)
    u = _f(u, "u") if (u is not None and perturb > 0.0) else None
    z = torch.empty(R, N, dtype=_F32, device=near.device)
    sb = torch.empty(R, N, dtype=_I32, device=near.device)
    _capi.check(_capi.lib().pnr_sample_intervals(
        _capi.ptr(near), _capi.ptr(far), _capi.ptr(t_vals), _capi.ptr(u), R, N, float(perturb),
        _capi.ptr(box_id, _I32), _capi.ptr(t_in), _capi.ptr(t_out), box_id.shape[1], _capi.ptr(z), _capi.ptr(sb),
        _capi.stream_ptr()), "pnr_sample_intervals")
    return z, sb


@_on_tensor_device
def tag_samples(z, box_id, t_in, t_out):
    z = _f(z, "z")
    sb = torch.empty(z.shape, dtype=_I32, device=z.device)
    _capi.check(_capi.lib().pnr_tag_samples(_capi.ptr(z), z.shape[0], z.shape[1], _capi.ptr(box_id, _I32),
                                            _capi.ptr(t_in), _capi.ptr(t_out), box_id.shape[1], _capi.ptr(sb),
                                            _capi.stream_ptr()), "pnr_tag_samples")
    return sb


def generate_rays(H: int, W: int, intr, c2w: torch.Tensor, camera: str = "pinhole", row0: int = 0,
                  rows: Optional[int] = None, device="cuda") -> torch.Tensor:
    """Camera rays on the device (SURVEY 8(f) rank 3): only 16 floats cross the host/device boundary."""
    rows = H - row0 if rows is None else rows
    rays = torch.empty(rows * W, 6, dtype=_F32, device=device)
    cam = {"pinhole": 0, "equirect": 1, "fisheye": 2}[camera]
    vals = [float(x) for x in intr]
    if len(vals) != (7 if cam == 2 else 4):
        raise ValueError(f"generate_rays: camera '{camera}' takes {7 if cam == 2 else 4} intrinsics, got {len(vals)}")
    k = (C.c_float * len(vals))(*vals)
    m = (C.c_float * 12)(*[float(x) for x in c2w.detach().to("cpu", _F32).reshape(-1)[:12].tolist()])
    with torch.cuda.device(rays.device):
        _capi.check(_capi.lib().pnr_generate_rays(int(H), int(W), int(row0), int(rows), cam,
                                                  k, m, _capi.ptr(rays), _capi.stream_ptr()), "pnr_generate_rays")
    return rays


@_on_tensor_device
def embed(x: torch.Tensor, L: int) -> torch.Tensor:
    """a7 standalone positional encoding (the Renderer uses the copy fused into the MLP kernel)."""
    xf = _f(x.reshape(-1, 3), "x")
    out = torch.empty(xf.shape[0], 3 + 6 * L, dtype=_F32, device=xf.device)
    _capi.check(_capi.lib().pnr_encode(_capi.ptr(xf), xf.shape[0], int(L), _capi.ptr(out), _capi.stream_ptr()),
                "pnr_encode")
    return out.reshape(*x.shape[:-1], 3 + 6 * L)


@_on_tensor_device
def raw2outputs(raw, z_vals, rays_d, raw_noise_std: float = 0.0, white_bkgd: bool = False,
                num_classes: int = 0, num_instances: int = 0, sem_activation: str = "none",
                sample_box: Optional[torch.Tensor] = None, box_sem: Optional[torch.Tensor] = None,
                box_inst: Optional[torch.Tensor] = None, mask_outside: bool = False,
                noise: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """a9.  raw [R,N,4+C+K], z_vals [R,N], rays_d [R,3] (or rays [R,6])."""
    raw, z_vals = _f(raw, "raw"), _f(z_vals, "z_vals")
    R, N = z_vals.shape
    Cn, Kn = int(num_classes), int(num_instances)
    if raw.shape[-1] != 4 + Cn + Kn:
        raise ValueError(f"raw2outputs: raw has {raw.shape[-1]} channels, expected {4 + Cn + Kn}")
    if raw_noise_std > 0.0:
        nz = noise if noise is not None else torch.randn(R, N, device=raw.device)
        raw = raw.clone()
        raw[..., 3] += nz.to(raw.device, _F32) * raw_noise_std
    rays = _rays(rays_d)
    sb, bs, bi, B = primitive_tables(raw, sample_box, box_sem, box_inst)
    out = empty_composite_maps(R, N, Cn, Kn, sb is not None and bs is not None, sb is not None and bi is not None,
                               raw.device)
    _capi.check(_capi.lib().pnr_composite(
        _capi.ptr(raw), _capi.ptr(z_vals), _capi.ptr(rays), R, N, Cn, Kn, int(bool(white_bkgd)),
        int(sem_activation == "softmax"), int(bool(mask_outside)), _capi.ptr(sb), _capi.ptr(bs), _capi.ptr(bi),
        B, C.byref(_capi.ptr_struct(_capi.PnrCompositeOut, out)), _capi.stream_ptr()), "pnr_composite")
    return out


@_on_tensor_device
def raw2outputs_backward(raw, z_vals, rays_d, grads: Dict[str, torch.Tensor], white_bkgd: bool = False,
                         num_classes: int = 0, num_instances: int = 0, sem_activation: str = "none",
                         sample_box: Optional[torch.Tensor] = None, box_sem: Optional[torch.Tensor] = None,
                         box_inst: Optional[torch.Tensor] = None, mask_outside: bool = False) -> torch.Tensor:
    """Gradient of a scalar loss with respect to `raw` [R,N,4+C+K], given its gradients with respect to the maps
    `raw2outputs` returns (`grads`: any subset of rgb_map, depth_map, acc_map, weights, semantic_map,
    instance_map, fixed_semantic_map, fixed_instance_map; `disp_map` is not differentiated).  First stage of
    the backward chain of the render path (SURVEY 8(f) rank 2); checked against autograd through the oracle."""
    raw, z_vals = _f(raw, "raw"), _f(z_vals, "z_vals")
    R, N = z_vals.shape
    Cn, Kn = int(num_classes), int(num_instances)
    if raw.shape[-1] != 4 + Cn + Kn:
        raise ValueError(f"raw2outputs_backward: raw has {raw.shape[-1]} channels, expected {4 + Cn + Kn}")
    if "disp_map" in grads:
        raise ValueError("raw2outputs_backward: disp_map is not differentiated")
    rays = _rays(rays_d)
    shapes = _map_shapes(R, N, Cn, Kn)
    held = {}
    for k, g in grads.items():
        if k not in shapes:
            raise ValueError(f"raw2outputs_backward: unknown map {k!r}")
        if g is None:
            continue
        g = _f(g, k)
        if tuple(g.shape) != shapes[k]:
            raise ValueError(f"raw2outputs_backward: grad of {k} has shape {tuple(g.shape)}, expected {shapes[k]}")
        held[k] = g
    sb, bs, bi, B = primitive_tables(raw, sample_box, box_sem, box_inst)
    d_raw = torch.empty_like(raw)
    _capi.check(_capi.lib().pnr_composite_backward(
        _capi.ptr(raw), _capi.ptr(z_vals), _capi.ptr(rays), R, N, Cn, Kn, int(bool(white_bkgd)),
        int(sem_activation == "softmax"), int(bool(mask_outside)), _capi.ptr(sb), _capi.ptr(bs), _capi.ptr(bi),
        B, C.byref(_capi.ptr_struct(_capi.PnrCompositeGrads, held)), _capi.ptr(d_raw), _capi.stream_ptr()),
        "pnr_composite_backward")
    return d_raw


class _Raw2OutputsFn(torch.autograd.Function):
    """`raw2outputs` as an autograd node: losses written in torch on the composited maps back-propagate to `raw`
    through `pnr_composite_backward`.  The maps are returned in the order of `composite_map_keys`, disp_map last."""

    @staticmethod
    def forward(ctx, raw, z_vals, rays_d, kw):
        out = raw2outputs(raw.detach(), z_vals, rays_d, **kw)
        ctx.save_for_backward(raw.detach(), z_vals, rays_d)
        ctx.kw = kw
        ctx.present = [k for k in out if k != "disp_map"]
        ctx.mark_non_differentiable(out["disp_map"])
        return tuple(out[k] for k in ctx.present) + (out["disp_map"],)

    @staticmethod
    def backward(ctx, *gs):
        raw, z_vals, rays_d = ctx.saved_tensors
        grads = {k: g for k, g in zip(ctx.present, gs[:-1]) if g is not None}
        return raw2outputs_backward(raw, z_vals, rays_d, grads, **ctx.kw), None, None, None


def raw2outputs_autograd(raw, z_vals, rays_d, white_bkgd: bool = False, num_classes: int = 0,
                         num_instances: int = 0, sem_activation: str = "none",
                         sample_box: Optional[torch.Tensor] = None, box_sem: Optional[torch.Tensor] = None,
                         box_inst: Optional[torch.Tensor] = None, mask_outside: bool = False) -> Dict[str, torch.Tensor]:
    """`raw2outputs` whose outputs carry gradients back to `raw` (z_vals and rays are treated as constants, as in
    the reference's training step where the sampler is not differentiated)."""
    kw = dict(white_bkgd=white_bkgd, num_classes=num_classes, num_instances=num_instances,
              sem_activation=sem_activation, sample_box=sample_box, box_sem=box_sem, box_inst=box_inst,
              mask_outside=mask_outside)
    res = _Raw2OutputsFn.apply(raw, z_vals, rays_d, kw)
    fixed = [sample_box is not None and t is not None for t in (box_sem, box_inst)]
    present = [k for k in composite_map_keys(int(num_classes), int(num_instances), *fixed) if k != "disp_map"]
    out = dict(zip(present, res[:-1]))
    out["disp_map"] = res[-1]
    return out


@_on_tensor_device
def sample_pdf(z, weights, N_importance: int, det: bool = True, u: Optional[torch.Tensor] = None,
               want_idx: bool = False):
    """a10 on coarse depths z [R,N] and coarse weights [R,N] (bins = mid points, pdf = weights[1:-1]).
    Returns (z_fine [R,Ni], z_all [R,N+Ni] sorted[, idx [R,Ni] i64])."""
    z, weights = _f(z, "z"), _f(weights, "weights")
    R, N = z.shape
    Ni = int(N_importance)
    if u is None:
        if det:
            u = torch.linspace(0.0, 1.0, Ni).to(z.device)[None].expand(R, Ni)   # host linspace = oracle's
        else:
            u = torch.rand(R, Ni, device=z.device)
    u = _f(u, "u")
    z_f = torch.empty(R, Ni, dtype=_F32, device=z.device)
    z_all = torch.empty(R, N + Ni, dtype=_F32, device=z.device)
    idx = torch.empty(R, Ni, dtype=torch.int64, device=z.device) if want_idx else None
    _capi.check(_capi.lib().pnr_sample_pdf(_capi.ptr(z), _capi.ptr(weights), R, N, Ni, _capi.ptr(u),
                                           _capi.ptr(z_f), _capi.ptr(idx), _capi.ptr(z_all), _capi.stream_ptr()),
                "pnr_sample_pdf")
    return (z_f, z_all, idx) if want_idx else (z_f, z_all)


# ------------------------------------------------------------------------------------------------
# Renderer
# ------------------------------------------------------------------------------------------------
class Renderer:
    """Renderer(cfg, net).render(batch) -> dict of per-ray maps (a3).  batch keys: rays [R,6] (o||d),
    optional near/far [R], scene_aabb [2,3], box_center/box_half [B,3], box_rot [B,3,3], box_sem/box_inst [B],
    mesh_tri_start [B+1] int32 / mesh_tris [T,3,3] (mesh primitives: include/pnr.h pnr_intersect_meshes),
    ray_frame [R] / frame_boxes [F,2] / static_boxes (a sequence table: include/pnr.h pnr_intersect_frames),
    u [R,N] / u_fine [R,Ni] (externally supplied jitter), perturb."""

    def __init__(self, cfg, net, net_fine=None):
        self.cfg, self.net = cfg, net
        self.net_fine = net_fine if net_fine is not None else net
        self._t_vals = {}
        self._ws = {}                 # pnr_render_fused scratch, one buffer per device
        N, Ni = int(cfg.N_samples), int(getattr(cfg, "N_importance", 0))
        if N < 1 or N + Ni > MAX_SAMPLES_PER_RAY:
            raise ValueError(f"Renderer: N_samples + N_importance = {N} + {Ni} exceeds the {MAX_SAMPLES_PER_RAY} samples "
                             "per ray the compositing kernel handles")

    def _tv(self, N: int, device) -> torch.Tensor:
        key = (N, str(device))
        if key not in self._t_vals:
            self._t_vals[key] = torch.linspace(0.0, 1.0, N).to(device)   # CPU linspace, as the oracle's
        return self._t_vals[key]

    def _auto_chunk(self, rays) -> int:
        """Largest ray chunk whose intermediates (raw is the big one: N x (4+C+K) floats per ray, coarse + fine)
        fit in half of the free device memory; usually the whole frame (results do not depend on it)."""
        cfg = self.cfg
        N, Ni = int(cfg.N_samples), int(getattr(cfg, "N_importance", 0))
        ch = 4 + int(getattr(cfg, "num_classes", 0)) + int(getattr(cfg, "num_instances", 0))
        per_ray = 4 * ((N + (N + Ni if Ni else 0)) * (ch + 4) + 64)
        free, _ = torch.cuda.mem_get_info(rays.device)
        chunk = max(1024, int(0.5 * free // per_ray) // 1024 * 1024)
        return min(rays.shape[0], chunk)

    # -- a4: results are invariant to `chunk`; None renders every ray in one pass of persistent kernels
    def batchify_rays(self, rays, near, far, batch, chunk: Optional[int] = None):
        R = rays.shape[0]
        chunk = int(chunk) if chunk else R
        if chunk >= R:
            return self.render_rays(rays, near, far, batch, slice(0, R))
        outs = []
        for i in range(0, R, chunk):
            sl = slice(i, min(i + chunk, R))
            outs.append(self.render_rays(rays[sl].contiguous(), near[sl].contiguous(), far[sl].contiguous(),
                                         batch, sl))
        return {k: torch.cat([o[k] for o in outs], 0) for k in outs[0]}

    def render_rays(self, rays, near, far, batch, sl, grad: bool = False):
        """Both passes for the rays `sl` of the batch.  grad=True: the maps carry gradients to the parameters of both
        networks (network_forward_rays_autograd + raw2outputs_autograd); the sampler is not differentiated (the fine
        pass reads the coarse weights detached), and cfg.raw_noise_std adds noise to sigma before compositing."""
        cfg = self.cfg
        N, Ni = int(cfg.N_samples), int(getattr(cfg, "N_importance", 0))
        Cn, Kn = int(getattr(cfg, "num_classes", 0)), int(getattr(cfg, "num_instances", 0))
        M = int(getattr(cfg, "max_hits", 4))
        perturb = float(batch.get("perturb", getattr(cfg, "perturb", 0.0)))
        out = {}
        has_boxes = "box_center" in batch and batch["box_center"].shape[0] > 0
        box_id = t_in = t_out = None
        if has_boxes:
            rf = batch["ray_frame"][sl] if batch.get("ray_frame") is not None else None
            hit, box_id, t_in, t_out = intersect(rays, batch["box_center"], batch["box_half"],
                                                 batch["box_rot"], M, batch.get("mesh_tri_start"), batch.get("mesh_tris"),
                                                 rf, batch.get("frame_boxes"), batch.get("static_boxes"))
            out.update(hit_mask=hit, box_id=box_id, t_in=t_in, t_out=t_out)
            if bool(getattr(cfg, "bound_by_primitives", False)):
                near, far = bound_by_primitives(hit, box_id, t_in, t_out, near, far)
        u = batch["u"][sl] if "u" in batch else None
        if has_boxes and str(getattr(cfg, "sample_mode", "uniform")) == "intervals":
            z, sb = interval_z(near, far, self._tv(N, rays.device), box_id, t_in, t_out, perturb, u)
        else:
            res = stratified_z(near, far, self._tv(N, rays.device), perturb, u, box_id, t_in, t_out,
                               want_tags=has_boxes)
            z, sb = res if has_boxes else (res, None)
        kw = dict(white_bkgd=bool(getattr(cfg, "white_bkgd", False)), num_classes=Cn, num_instances=Kn,
                  sem_activation=str(getattr(cfg, "sem_activation", "none")),
                  mask_outside=bool(getattr(cfg, "mask_outside", False)))
        if has_boxes:
            kw.update(box_sem=batch.get("box_sem"), box_inst=batch.get("box_inst"))
        raw, res = self._pass(self.net, rays, z, sb, kw, batch.get("noise"), sl, grad)
        if Ni > 0:
            for k, v in res.items():
                out[k + "_0"] = v
            out["z_vals_0"] = z
            u_f = batch["u_fine"][sl] if "u_fine" in batch else None
            _, z = sample_pdf(z, res["weights"].detach(), Ni, det=(perturb == 0.0), u=u_f)
            sb = tag_samples(z, box_id, t_in, t_out) if has_boxes else None
            raw, res = self._pass(self.net_fine, rays, z, sb, kw, batch.get("noise_fine"), sl, grad)
        out.update(res)
        out["z_vals"] = z
        if sb is not None:
            out["sample_box"] = sb
        if bool(getattr(cfg, "return_raw", False)):
            out["raw"] = raw
        return out

    def _pass(self, net, rays, z, sb, kw, noise, sl, grad: bool):
        """raw and the composited maps of one pass over the depths z."""
        if not grad:
            raw = net.forward_rays(rays, z)
            return raw, raw2outputs(raw, z, rays, sample_box=sb, **kw)
        from ...train.mlp_backward import network_forward_rays_autograd
        raw = network_forward_rays_autograd(net, rays, z)
        std = float(getattr(self.cfg, "raw_noise_std", 0.0))
        if std > 0.0:
            nz = noise[sl] if noise is not None else torch.randn(z.shape, device=z.device)
            raw = torch.cat([raw[..., :3], raw[..., 3:4] + _f(nz, "noise")[..., None] * std, raw[..., 4:]], -1)
        return raw, raw2outputs_autograd(raw, z, rays, sample_box=sb, **kw)

    def _rays_near_far(self, batch):
        cfg = self.cfg
        if "rays" not in batch and "c2w" in batch:     # camera given instead of rays: generate them on the device
            dev = next(self.net.parameters()).device
            batch = dict(batch)
            batch["rays"] = generate_rays(int(cfg.H), int(cfg.W_img), batch.get("intrinsics", (cfg.fx, cfg.fy, cfg.cx, cfg.cy)),
                                          batch["c2w"], getattr(cfg, "camera", "pinhole"),
                                          int(batch.get("row0", 0)), batch.get("rows"), dev)
        rays = _f(batch["rays"], "batch['rays']")
        if "near" in batch and "far" in batch:
            near, far = _f(batch["near"], "near"), _f(batch["far"], "far")
        elif "scene_aabb" in batch:
            near, far = scene_near_far(rays, batch["scene_aabb"], float(cfg.near), float(cfg.far))
        else:
            near = torch.full((rays.shape[0],), float(cfg.near), dtype=_F32, device=rays.device)
            far = torch.full((rays.shape[0],), float(cfg.far), dtype=_F32, device=rays.device)
        return rays, near, far

    def _check_range(self):
        if bool(getattr(self.cfg, "check_range", True)):
            self.net.check_range()
            if self.net_fine is not self.net:
                self.net_fine.check_range()

    # -- a3
    @torch.no_grad()
    def render(self, batch: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        cfg = self.cfg
        rays, near, far = self._rays_near_far(batch)
        staged = str(getattr(cfg, "render_path", "fused")) == "staged" or bool(getattr(cfg, "return_raw", False))
        with torch.cuda.device(rays.device):
            if staged:     # stage by stage from Python (one libpnr call per stage and chunk; keeps `raw`)
                chunk = getattr(cfg, "gpu_chunk", None) or self._auto_chunk(rays)
                out = self.batchify_rays(rays, near, far, batch, chunk)
                out["near"], out["far"] = near, far
            else:          # the whole frame in ONE libpnr call (pnr_render_fused), chunked inside by the workspace
                out = self.render_fused(rays, near, far, batch)
            self._check_range()
        return out

    def render_train(self, batch: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """The staged render of a training batch (all its rays in one pass) whose maps carry gradients back to the
        parameters of both networks: the same keys as `render` with render_path "staged" (coarse maps with the
        suffix _0, z_vals, sample_box and the fixed maps when box_inst / box_sem are given).  Jitter from batch u /
        u_fine when given; with cfg.raw_noise_std > 0, batch noise [R,N] / noise_fine [R,N+Ni] (else torch.randn)
        times the std is added to sigma before compositing."""
        rays, near, far = self._rays_near_far(batch)
        with torch.cuda.device(rays.device):
            out = self.render_rays(rays, near, far, batch, slice(0, rays.shape[0]), grad=True)
            out["near"], out["far"] = near, far
            self._check_range()
        return out

    # -- a3/a4 through the single C-ABI entry point
    def _workspace(self, ctx, R: int, N: int, Ni: int, device) -> torch.Tensor:
        want = int(getattr(self.cfg, "workspace_mb", 0)) << 20
        chunk = int(getattr(self.cfg, "gpu_chunk", 0) or 0)
        if want <= 0 and chunk > 0:     # rays per chunk given instead of bytes
            ws = lambda r: int(_capi.lib().pnr_workspace_bytes(ctx, r, N, Ni))
            want = ws(min(chunk, 1 << 16))
            if chunk > 1 << 16:
                # chunk rays of its layout.  pnr_workspace_bytes(R) is exactly R x the bytes per ray of that layout at R
                # a multiple of 256 between the few softmax rays it always holds (< 2^14 rays) and its own chunk size,
                # where it stops growing: find such an R (proportional to R + 256 as well); if there is none, fall back
                # to the bytes of one ray.  Plus the alignment of up to 12 sub-buffers.
                per_ray = ws(1)
                for r in (1 << 14, 1 << 15, 1 << 16, 1 << 17):
                    a, b = ws(r), ws(r + 256)
                    if a * (r + 256) == b * r:
                        per_ray = a // r
                        break
                want = max(want, chunk * per_ray + 12 * 256)
        if want <= 0:
            want = int(_capi.lib().pnr_workspace_bytes(ctx, R, N, Ni))
        ws = self._ws.get(str(device))
        if ws is None or ws.numel() < want:
            ws = torch.empty(want, dtype=torch.uint8, device=device)
            self._ws[str(device)] = ws
        return ws

    def render_fused(self, rays, near, far, batch) -> Dict[str, torch.Tensor]:
        cfg = self.cfg
        dev = rays.device
        R = rays.shape[0]
        N, Ni = int(cfg.N_samples), int(getattr(cfg, "N_importance", 0))
        Nt = N + Ni
        Cn, Kn = int(getattr(cfg, "num_classes", 0)), int(getattr(cfg, "num_instances", 0))
        M = int(getattr(cfg, "max_hits", 4))
        perturb = float(batch.get("perturb", getattr(cfg, "perturb", 0.0)))
        has_boxes = "box_center" in batch and batch["box_center"].shape[0] > 0
        ctx = self.net.pack(dev)
        ctx_fine = self.net_fine.pack(dev) if self.net_fine is not self.net else None
        e = lambda *shape, dtype=_F32: torch.empty(*shape, dtype=dtype, device=dev)
        fixed = [has_boxes and batch.get(k) is not None for k in ("box_sem", "box_inst")]
        final = empty_composite_maps(R, Nt, Cn, Kn, *fixed, dev)
        coarse = empty_composite_maps(R, N, Cn, Kn, *fixed, dev) if Ni > 0 else {}
        keep = [rays, near, far]                      # tensors the call reads: alive until it is enqueued
        a = _capi.PnrRenderArgs()
        a.rays, a.R, a.near, a.far = _capi.ptr(rays), R, _capi.ptr(near), _capi.ptr(far)
        a.near_min, a.far_default = float(cfg.near), float(cfg.far)
        out: Dict[str, torch.Tensor] = {}
        if has_boxes:
            bc, bh, br = _f(batch["box_center"], "box_center"), _f(batch["box_half"], "box_half"), _f(batch["box_rot"], "box_rot")
            out.update(box_id=e(R, M, dtype=_I32), t_in=e(R, M), t_out=e(R, M), sample_box=e(R, Nt, dtype=_I32))
            tables = [batch[k].to(dev) if batch.get(k) is not None else None for k in ("box_sem", "box_inst")]
            _, bs, bi, _ = primitive_tables(rays, out["sample_box"], *tables)
            keep += [bc, bh, br, bs, bi]
            a.box_center, a.box_half, a.box_rot = _capi.ptr(bc), _capi.ptr(bh), _capi.ptr(br)
            a.box_sem, a.box_inst, a.B, a.M = _capi.ptr(bs), _capi.ptr(bi), bc.shape[0], M
            hit8 = e(R, dtype=torch.uint8)
            a.hit_mask, a.box_id, a.t_in, a.t_out = _capi.ptr(hit8), _capi.ptr(out["box_id"]), _capi.ptr(out["t_in"]), _capi.ptr(out["t_out"])
            a.sample_box = _capi.ptr(out["sample_box"])
            if batch.get("mesh_tri_start") is not None or batch.get("mesh_tris") is not None:
                starts, tris = _mesh_table(batch.get("mesh_tri_start"), batch.get("mesh_tris"), bc.shape[0], dev)
                keep += [starts, tris]
                a.mesh_tri_start, a.mesh_tris, a.T = _capi.ptr(starts), _capi.ptr(tris), tris.shape[0]
            frames = _frame_table(batch.get("ray_frame"), batch.get("frame_boxes"), batch.get("static_boxes"), R, dev)
            if frames is not None:
                keep.append(frames[1])
        a.N, a.Ni = N, Ni
        tv = self._tv(N, dev)
        a.t_vals = _capi.ptr(tv)
        if perturb > 0.0:
            u = _f(batch["u"], "u") if "u" in batch else torch.rand(R, N, device=dev, dtype=_F32)
            keep.append(u)
            a.u = _capi.ptr(u)
        a.perturb = perturb
        if Ni > 0:
            if "u_fine" in batch:
                uf = _f(batch["u_fine"], "u_fine")
                a.u_fine_stride = Ni
            elif perturb == 0.0:
                uf = self._tv(Ni, dev)                 # deterministic sampler: one host-linspace row for every ray
                a.u_fine_stride = 0
            else:
                uf = torch.rand(R, Ni, device=dev, dtype=_F32)
                a.u_fine_stride = Ni
            keep.append(uf)
            a.u_fine = _capi.ptr(uf)
        a.sample_mode = _capi.SAMPLE_MODE[str(getattr(cfg, "sample_mode", "uniform"))] if has_boxes else 0
        a.white_bkgd = int(bool(getattr(cfg, "white_bkgd", False)))
        a.sem_softmax = int(str(getattr(cfg, "sem_activation", "none")) == "softmax")
        a.mask_outside = int(bool(getattr(cfg, "mask_outside", False)))
        a.bound_by_primitives = int(bool(getattr(cfg, "bound_by_primitives", False)))
        a.out, a.out0 = _capi.ptr_struct(_capi.PnrCompositeOut, final), _capi.ptr_struct(_capi.PnrCompositeOut, coarse)
        out["z_vals"] = e(R, Nt)
        a.z_vals = _capi.ptr(out["z_vals"])
        if Ni > 0:
            out["z_vals_0"] = e(R, N)
            a.z_vals0 = _capi.ptr(out["z_vals_0"])
        out["near"], out["far"] = near, far          # as given (bound_by_primitives works on a private copy)
        ws = self._workspace(ctx, R, N, Ni, dev)
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        if has_boxes and frames is not None:
            _capi.check(_capi.lib().pnr_render_fused_frames(ctx, ctx_fine, C.byref(a), C.byref(frames[0]),
                                                            _capi.stream_ptr()), "pnr_render_fused_frames")
        else:
            _capi.check(_capi.lib().pnr_render_fused(ctx, ctx_fine, C.byref(a), _capi.stream_ptr()), "pnr_render_fused")
        del keep
        if has_boxes:
            out["hit_mask"] = hit8.bool()
        out.update({k + "_0": v for k, v in coarse.items()})
        out.update(final)
        return out
