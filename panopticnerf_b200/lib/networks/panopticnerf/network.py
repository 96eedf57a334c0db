"""Network — the PanopticNeRF MLP (SURVEY.md 8(a) a8; reference: the Network class of the task's
network module under lib/networks/, not in the mount).

Parameter names follow nerf-pytorch, which the reference is recalled to inherit, so a reference
``state_dict`` loads with ``load_state_dict`` unchanged:
    pts_linears.{i}, alpha_linear, feature_linear, views_linears.0, rgb_linear,
    semantic_linears.{0,1}, instance_linears.{0,1}

``forward(pts, viewdirs)`` runs the fused sm_90a kernel (positional encoding + all layers + heads in one
launch, activations kept in shared memory) through the libpnr C ABI.  There is no PyTorch forward:
CPU tensors raise.

``cfg.xyz_encoding = "hashgrid"`` (a rule chosen here: the reference's 360 architecture is not in the mount) replaces
gamma(x) in layer 0 and in the skip concatenation by h(x), the features of a multi-resolution hash grid
(``xyz_encoder``, a `HashGrid`: parameter ``xyz_encoder.table`` [L, 2^T, F], buffer ``xyz_encoder.aabb``), E = L*F
<= 64 columns.  The fused kernel gathers h(x) on chip from the table in place, so an optimiser step on the table is
seen by the next launch without a repack.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional

import torch
import torch.nn as nn

from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.networks.encoding import HashGrid
from panopticnerf_b200.lib.networks.renderer.panopticnerf_renderer import empty_composite_maps, primitive_tables


def embed_dim(L: int) -> int:
    return 3 + 6 * L


def make_xyz_encoder(cfg) -> Optional[HashGrid]:
    """The hash grid of a cfg.xyz_encoding = "hashgrid" network (None for "frequency"), its limits checked."""
    enc = str(getattr(cfg, "xyz_encoding", "frequency"))
    if enc == "frequency":
        return None
    if enc != "hashgrid":
        raise ValueError(f"cfg.xyz_encoding={enc!r}: 'frequency' or 'hashgrid'")
    L, F_ = int(getattr(cfg, "hash_levels", 16)), int(getattr(cfg, "hash_features", 2))
    if F_ not in (1, 2, 4, 8) or not 1 <= L <= 32:
        raise ValueError(f"hash grid: hash_features={F_} must be in {{1, 2, 4, 8}} and hash_levels={L} in [1, 32]")
    if L * F_ > 64:
        raise ValueError(f"hash grid: E = hash_levels * hash_features = {L * F_} > 64 (the fused kernel's embedding operand)")
    aabb = getattr(cfg, "hash_aabb", None)
    if aabb is None:
        raise ValueError("cfg.xyz_encoding='hashgrid' needs cfg.hash_aabb = [lo.xyz, hi.xyz]")
    grad = str(getattr(cfg, "hash_grad", "atomic"))
    if grad not in ("atomic", "fixed"):
        raise ValueError(f"cfg.hash_grad={grad!r}: 'atomic' or 'fixed'")
    return HashGrid(L, F_, int(getattr(cfg, "hash_log2_size", 19)), float(getattr(cfg, "hash_base_resolution", 16.0)),
                    float(getattr(cfg, "hash_per_level_scale", 1.3819)), aabb=torch.as_tensor(aabb, dtype=torch.float32),
                    grad=grad)


class Network(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.D, self.W = int(cfg.D), int(cfg.W)
        self.Lx, self.Ld = int(cfg.xyz_res), int(cfg.view_res)
        self.C = int(getattr(cfg, "num_classes", 0))
        self.K = int(getattr(cfg, "num_instances", 0))
        self.precision = str(getattr(cfg, "precision", "fp16x3"))
        self.skip = self.D // 2
        encoder = make_xyz_encoder(cfg)
        Ex, Ed, W = embed_dim(self.Lx) if encoder is None else encoder.out_dim, embed_dim(self.Ld), self.W
        self.in_dim = Ex                          # trunk input width: 3 + 6*xyz_res, or E = L*F of the hash grid
        self.pts_linears = nn.ModuleList(
            [nn.Linear(Ex, W)] + [nn.Linear(W + Ex if i == self.skip + 1 else W, W) for i in range(1, self.D)])
        self.alpha_linear = nn.Linear(W, 1)
        self.feature_linear = nn.Linear(W, W)
        self.views_linears = nn.ModuleList([nn.Linear(W + Ed, W // 2)])
        self.rgb_linear = nn.Linear(W // 2, 3)
        if self.C > 0:
            self.semantic_linears = nn.ModuleList([nn.Linear(W, W // 2), nn.Linear(W // 2, self.C)])
        if self.K > 0:
            self.instance_linears = nn.ModuleList([nn.Linear(W, W // 2), nn.Linear(W // 2, self.K)])
        if encoder is not None:
            self.xyz_encoder = encoder
        self._ctx: Optional[int] = None
        self._ctx_key = None

    # The libpnr handle is a raw pointer owned by THIS object: copies (copy.deepcopy for EMA weights, pickling /
    # torch.save of the module, DataParallel replicas) must not share it - the copy would destroy the context the
    # original still uses.  A copy starts without a context and packs its own on first use.
    def __getstate__(self):
        state = self.__dict__.copy()
        state["_ctx"], state["_ctx_key"] = None, None
        return state

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k in ("_ctx", "_ctx_key") else copy.deepcopy(v, memo)
        return new

    def _replicate_for_data_parallel(self):
        replica = super()._replicate_for_data_parallel()
        replica._ctx, replica._ctx_key = None, None
        return replica

    # ------------------------------------------------------------------ libpnr context
    @property
    def out_channels(self) -> int:
        return 4 + self.C + self.K

    def _linears(self) -> List[nn.Linear]:
        ls = list(self.pts_linears) + [self.alpha_linear, self.feature_linear, self.views_linears[0],
                                       self.rgb_linear]
        if self.C > 0:
            ls += list(self.semantic_linears)
        if self.K > 0:
            ls += list(self.instance_linears)
        return ls

    @property
    def hashgrid(self) -> bool:
        return hasattr(self, "xyz_encoder")

    def _weights_key(self, device):
        # the hash-grid table is not packed (the kernel reads it in place): its updates do not repack the linears
        return (str(device), self.precision) + tuple((p.data_ptr(), p._version) for n, p in self.named_parameters()
                                                     if not n.startswith("xyz_encoder."))

    def _bind_table(self, device) -> None:
        """Hand the current table tensor to the context (every pack: a replaced parameter is picked up)."""
        t = self.xyz_encoder.table
        if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
            raise _capi.PnrError(f"Network: xyz_encoder.table must be a contiguous float32 tensor on {device}, got "
                                 f"{t.dtype} on {t.device}")
        _capi.check(_capi.lib().pnr_bind_hashgrid_table(self._ctx, t.data_ptr()), "pnr_bind_hashgrid_table")

    def pack(self, device=None) -> int:
        """The libpnr context of this network on `device` (built on first use, refreshed when a linear changed); a
        hash-grid network's table is (re)bound on every call."""
        ctx = self._pack(device)
        if self.hashgrid:
            self._bind_table(torch.device(self._ctx_key[0]))
        return ctx

    def _pack(self, device=None) -> int:
        """(Re)build the libpnr context: weights are split into 16-bit hi/lo wgmma stage images (fp16 or bf16 per cfg.precision; csrc/mlp_program.h) once, and
        again only when a parameter changed (SURVEY.md section 5, 'weight packer')."""
        device = torch.device(device if device is not None else next(self.parameters()).device)
        if device.type != "cuda":
            raise _capi.PnrError("Network.pack: parameters live on CPU - move the module to a CUDA device "
                                 "(panopticnerf_b200 has no CPU path)")
        key = self._weights_key(device)
        if self._ctx is not None and key == self._ctx_key:
            return self._ctx
        L = _capi.lib()
        if self._ctx is not None and key[:2] == self._ctx_key[:2] and self._fast_update:
            # same device, precision and architecture, new values (an optimiser step): refresh the packed streams on the
            # device from the parameters themselves (pnr_update_weights) - no host copy, no rebuild
            dev_t = []
            for lin in self._linears():
                dev_t += [lin.weight.detach().to(torch.float32).contiguous(), lin.bias.detach().to(torch.float32).contiguous()]
            ptrs = (C.c_void_p * len(dev_t))(*[_capi.ptr(t, torch.float32, "parameter") for t in dev_t])
            with torch.cuda.device(device):
                _capi.check(L.pnr_update_weights(self._ctx, ptrs, len(dev_t), _capi.stream_ptr()), "pnr_update_weights")
            self._ctx_key = key
            return self._ctx
        self.release()
        cfg = _capi.PnrConfig(self.D, self.W, self.Lx, self.Ld, self.C, self.K,
                              _capi.PREC[self.precision], device.index if device.index is not None
                              else torch.cuda.current_device())
        if self.hashgrid:
            e = self.xyz_encoder
            cfg.xyz_encoding = _capi.XYZ_ENCODING["hashgrid"]
            cfg.hash_levels, cfg.hash_features, cfg.hash_log2_size = e.L, e.F, e.T_log2
            cfg.hash_base_resolution, cfg.hash_per_level_scale = e.base, e.scale
            cfg.hash_aabb[:] = [float(v) for v in e.aabb.detach().cpu().reshape(6)]
        handle = C.c_void_p()
        _capi.check(L.pnr_create(C.byref(cfg), C.byref(handle)), "pnr_create")
        host, shapes = [], []
        for lin in self._linears():
            w = lin.weight.detach().to("cpu", torch.float32).contiguous()
            b = lin.bias.detach().to("cpu", torch.float32).contiguous()
            host += [w, b]
            shapes += [w.shape[0], w.shape[1], b.shape[0], 1]
        ptrs = (C.c_void_p * len(host))(*[t.data_ptr() for t in host])
        shp = (C.c_int64 * len(shapes))(*shapes)
        rc = L.pnr_load_weights(handle, ptrs, shp, len(host))
        if rc != 0:
            msg = L.pnr_last_error()
            L.pnr_destroy(handle)
            raise _capi.PnrError(f"pnr_load_weights failed (rc={rc}): {msg.decode()}")
        self._ctx, self._ctx_key = handle.value, key
        return self._ctx

    def release(self) -> None:
        if self._ctx is not None:
            _capi.lib().pnr_destroy(C.c_void_p(self._ctx))
            self._ctx, self._ctx_key = None, None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    # ------------------------------------------------------------------ forward
    def forward(self, pts: torch.Tensor, viewdirs: torch.Tensor) -> torch.Tensor:
        """raw[..., 4+C+K] = [rgb_raw(3), sigma_raw(1), semantic logits(C), instance logits(K)]."""
        if pts.shape != viewdirs.shape or pts.shape[-1] != 3:
            raise ValueError(f"Network.forward: pts {tuple(pts.shape)} / viewdirs {tuple(viewdirs.shape)}")
        p = pts.reshape(-1, 3).to(torch.float32).contiguous()
        v = viewdirs.reshape(-1, 3).to(torch.float32).contiguous()
        ctx = self.pack(p.device if p.is_cuda else None)
        pp, vp = _capi.ptr(p, torch.float32, "pts"), _capi.ptr(v, torch.float32, "viewdirs")   # CPU tensors raise here
        raw = torch.empty(p.shape[0], self.out_channels, device=p.device, dtype=torch.float32)
        with torch.cuda.device(p.device):        # the stream handed to libpnr is the tensors' device's current one
            _capi.check(_capi.lib().pnr_mlp_forward(ctx, pp, vp, None, None, p.shape[0], 1, _capi.ptr(raw),
                                                    _capi.stream_ptr()), "pnr_mlp_forward")
        return raw.reshape(*pts.shape[:-1], self.out_channels)

    def forward_rays(self, rays: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
        """Fused form used by the Renderer: pts = o + d*z and viewdirs = d/|d| are formed in-kernel."""
        R, N = z.shape
        ctx = self.pack(rays.device if rays.is_cuda else None)
        rp, zp = _capi.ptr(rays, torch.float32, "rays"), _capi.ptr(z, torch.float32, "z")       # CPU tensors raise here
        raw = torch.empty(R, N, self.out_channels, device=rays.device, dtype=torch.float32)
        with torch.cuda.device(rays.device):
            _capi.check(_capi.lib().pnr_mlp_forward(ctx, None, None, rp, zp, R, N, _capi.ptr(raw),
                                                    _capi.stream_ptr()), "pnr_mlp_forward")
        return raw

    def forward_composite(self, rays: torch.Tensor, z: torch.Tensor, white_bkgd: bool = False,
                          mask_outside: bool = False, sample_box: Optional[torch.Tensor] = None,
                          box_sem: Optional[torch.Tensor] = None, box_inst: Optional[torch.Tensor] = None):
        """Network.forward + raw2outputs in ONE kernel (pnr_mlp_composite): the compositing runs in the MLP's epilogue
        and `raw` is never written.  Returns the dict raw2outputs returns.  Needs N % 32 == 0; the primitive tables are
        refused, as by raw2outputs, when they live on another device or the id tables differ in length."""
        R, N = z.shape
        dev = rays.device
        ctx = self.pack(dev if rays.is_cuda else None)
        rp, zp = _capi.ptr(rays, torch.float32, "rays"), _capi.ptr(z, torch.float32, "z")
        sb, bs, bi, B = primitive_tables(rays, sample_box, box_sem, box_inst)
        out = empty_composite_maps(R, N, self.C, self.K, sb is not None and bs is not None,
                                   sb is not None and bi is not None, dev)
        co = _capi.ptr_struct(_capi.PnrCompositeOut, out)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().pnr_mlp_composite(ctx, rp, zp, R, N, int(bool(white_bkgd)), int(bool(mask_outside)),
                                                      _capi.ptr(sb), _capi.ptr(bs), _capi.ptr(bi), B, C.byref(co),
                                                      _capi.stream_ptr()), "pnr_mlp_composite")
        return out

    def _samples(self, pts, rays, z):
        if pts is not None:
            return pts.shape[0], 1, pts.shape[0], pts.device
        R, N = z.shape
        return R, N, R * N, rays.device

    def trunk_forward(self, pts: Optional[torch.Tensor] = None, rays: Optional[torch.Tensor] = None,
                      z: Optional[torch.Tensor] = None) -> torch.Tensor:
        """h [S, W]: the output of the trunk (`pts_linears`, after the last ReLU) for the samples given as pts [S,3]
        or as (rays [R,6], z [R,N]) - pnr_mlp_trunk_forward.  The input of alpha / feature / view / rgb / heads."""
        R, N, S_, dev = self._samples(pts, rays, z)
        ctx = self.pack(dev if (pts if pts is not None else rays).is_cuda else None)
        h = torch.empty(S_, self.W, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().pnr_mlp_trunk_forward(
                ctx, _capi.ptr(pts, torch.float32, "pts"), _capi.ptr(rays, torch.float32, "rays"),
                _capi.ptr(z, torch.float32, "z"), R, N, _capi.ptr(h), _capi.stream_ptr()), "pnr_mlp_trunk_forward")
        return h

    def backward_trunk(self, grad_h: torch.Tensor, pts: Optional[torch.Tensor] = None,
                       rays: Optional[torch.Tensor] = None, z: Optional[torch.Tensor] = None,
                       stash: bool = False, grad_scale: Optional[float] = None, absmax: bool = False):
        """The tensor-core part of the MLP backward (pnr_mlp_backward_trunk): dL/d(trunk input) [S, in_dim] (gamma(x), or
        h(x) for a hash-grid network) from
        grad_h = dL/dh of the trunk output [S, W], for the samples given as pts [S,3] or as (rays [R,6], z [R,N]).
        What autograd computes through `pts_linears` (ReLUs, skip concatenation) of the reference Network.
        stash=True also returns the operands of the weight-gradient GEMMs, [2D-1, S, W] fp32: slot i < D-1 = the
        activations H_i of layer i, slot 2D-2-j = dZ_j, the gradient w.r.t. layer j's pre-activation.
        grad_scale: the power of two grad_h is multiplied by inside the kernel (and the results divided by); default:
        the one that brings max |grad_h| to ~256 (one reduction over grad_h; the pass is linear, the scaling exact).
        absmax=True (with stash) also returns a device tensor [2D-1] fp32: the largest |value| in every stash slot (to
        the 11 / 8 bits of the operand format's hi part), collected by the kernel itself - what picks the
        power-of-two scale of the weight-gradient GEMMs without another pass over the stash."""
        R, N, S_, dev = self._samples(pts, rays, z)
        assert grad_h.shape == (S_, self.W), f"grad_h must be [{S_}, {self.W}]"
        ctx = self.pack(dev if grad_h.is_cuda else None)
        Ex = self.in_dim
        ld = (Ex + 15) // 16 * 16                  # rows padded to whole 16-column groups: 16-byte stores in the kernel
        out = torch.empty(S_, ld, dtype=torch.float32, device=dev)
        st = torch.empty(2 * self.D - 1, S_, self.W, dtype=torch.float32, device=dev) if stash else None
        am = torch.empty(2 * self.D - 1, dtype=torch.int32, device=dev) if (stash and absmax) else None
        if grad_scale is None:
            m = float(grad_h.abs().max()) if grad_h.is_cuda else 0.0
            grad_scale = 2.0 ** max(-100, min(100, round(math.log2(256.0 / m)))) if m > 0.0 and math.isfinite(m) else 1.0
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().pnr_mlp_backward_trunk(
                ctx, _capi.ptr(pts, torch.float32, "pts"), _capi.ptr(rays, torch.float32, "rays"),
                _capi.ptr(z, torch.float32, "z"), R, N, _capi.ptr(grad_h, torch.float32, "grad_h"), float(grad_scale),
                _capi.ptr(out), ld, _capi.ptr(st), _capi.ptr(am), _capi.stream_ptr()), "pnr_mlp_backward_trunk")
        if am is not None:
            # 16-bit patterns of the operand format -> magnitudes; the gradient slots (D-1 ..) were seen scaled
            half = torch.float16 if self.precision.startswith("fp16") else torch.bfloat16
            mag = am.to(torch.int16).view(half).to(torch.float32)
            mag[self.D - 1:] /= float(grad_scale)
            return out[:, :Ex], st, mag
        return (out[:, :Ex], st) if stash else out[:, :Ex]

    _fast_update = True      # class-level switch (tests compare against the full reload)

    def range_status(self, reset: bool = True) -> int:
        """Sticky range-check word of this network's fused-MLP launches (synchronises the current stream).
        Bit 0 set: a value written into a 16-bit operand (an embedding, an activation, a scaled gradient) rounded to inf
        in that format (fp16 modes: |x| >= 65520) or was NaN - those outputs are wrong; for a finite overflow use
        precision='bf16x3' for this network.  A NaN input or parameter also reaches the outputs as NaN.
        Bit 1 set: pnr_update_weights packed a weight outside the fp16 range."""
        if self._ctx is None:
            return 0
        dev = torch.device(self._ctx_key[0])
        out = C.c_uint32(0)
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().pnr_status(self._ctx, C.byref(out), int(bool(reset)), _capi.stream_ptr()),
                        "pnr_status")
        return int(out.value)

    def check_range(self) -> None:
        """Raise if a launch since the last check overflowed the operand format (never silent)."""
        st = self.range_status(reset=True)
        if st & 2:
            raise _capi.PnrError(f"Network: a weight is outside the fp16 range (|w| > 65504 or not finite) after an update - "
                                 "the packed weights are invalid; use cfg.precision = 'bf16x3'")
        if st & 1:
            raise _capi.PnrError(
                f"Network: an activation left the range of the {self.precision} tensor-core operands (|x| >= 65520 in "
                "fp16, or NaN) - the MLP outputs of this call are invalid; use cfg.precision = 'bf16x3'")
