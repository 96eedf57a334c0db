"""Multi-resolution hash-grid feature encoder (SURVEY 8(f) rank 4: the 360 model's extra encoder): `pnr_hashgrid_encode`
forward, `pnr_hashgrid_backward` for the gradient w.r.t. the table (an fp32 parameter [L, 2^T_log2, F]); the points
are treated as constants."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from .... import _capi


class _HashGridFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, xc, aabb, L, F, T_log2, base, scale):
        p = _capi.ptr
        out = torch.empty(xc.shape[0], L * F, dtype=torch.float32, device=xc.device)
        with torch.cuda.device(xc.device):
            _capi.check(_capi.lib().pnr_hashgrid_encode(p(xc, torch.float32, "x"), xc.shape[0], p(aabb), p(table, torch.float32, "table"),
                                                        L, F, T_log2, base, scale, p(out), _capi.stream_ptr()), "pnr_hashgrid_encode")
        ctx.save_for_backward(xc, aabb if aabb is not None else torch.empty(0, device=xc.device))
        ctx.meta = (tuple(table.shape), aabb is not None, L, F, T_log2, base, scale)
        return out

    @staticmethod
    def backward(ctx, g):
        xc, aabb = ctx.saved_tensors
        shape, has_aabb, L, F, T_log2, base, scale = ctx.meta
        gt = _table_grad(shape, xc, aabb if has_aabb else None, g, L, F, T_log2, base, scale)
        return gt, None, None, None, None, None, None, None


def _table_grad(shape, xc, aabb, g, L, F, T_log2, base, scale) -> torch.Tensor:
    p = _capi.ptr
    gt = torch.zeros(shape, dtype=torch.float32, device=xc.device)
    gc = g.to(torch.float32).contiguous()
    with torch.cuda.device(xc.device):
        _capi.check(_capi.lib().pnr_hashgrid_backward(p(xc), xc.shape[0], p(aabb), p(gc), L, F, T_log2,
                                                      base, scale, p(gt), _capi.stream_ptr()), "pnr_hashgrid_backward")
    return gt


class HashGrid(nn.Module):
    def __init__(self, n_levels: int = 16, n_features: int = 2, log2_hashmap_size: int = 19, base_resolution: float = 16.0,
                 per_level_scale: float = 1.3819, aabb: Optional[torch.Tensor] = None, seed: int = 0):
        super().__init__()
        self.L, self.F, self.T_log2 = int(n_levels), int(n_features), int(log2_hashmap_size)
        self.base, self.scale = float(base_resolution), float(per_level_scale)
        g = torch.Generator().manual_seed(seed)
        self.table = nn.Parameter((torch.rand(self.L, 1 << self.T_log2, self.F, generator=g) * 2 - 1) * 1e-4)
        self.register_buffer("aabb", None if aabb is None else torch.as_tensor(aabb, dtype=torch.float32).reshape(6).clone())

    @property
    def out_dim(self) -> int:
        return self.L * self.F

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        xc = x.reshape(-1, 3).to(torch.float32).contiguous()
        _capi.ptr(xc, torch.float32, "x")                                          # CPU tensors raise here
        out = _HashGridFn.apply(self.table, xc, self.aabb, self.L, self.F, self.T_log2, self.base, self.scale)
        return out.reshape(*x.shape[:-1], self.out_dim)

    def table_grad(self, x: torch.Tensor, grad_out: torch.Tensor) -> torch.Tensor:
        """dL/dtable [L, 2^T_log2, F] for dL/d(features) grad_out [n, L*F] at the points x [n, 3] (pnr_hashgrid_backward;
        fp32 atomics, so the last bits vary between runs)."""
        xc = x.reshape(-1, 3).to(torch.float32).contiguous()
        return _table_grad(tuple(self.table.shape), xc, self.aabb, grad_out.reshape(xc.shape[0], self.out_dim), self.L,
                           self.F, self.T_log2, self.base, self.scale)
