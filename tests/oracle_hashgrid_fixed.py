"""Oracle of pnr_hashgrid_backward_fixed: steps 1-5 of the rule in include/pnr.h, restated in numpy.  The corner weights
and rows are those of oracle/reference_panoptic.hashgrid_encode (its level resolutions and its fp32 operations, in its
order; `forward_from_corners` recomposes that function's output from them, bit for bit); the sums are int64
(`np.add.at`), and every level's absolute sum is checked in Python integers against the int64 range.  Test
infrastructure only."""
from __future__ import annotations

import numpy as np
import torch

from oracle import reference_panoptic as OP

F32 = np.float32


def ceil_log2(n: int) -> int:
    return (int(n) - 1).bit_length()


def frexp_exponent(m: float) -> int:
    return int(np.frexp(np.float64(m))[1])


def level_scale(m: float, n: int):
    """s_l of a level whose largest finite |g| is m (None when m = 0: the level adds nothing)."""
    return None if m == 0 else 61 - ceil_log2(n) - frexp_exponent(m)


def corners(x, aabb, L: int, T: int, base: float, scale: float):
    """[(w [n, 8] fp32, idx [n, 8] int64)] per level: the weight and the table row of each corner, corner order x fastest
    (the arithmetic of reference_panoptic.hashgrid_encode)."""
    v = torch.as_tensor(x, dtype=torch.float32).reshape(-1, 3)
    if aabb is not None:
        a = torch.as_tensor(aabb, dtype=torch.float32).reshape(2, 3)
        v = (v - a[0]) / (a[1] - a[0])
    v = torch.clamp(v, 0.0, 1.0)
    out = []
    for res in OP.hashgrid_resolutions(L, base, scale):
        res_f = torch.tensor(float(res), dtype=torch.float32)
        p = v * res_f
        fl = torch.floor(p)
        fl = torch.where(fl >= res_f, res_f - 1.0, fl)
        w = p - fl
        c = fl.to(torch.int64)
        res1 = res + 1
        dense = res1 ** 3 <= T
        ws, idxs = [], []
        for k in range(8):
            dx, dy, dz = k & 1, (k >> 1) & 1, k >> 2
            wx = w[:, 0] if dx else 1.0 - w[:, 0]
            wy = w[:, 1] if dy else 1.0 - w[:, 1]
            wz = w[:, 2] if dz else 1.0 - w[:, 2]
            cx, cy, cz = c[:, 0] + dx, c[:, 1] + dy, c[:, 2] + dz
            if dense:
                idx = cx + cy * res1 + cz * res1 * res1
            else:
                idx = ((cx & 0xFFFFFFFF) ^ ((cy * 2654435761) & 0xFFFFFFFF) ^ ((cz * 805459861) & 0xFFFFFFFF)) & (T - 1)
            ws.append((wx * wy) * wz)
            idxs.append(idx)
        out.append((torch.stack(ws, 1).numpy(), torch.stack(idxs, 1).numpy()))
    return out


def forward_from_corners(cs, table) -> torch.Tensor:
    """The encoder's output from `corners` and a table [L, T, F], summed in the forward's order."""
    outs = []
    for l, (w, idx) in enumerate(cs):
        tab = torch.as_tensor(table[l], dtype=torch.float32)
        acc = torch.zeros(w.shape[0], tab.shape[1], dtype=torch.float32)
        for k in range(8):
            acc = acc + torch.from_numpy(w[:, k])[:, None] * tab[torch.from_numpy(idx[:, k])]
        outs.append(acc)
    return torch.cat(outs, -1)


def _abs_sum(q: np.ndarray) -> int:
    """sum |q| exactly, in Python integers (two 32-bit halves, each summed in int64 without overflow)."""
    a = np.abs(q.astype(np.int64)).astype(np.uint64)
    lo = int((a & np.uint64(0xFFFFFFFF)).astype(np.int64).sum())
    hi = int((a >> np.uint64(32)).astype(np.int64).sum())
    return (hi << 32) + lo


def table_grad_fixed(x, aabb, grad_out, L: int, F: int, T_log2: int, base: float, scale: float, grad_table=None,
                     cs=None, stats=None):
    """grad_table [L, T, F] fp32 after pnr_hashgrid_backward_fixed (ACCUMULATES into a copy of grad_table, zeros when
    None).  `cs`: the points' corners, when the caller already has them.  `stats` (a dict) receives per level m_l, s_l,
    the exact absolute sum of the quantized contributions and the int64 sums."""
    T = 1 << T_log2
    g = np.ascontiguousarray(np.asarray(grad_out, dtype=F32)).reshape(-1, L, F)
    n = g.shape[0]
    out = np.zeros((L, T, F), F32) if grad_table is None else np.array(grad_table, dtype=F32).reshape(L, T, F).copy()
    if n == 0:
        return out
    cs = corners(x, aabb, L, T, base, scale) if cs is None else cs
    fin = np.isfinite(g)
    for l, (w, idx) in enumerate(cs):
        gl = np.where(fin[:, l], g[:, l], F32(0))
        m = float(np.abs(gl).max())
        s = level_scale(m, n)
        poison = np.zeros((T, F), bool)
        acc = np.zeros((T, F), np.int64)
        total = 0
        for k in range(8):
            for f in range(F):
                bad = ~fin[:, l, f]
                poison[idx[bad, k], f] = True
                if s is None:
                    continue
                c = (w[:, k] * gl[:, f]).astype(F32)              # one fp32 product (w, g fp32)
                q = np.rint(c.astype(np.float64) * 2.0 ** s).astype(np.int64)
                total += _abs_sum(q)
                np.add.at(acc[:, f], idx[:, k], q)
        assert total < 2 ** 63, f"level {l}: |sum| = {total} overflows int64"
        if stats is not None:
            stats[l] = dict(m=m, s=s, abs_sum=total, acc=acc)
        if s is not None:
            out[l] = (out[l] + (acc.astype(np.float64) * 2.0 ** -s).astype(F32)).astype(F32)
        out[l][poison] = np.nan
    return out
