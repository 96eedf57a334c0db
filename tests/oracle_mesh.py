"""Oracle of the mesh primitives of a5 (DESIGN 3.2): `pnr_intersect_meshes` restated in torch fp32 with the
operation order of csrc/ray_math.h (pnr_shear, pnr_tri_cross, PnrMeshCross), vectorised over rays x triangles.  It
extends oracle/reference_renderer.py::intersect, which it calls unchanged for a table without meshes, and runs on the
device of its inputs (every op is a separately rounded IEEE op on either)."""
from __future__ import annotations

import contextlib
from typing import Optional

import torch

from oracle import reference_renderer as O

INF = float("inf")


def _pick(a0, a1, a2, k):
    return torch.where(k == 0, a0, torch.where(k == 1, a1, a2))


def shear(d):
    """Per ray: kx, ky, kz [R,1] and sx, sy, sz [R,1] (ray_math.h pnr_shear)."""
    ad = d.abs()
    kz = torch.where(ad[:, 1] > ad[:, 0], 1, 0)
    kz = torch.where(ad[:, 2] > torch.where(kz == 0, ad[:, 0], ad[:, 1]), 2, kz)
    kx = torch.where(kz == 2, 0, kz + 1)
    ky = torch.where(kx == 2, 0, kx + 1)
    dk = _pick(d[:, 0], d[:, 1], d[:, 2], kz)
    neg = dk < 0
    kx, ky = torch.where(neg, ky, kx), torch.where(neg, kx, ky)
    sx = _pick(d[:, 0], d[:, 1], d[:, 2], kx) / dk
    sy = _pick(d[:, 0], d[:, 1], d[:, 2], ky) / dk
    sz = torch.ones_like(dk) / dk
    return [x[:, None] for x in (kx, ky, kz, sx, sy, sz)]


def _tie(px, py, qx, qy):
    one = torch.ones_like(px, dtype=torch.int8)
    return torch.where(py != qy, torch.where(py > qy, one, -one),
                       torch.where(qx != px, torch.where(qx > px, one, -one), 0 * one))


def _sign(x):
    return torch.sign(x).to(torch.int8)


def crossings(o, d, tris):
    """o, d [R,3]; tris [T,3,3] -> (cross [R,T] bool, t [R,T]) (ray_math.h pnr_tri_cross)."""
    kx, ky, kz, sx, sy, sz = shear(d)
    v = tris.reshape(-1, 9)
    rel = [v[None, :, j] - o[:, None, j % 3] for j in range(9)]          # vertex - origin, [R,T] each
    sh = []
    for p in range(3):
        a0, a1, a2 = rel[3 * p:3 * p + 3]
        z = _pick(a0, a1, a2, kz)
        sh.append((_pick(a0, a1, a2, kx) - sx * z, _pick(a0, a1, a2, ky) - sy * z, z))
    (ax, ay, az), (bx, by, bz), (cx, cy, cz) = sh
    U = cx * by - cy * bx
    V = ax * cy - ay * cx
    W = bx * ay - by * ax
    redo = (U == 0) | (V == 0) | (W == 0)
    dd = lambda x: x.double()
    Ud = dd(cx) * dd(by) - dd(cy) * dd(bx)
    Vd = dd(ax) * dd(cy) - dd(ay) * dd(cx)
    Wd = dd(bx) * dd(ay) - dd(by) * dd(ax)
    U, V, W = torch.where(redo, Ud.float(), U), torch.where(redo, Vd.float(), V), torch.where(redo, Wd.float(), W)
    su = torch.where(redo, _sign(Ud), _sign(U))
    sv = torch.where(redo, _sign(Vd), _sign(V))
    sw = torch.where(redo, _sign(Wd), _sign(W))
    su = torch.where(su == 0, _tie(cx, cy, bx, by), su)
    sv = torch.where(sv == 0, _tie(ax, ay, cx, cy), sv)
    sw = torch.where(sw == 0, _tie(bx, by, ax, ay), sw)
    cross = ((su > 0) & (sv > 0) & (sw > 0)) | ((su < 0) & (sv < 0) & (sw < 0))
    det = (U + V) + W
    T = ((U * (sz * az)) + (V * (sz * bz))) + (W * (sz * cz))
    t = T / det
    cross = cross & (det != 0) & (t == t)
    return cross, t


def mesh_intervals(cross, t, M: int):
    """Crossings [R,T] of one mesh -> (a, b, hit) [R,M]: the mesh's hit intervals in order (ray_math.h PnrMeshCross).
    Sorted along the line the crossings pair up; an odd count gives the hull; of the intervals with b > 0 the first
    M are kept, and the ones with b > max(a, 0) are hits."""
    R = cross.shape[0]
    n = cross.sum(1)
    s = torch.sort(torch.where(cross, t, torch.full_like(t, INF)), 1).values
    if s.shape[1] % 2:
        s = torch.cat([s, torch.full_like(s[:, :1], INF)], 1)
    a, b = s[:, 0::2], s[:, 1::2]
    P = a.shape[1]
    valid = torch.arange(P, device=t.device)[None] < (n // 2)[:, None]
    cand = valid & (b > 0)
    keep = cand & (torch.cumsum(cand.to(torch.int64), 1) <= M)
    hit = keep & (b > torch.maximum(a, torch.zeros_like(a)))
    odd = (n % 2) == 1
    lo = s[:, 0]
    hi = torch.gather(s, 1, (n - 1).clamp(min=0)[:, None])[:, 0]
    # compact the hits to the front, in order
    rank = torch.cumsum(hit.to(torch.int64), 1) - 1
    out_a = torch.zeros(R, M + 1, dtype=t.dtype, device=t.device)
    out_b = torch.zeros(R, M + 1, dtype=t.dtype, device=t.device)
    out_h = torch.zeros(R, M + 1, dtype=torch.bool, device=t.device)
    slot = torch.where(hit, rank, torch.full_like(rank, M))
    out_a.scatter_(1, slot, torch.where(hit, a, torch.zeros_like(a)))
    out_b.scatter_(1, slot, torch.where(hit, b, torch.zeros_like(b)))
    out_h.scatter_(1, slot, hit)
    out_a, out_b, out_h = out_a[:, :M], out_b[:, :M], out_h[:, :M]
    hull_hit = odd & (hi > torch.maximum(lo, torch.zeros_like(lo)))
    out_a[:, 0] = torch.where(odd, lo, out_a[:, 0])
    out_b[:, 0] = torch.where(odd, hi, out_b[:, 0])
    out_h[:, 0] = torch.where(odd, hull_hit, out_h[:, 0])
    out_h[:, 1:] &= ~odd[:, None]
    return out_a, out_b, out_h


def intersect(o, d, center, half, rot, max_hits: int, mesh_tri_start=None, mesh_tris=None, chunk: Optional[int] = None):
    """`oracle.reference_renderer.intersect` with an optional mesh table (include/pnr.h pnr_intersect_meshes)."""
    if mesh_tri_start is None:
        return O.intersect(o, d, center, half, rot, max_hits)
    R, B, M = o.shape[0], center.shape[0], int(max_hits)
    dev = o.device
    T = mesh_tris.shape[0]
    start = mesh_tri_start.to(torch.int64).cpu()
    lo_r = start[:-1].clamp(0, T)
    hi_r = torch.maximum(start[1:], lo_r).clamp(max=T)
    chunk = chunk or max(1, (1 << 24) // max(1, B * M))
    outs = []
    for r0 in range(0, R, chunk):
        oc, dc = o[r0:r0 + chunk], d[r0:r0 + chunk]
        Rc = oc.shape[0]
        tmin, tmax, hit = O.slab_test(oc, dc, center, half, rot)        # [Rc,B]
        key = torch.full((Rc, B, M), INF, device=dev)
        tout = torch.zeros(Rc, B, M, device=dev)
        h = torch.zeros(Rc, B, M, dtype=torch.bool, device=dev)
        key[:, :, 0], tout[:, :, 0], h[:, :, 0] = tmin, tmax, hit
        for b in range(B):
            k0, k1 = int(lo_r[b]), int(hi_r[b])
            if k0 == k1:
                continue
            h[:, b] = False
            rows = torch.nonzero(hit[:, b]).flatten()
            step = max(1, (1 << 21) // (k1 - k0))
            for i in range(0, rows.numel(), step):
                rr = rows[i:i + step]
                cross, t = crossings(oc[rr], dc[rr], mesh_tris[k0:k1])
                a, bb, hh = mesh_intervals(cross, t, M)
                key[rr, b], tout[rr, b], h[rr, b] = a, bb, hh
        key = torch.where(h, key, torch.full_like(key, INF)).reshape(Rc, B * M)
        tout, h = tout.reshape(Rc, B * M), h.reshape(Rc, B * M)
        order = torch.sort(key, dim=1, stable=True).indices[:, :M]
        hs = torch.gather(h, 1, order)
        bid = torch.where(hs, (order // M).to(torch.int32), torch.full_like(order, -1, dtype=torch.int32))
        t_in = torch.where(hs, torch.maximum(torch.gather(key, 1, order), torch.zeros((), device=dev)),
                           torch.zeros((), device=dev))
        t_out = torch.where(hs, torch.gather(tout, 1, order), torch.zeros((), device=dev))
        pad = M - order.shape[1]
        if pad:
            bid = torch.nn.functional.pad(bid, (0, pad), value=-1)
            t_in, t_out = torch.nn.functional.pad(t_in, (0, pad)), torch.nn.functional.pad(t_out, (0, pad))
        outs.append((h.any(1), bid, t_in, t_out))
    return tuple(torch.cat([x[i] for x in outs], 0).contiguous() for i in range(4))


@contextlib.contextmanager
def oracle_renderer_with_meshes():
    """While active, the oracle Renderer's intersection reads the batch keys mesh_tri_start / mesh_tris (the oracle
    module itself takes a cuboid table only)."""
    orig, orig_render_rays = O.intersect, O.Renderer.render_rays
    state = {}

    def render_rays(self, rays, near, far, batch, sl):
        state["mesh"] = (batch.get("mesh_tri_start"), batch.get("mesh_tris"))
        return orig_render_rays(self, rays, near, far, batch, sl)

    def patched(o, d, center, half, rot, max_hits):
        mts, mt = state.get("mesh", (None, None))
        if mts is None:
            return orig(o, d, center, half, rot, max_hits)
        return intersect(o, d, center, half, rot, max_hits, mts, mt)

    O.intersect, O.Renderer.render_rays = patched, render_rays
    try:
        yield
    finally:
        O.intersect, O.Renderer.render_rays = orig, orig_render_rays
