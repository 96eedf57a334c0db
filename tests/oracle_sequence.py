"""Oracle of a5 on a sequence table (DESIGN 3.2, include/pnr.h pnr_intersect_frames): the rays of each frame are
intersected with that frame's own table cat(static, block) by any single-table intersection (the torch oracle, the host
build, the device kernel), and the dynamic ids are mapped back to the sequence table (seq_id = id + begin - S).  Also a
random sequence table and the per-frame tables the renderer tests compare against."""
from __future__ import annotations

import torch

PRIM_KEYS = ("box_center", "box_half", "box_rot", "box_sem", "box_inst")


def frame_range(f: int, frame_boxes, F: int, S: int, B: int):
    """[b0, b1) of frame f's block, clamped as ray_math.h pnr_frame_range."""
    if not 0 <= f < F:
        return S, S
    a, e = int(frame_boxes[f][0]), int(frame_boxes[f][1])
    lo = min(max(a, S), B)
    return lo, min(max(e, lo), B)


def frame_table(prims, S: int, b0: int, b1: int):
    """The per-frame table cat(static, block [b0, b1)) of a sequence table (mesh ranges clamped as the kernel does)."""
    sel = list(range(S)) + list(range(b0, b1))
    idx = torch.tensor(sel, dtype=torch.int64)
    out = {k: prims[k][idx.to(prims[k].device)].contiguous() for k in PRIM_KEYS if k in prims}
    if prims.get("mesh_tri_start") is not None:
        start = prims["mesh_tri_start"].to(torch.int64).cpu()
        tris = prims["mesh_tris"]
        T = tris.shape[0]
        lo = start[:-1].clamp(0, T)
        hi = torch.maximum(start[1:], lo).clamp(max=T)
        parts, st = [], [0]
        for b in sel:
            parts.append(tris[int(lo[b]):int(hi[b])])
            st.append(st[-1] + int(hi[b] - lo[b]))
        if st[-1] == 0:    # no triangle left: a cuboid table
            return out
        out["mesh_tri_start"] = torch.tensor(st, dtype=torch.int32, device=prims["mesh_tri_start"].device)
        out["mesh_tris"] = torch.cat(parts, 0).contiguous()
    return out


def groups(ray_frame, frame_boxes, S: int, B: int):
    """{(b0, b1): ray indices} for the rays of each distinct clamped block."""
    F = int(frame_boxes.shape[0])
    rf = ray_frame.cpu()
    fb = frame_boxes.cpu().tolist()
    out = {}
    for f in torch.unique(rf).tolist():
        key = frame_range(int(f), fb, F, S, B)
        rows = torch.nonzero(rf == f).flatten()
        out[key] = torch.cat([out[key], rows]) if key in out else rows
    return {k: torch.sort(v).values for k, v in out.items()}


def per_frame(intersect_one, rays, prims, S: int, frame_boxes, ray_frame, M: int):
    """(hit, box_id, t_in, t_out) of the sequence table from `intersect_one(rays, table, M)` on each frame's table."""
    R, B = rays.shape[0], prims["box_center"].shape[0]
    dev = rays.device
    hit = torch.zeros(R, dtype=torch.bool, device=dev)
    bid = torch.full((R, M), -1, dtype=torch.int32, device=dev)
    tin, tout = torch.zeros(R, M, device=dev), torch.zeros(R, M, device=dev)
    for (b0, b1), rows in groups(ray_frame, frame_boxes, S, B).items():
        rows = rows.to(dev)
        h, i, a, b = intersect_one(rays[rows].contiguous(), frame_table(prims, S, b0, b1), M)
        i = torch.where(i >= S, i + (b0 - S), i)
        hit[rows], bid[rows], tin[rows], tout[rows] = h.bool().to(dev), i.to(dev), a.to(dev), b.to(dev)
    return hit, bid, tin, tout


def random_sequence(prims, S: int, F: int, max_block: int, seed: int, shared: int = 0):
    """frame_boxes [F,2] int32 over the dynamic part [S, B) of `prims`: blocks of 0..max_block primitives, drawn at
    random positions (blocks overlap and repeat), the last `shared` frames reusing earlier frames' rows."""
    B = prims["box_center"].shape[0]
    g = torch.Generator().manual_seed(seed)
    n = torch.randint(0, max_block + 1, (F,), generator=g)
    n = torch.minimum(n, torch.tensor(B - S))
    begin = S + (torch.rand(F, generator=g) * (B - S - n + 1).float()).long().clamp(max=B)
    fb = torch.stack([begin, begin + n], 1).to(torch.int32)
    if shared:
        fb[F - shared:] = fb[torch.randint(0, F - shared, (shared,), generator=g)]
    return fb.contiguous()
