"""Seeded synthetic inputs of KITTI-360 shape (SURVEY.md section 8(d)): pinhole / equirect rays,
a scene AABB, B oriented bounding primitives, and network weights.  Pure CPU torch, deterministic;
both bench arms and the tests draw their inputs from here so they see identical data.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

SCENE_AABB = ((-16.0, -4.0, 0.0), (16.0, 12.0, 64.0))


def make_rays(cfg, seed: int = 0, row0: int = 0, rows: Optional[int] = None) -> torch.Tensor:
    """[rows*W, 6] fp32 = origin || unnormalised direction, row-major over (v, u)."""
    H, W = int(cfg.H), int(cfg.W_img)
    rows = H - row0 if rows is None else rows
    g = torch.Generator().manual_seed(seed)
    yaw = (torch.rand((), generator=g).item() - 0.5) * 0.1
    v, u = torch.meshgrid(torch.arange(row0, row0 + rows, dtype=torch.float32),
                          torch.arange(W, dtype=torch.float32), indexing="ij")
    if getattr(cfg, "camera", "pinhole") == "equirect":
        lon = (u / W - 0.5) * (2.0 * math.pi)
        lat = (0.5 - v / H) * math.pi
        d = torch.stack([torch.cos(lat) * torch.sin(lon), -torch.sin(lat),
                         torch.cos(lat) * torch.cos(lon)], -1)
        origin = torch.tensor([0.0, 4.0, 32.0])          # panorama taken inside the scene
    else:
        d = torch.stack([(u - cfg.cx) / cfg.fx, (v - cfg.cy) / cfg.fy, torch.ones_like(u)], -1)
        origin = torch.tensor([0.0, 0.0, 0.0])
    c, s = math.cos(yaw), math.sin(yaw)
    rot = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
    d = (d.reshape(-1, 3) @ rot.T).contiguous()
    o = origin[None].expand_as(d)
    return torch.cat([o, d], -1).contiguous()


def make_boxes(num_boxes: int = 64, num_classes: int = 45, num_instances: int = 64,
               seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed + 1)
    lo = torch.tensor(SCENE_AABB[0])
    hi = torch.tensor(SCENE_AABB[1])
    center = lo + (hi - lo) * torch.rand(num_boxes, 3, generator=g)
    half = 0.5 + 3.5 * torch.rand(num_boxes, 3, generator=g)
    yaw = 2.0 * math.pi * torch.rand(num_boxes, generator=g)
    c, s = torch.cos(yaw), torch.sin(yaw)
    z, one = torch.zeros_like(c), torch.ones_like(c)
    rot = torch.stack([torch.stack([c, z, s], -1), torch.stack([z, one, z], -1),
                       torch.stack([-s, z, c], -1)], -2)       # [B,3,3], columns = box axes
    sem = torch.randint(0, max(num_classes, 1), (num_boxes,), generator=g, dtype=torch.int32)
    inst = torch.randint(0, max(num_instances, 1), (num_boxes,), generator=g, dtype=torch.int32)
    return dict(box_center=center.contiguous(), box_half=half.contiguous(), box_rot=rot.contiguous(),
                box_sem=sem, box_inst=inst)


def make_batch(cfg, seed: int = 0, row0: int = 0, rows: Optional[int] = None, num_boxes: int = 64,
               with_boxes: bool = True) -> Dict[str, torch.Tensor]:
    batch = {"rays": make_rays(cfg, seed, row0, rows),
             "scene_aabb": torch.tensor(SCENE_AABB, dtype=torch.float32)}
    if with_boxes and num_boxes > 0:
        batch.update(make_boxes(num_boxes, int(cfg.num_classes), int(cfg.num_instances), seed))
    return batch


def init_network_weights(net: torch.nn.Module, seed: int = 0) -> torch.nn.Module:
    """Re-draws every nn.Linear with PyTorch's default init from a fixed seed, then shifts the sigma
    bias so that accumulated opacity is non-trivial on the synthetic scene.  A hash-grid network's table is drawn
    U(-1, 1) after the linears (features of O(1)); the linears get the same values as without it."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(net.named_parameters()):
            if name.startswith("xyz_encoder."):
                continue
            if p.dim() == 2:
                bound = 1.0 / math.sqrt(p.shape[1])
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * bound)
            else:
                w = dict(net.named_parameters())[name.replace("bias", "weight")]
                bound = 1.0 / math.sqrt(w.shape[1])
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * bound)
        net.alpha_linear.bias.add_(0.1)
        enc = getattr(net, "xyz_encoder", None)
        if enc is not None:
            enc.table.copy_(torch.rand(enc.table.shape, generator=g) * 2 - 1)
    return net


# ------------------------------------------------------------------------------------------------ mesh primitives
# Closed triangle meshes of the kinds KITTI-360 annotates stuff with (DESIGN 3.2): [T,3,3] fp32 world-space vertices,
# each vertex rounded to fp32 once so that the triangles that share it share its floats (watertightness needs that).
def _tri_mesh(verts, faces) -> torch.Tensor:
    v = torch.as_tensor(verts, dtype=torch.float64).to(torch.float32)
    return v[torch.as_tensor(faces, dtype=torch.int64)].contiguous()


def icosphere_ellipsoid(center, radii, yaw: float = 0.0, subdiv: int = 2) -> torch.Tensor:
    """An icosphere (20 * 4^subdiv triangles) scaled to the semi-axes `radii`, turned by `yaw` about y."""
    p = (1.0 + math.sqrt(5.0)) / 2.0
    verts = [(-1, p, 0), (1, p, 0), (-1, -p, 0), (1, -p, 0), (0, -1, p), (0, 1, p), (0, -1, -p), (0, 1, -p),
             (p, 0, -1), (p, 0, 1), (-p, 0, -1), (-p, 0, 1)]
    verts = [tuple(c / math.sqrt(1 + p * p) for c in v) for v in verts]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
             (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
             (8, 6, 7), (9, 8, 1)]
    for _ in range(subdiv):
        mid, nf = {}, []

        def m(i, j):
            k = (min(i, j), max(i, j))
            if k not in mid:
                a, b = verts[i], verts[j]
                c = [(x + y) / 2 for x, y in zip(a, b)]
                n = math.sqrt(sum(x * x for x in c))
                verts.append(tuple(x / n for x in c))
                mid[k] = len(verts) - 1
            return mid[k]
        for a, b, c in faces:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    cy, sy = math.cos(yaw), math.sin(yaw)
    out = []
    for x, y, z in verts:
        x, y, z = x * radii[0], y * radii[1], z * radii[2]
        out.append((center[0] + cy * x + sy * z, center[1] + y, center[2] - sy * x + cy * z))
    return _tri_mesh(out, faces)


def extrusion(poly_xz, cap_faces, y0: float, y1: float) -> torch.Tensor:
    """The closed prism of a simple polygon (x, z) [n,2] between heights y0 and y1; cap_faces triangulate the polygon
    with its own vertices (no T-junctions)."""
    n = len(poly_xz)
    verts = [(x, y0, z) for x, z in poly_xz] + [(x, y1, z) for x, z in poly_xz]
    faces = [(c, b, a) for a, b, c in cap_faces] + [(a + n, b + n, c + n) for a, b, c in cap_faces]
    for i in range(n):
        j = (i + 1) % n
        faces += [(i, j, j + n), (i, j + n, i + n)]
    return _tri_mesh(verts, faces)


def u_extrusion(x0: float, z0: float, size: float, y0: float, y1: float) -> torch.Tensor:
    """A non-convex U (3 x 3 units of `size`, the notch open towards +z): a ray can leave it and re-enter it."""
    u = [(0, 0), (3, 0), (3, 3), (2, 3), (2, 1), (1, 1), (1, 3), (0, 3)]
    caps = [(0, 1, 4), (0, 4, 5), (1, 2, 4), (2, 3, 4), (0, 5, 7), (5, 6, 7)]
    return extrusion([(x0 + size * a, z0 + size * b) for a, b in u], caps, y0, y1)


def road_extrusion(segments: int = 250, width: float = 7.0, y0: float = 1.45, y1: float = 1.7, z0: float = 1.0,
                   z1: float = 63.0, seed: int = 0) -> torch.Tensor:
    """A long curved road slab under the camera: 8 * segments - 4 triangles (~2000 by default)."""
    g = torch.Generator().manual_seed(seed + 7)
    amp, ph = 2.0 + 2.0 * torch.rand((), generator=g).item(), 6.283 * torch.rand((), generator=g).item()
    left, right = [], []
    for i in range(segments):
        z = z0 + (z1 - z0) * i / (segments - 1)
        xc = amp * math.sin(z / 12.0 + ph) - amp * math.sin(ph)
        left.append((xc - width / 2, z))
        right.append((xc + width / 2, z))
    poly = left + right[::-1]                      # vertex i of left, 2K-1-i of right
    K = segments
    caps = []
    for i in range(K - 1):
        caps += [(i, i + 1, 2 * K - 2 - i), (i, 2 * K - 2 - i, 2 * K - 1 - i)]
    return extrusion(poly, caps, y0, y1)


def box_triangles(center, half, rot) -> torch.Tensor:
    """The oriented cuboid (center, half extents, rot with the box axes as columns) as 12 triangles."""
    c = torch.as_tensor(center, dtype=torch.float64)
    h = torch.as_tensor(half, dtype=torch.float64)
    r = torch.as_tensor(rot, dtype=torch.float64)
    s = torch.tensor([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)], dtype=torch.float64) * 2 - 1
    verts = c + (s * h) @ r.T
    faces = [(0, 2, 1), (1, 2, 3), (4, 5, 6), (5, 7, 6), (0, 1, 4), (1, 5, 4), (2, 6, 3), (3, 6, 7), (0, 4, 2),
             (2, 4, 6), (1, 3, 5), (3, 7, 5)]
    return _tri_mesh(verts.tolist(), faces)


def cull_box(tris: torch.Tensor):
    """(center, half, rot = I) of a world AABB padded outward until it contains every fp32 vertex of `tris`."""
    v = tris.reshape(-1, 3)
    lo, hi = v.min(0).values.double(), v.max(0).values.double()
    c = ((lo + hi) / 2).to(torch.float32)
    h = ((hi - lo) / 2).to(torch.float32)
    while True:
        lo32, hi32 = c - h, c + h
        if bool((lo32 <= v).all() and (v <= hi32).all()):
            return c, h, torch.eye(3)
        h = torch.nextafter(h * (1 + 2.0 ** -20), torch.full_like(h, float("inf")))


def mesh_table(meshes):
    """[T_b,3,3] meshes -> (mesh_tris [T,3,3], the start of each) in order."""
    starts, n = [], 0
    for m in meshes:
        starts.append(n)
        n += m.shape[0]
    return torch.cat(list(meshes), 0).contiguous(), starts


def make_mesh_primitives(num_boxes: int = 64, num_classes: int = 45, num_instances: int = 64, seed: int = 0,
                         road_segments: int = 250) -> Dict[str, torch.Tensor]:
    """`make_boxes(num_boxes)` followed by five mesh primitives - an ellipsoid, a U extrusion, the road slab under the
    camera, a cuboid given as 12 triangles and a second ellipsoid nested inside the first - with their cull boxes, plus
    the batch keys mesh_tri_start [B+1] int32 and mesh_tris [T,3,3]."""
    bx = make_boxes(num_boxes, num_classes, num_instances, seed)
    g = torch.Generator().manual_seed(seed + 11)
    j = lambda: (torch.rand((), generator=g).item() - 0.5)
    ell = icosphere_ellipsoid((-3.0 + 2 * j(), 1.0, 22.0 + 4 * j()), (3.0, 2.5, 4.0), yaw=0.3 + j())
    inner = icosphere_ellipsoid((-3.0, 1.0, 22.0), (1.0, 0.8, 1.2), yaw=0.1, subdiv=1)
    u = u_extrusion(1.0 + j(), 12.0 + 2 * j(), 2.5, -2.0, 1.4)
    road = road_extrusion(road_segments, seed=seed)
    cub = box_triangles((6.0 + j(), -1.0, 30.0 + 4 * j()), (1.5, 2.0, 2.5),
                        [[math.cos(0.4), 0.0, math.sin(0.4)], [0.0, 1.0, 0.0], [-math.sin(0.4), 0.0, math.cos(0.4)]])
    meshes = [ell, u, road, cub, inner]
    tris, starts = mesh_table(meshes)
    cb = [cull_box(m) for m in meshes]
    B0 = bx["box_center"].shape[0]
    start = torch.tensor([0] * B0 + starts + [tris.shape[0]], dtype=torch.int32)
    sem = torch.randint(0, max(num_classes, 1), (len(meshes),), generator=g, dtype=torch.int32)
    inst = torch.randint(0, max(num_instances, 1), (len(meshes),), generator=g, dtype=torch.int32)
    return dict(box_center=torch.cat([bx["box_center"], torch.stack([c for c, _, _ in cb])]).contiguous(),
                box_half=torch.cat([bx["box_half"], torch.stack([h for _, h, _ in cb])]).contiguous(),
                box_rot=torch.cat([bx["box_rot"], torch.stack([r for _, _, r in cb])]).contiguous(),
                box_sem=torch.cat([bx["box_sem"], sem]), box_inst=torch.cat([bx["box_inst"], inst]),
                mesh_tri_start=start, mesh_tris=tris)
