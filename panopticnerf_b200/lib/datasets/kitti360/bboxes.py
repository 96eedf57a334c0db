"""KITTI-360 3D bounding-box annotations (data_3d_bboxes/*/<sequence>.xml) -> the primitive table of the render
path (center [B,3], half extents [B,3], rotation [B,3,3] with the box axes as columns, class id, instance id).

XML layout (public annotation format, recalled): <opencv_storage> holds one <objectN> per box with
  <transform type_id="opencv-matrix"> rows 4, cols 4, data = 16 floats, row-major  (box frame -> world: [A | T])
  <vertices  type_id="opencv-matrix"> rows 8 (or more for meshes), cols 3, in the box frame
  <faces     type_id="opencv-matrix"> rows F, cols 3: 0-based vertex indices of the triangles (mesh annotations)
  <semanticId>, <instanceId>, <timestamp> (-1: static, else the frame a dynamic box belongs to), <dynamic>
A = R diag(s): the annotation's cuboids are axis-aligned boxes of the box frame, rotated and scaled into the world.
Stuff (road, sidewalk, terrain, ...) is annotated with other shapes - ellipsoids, extruded polygons - stored as the
triangle mesh of <vertices> and <faces>; boxes_to_primitives(..., meshes=True) keeps them as meshes (DESIGN 3.2)."""
from __future__ import annotations

import xml.etree.ElementTree as ET
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np


@dataclass
class Box3D:
    name: str
    transform: np.ndarray      # 4x4, box frame -> world
    vertices: np.ndarray       # [V,3] in the box frame
    semantic_id: int
    instance_id: int
    timestamp: int = -1        # -1 = static
    dynamic: int = 0
    faces: Optional[np.ndarray] = None   # [F,3] int64 vertex indices, when the annotation has <faces>

    def world_vertices(self) -> np.ndarray:
        return self.vertices @ self.transform[:3, :3].T + self.transform[:3, 3]


def _matrix(node, what: str) -> np.ndarray:
    rows, cols = int(node.findtext("rows")), int(node.findtext("cols"))
    data = np.array(node.findtext("data").split(), dtype=np.float64)
    if data.size != rows * cols:
        raise ValueError(f"{what}: {data.size} values for a {rows}x{cols} matrix")
    return data.reshape(rows, cols)


def parse_bboxes_xml(path) -> List[Box3D]:
    root = ET.parse(str(path)).getroot()
    out = []
    for obj in root:
        if obj.find("transform") is None:
            continue
        tr, vt = _matrix(obj.find("transform"), f"{obj.tag}/transform"), _matrix(obj.find("vertices"), f"{obj.tag}/vertices")
        if tr.shape != (4, 4) or vt.shape[1] != 3:
            raise ValueError(f"{path}: {obj.tag}: transform {tr.shape}, vertices {vt.shape}")
        gi = lambda k, d: int(float(obj.findtext(k))) if obj.findtext(k) not in (None, "") else d
        faces = None
        if obj.find("faces") is not None:
            fc = _matrix(obj.find("faces"), f"{obj.tag}/faces")
            if fc.shape[1] != 3 or np.any(fc != np.round(fc)):
                raise ValueError(f"{path}: {obj.tag}: faces {fc.shape} must be integer triangles")
            faces = fc.astype(np.int64)
        out.append(Box3D(obj.tag, tr, vt, gi("semanticId", -1), gi("instanceId", -1), gi("timestamp", -1), gi("dynamic", 0),
                         faces))
    return out


def _is_cuboid(b: Box3D, ortho: bool) -> bool:
    """An orthogonal transform and 8 vertices that are the corners of their box-frame bounds."""
    v = b.vertices
    if not ortho or v.shape[0] != 8:
        return False
    lo, hi = v.min(0), v.max(0)
    on = (v == lo) | (v == hi)
    corners = {tuple(v[i] == hi) for i in range(8)}
    return bool(on.all()) and len(corners) == 8


def _check_closed(b: Box3D) -> None:
    """Refuse faces outside [0, V) and, after welding equal vertices, any edge not shared by exactly two faces."""
    V = b.vertices.shape[0]
    if b.faces is None:
        raise ValueError(f"{b.name}: a non-cuboid annotation needs <faces> to be a mesh primitive")
    f = b.faces
    if f.size == 0 or f.min() < 0 or f.max() >= V:
        raise ValueError(f"{b.name}: face index outside [0, {V}) (min {f.min() if f.size else '-'}, max "
                         f"{f.max() if f.size else '-'}); faces are 0-based")
    _, weld = np.unique(b.vertices, axis=0, return_inverse=True)
    w = weld.reshape(-1)[f]
    edges = np.sort(np.concatenate([w[:, [0, 1]], w[:, [1, 2]], w[:, [2, 0]]]), 1)
    if np.any(edges[:, 0] == edges[:, 1]):
        raise ValueError(f"{b.name}: degenerate face (a repeated vertex): not a closed manifold mesh")
    _, count = np.unique(edges, axis=0, return_counts=True)
    if np.any(count != 2):
        raise ValueError(f"{b.name}: open or non-manifold mesh ({int((count != 2).sum())} edges not shared by exactly "
                         "two faces)")


def _pad_to_contain(c, h, R, pts):
    """Half extents h (float32) grown until the box (c, h, R) contains every point of pts [n,3] (float64 check)."""
    c64, R64 = c.astype(np.float64), R.astype(np.float32).astype(np.float64)
    h = h.astype(np.float32)
    for _ in range(64):
        if np.all(np.abs((pts - c64) @ R64) <= h.astype(np.float64)):
            return h
        h = np.nextafter(h * np.float32(1 + 2.0 ** -20), np.float32(np.inf)).astype(np.float32)
    raise ValueError("cull box: cannot contain the mesh")   # unreachable for finite vertices


def boxes_to_primitives(boxes: Iterable[Box3D], frame: Optional[int] = None, ortho_tol: float = 1e-3,
                        meshes: bool = False) -> Dict[str, np.ndarray]:
    """Static boxes (+ the dynamic ones stamped `frame`) as oriented cuboids.  Per box, with [lo, hi] the bounds of
    its vertices in the box frame and A the 3x3 of its transform: s_j = |A[:, j]|, rot = A / s (a reflection is
    removed by flipping the last axis - a cuboid does not care), half = (hi - lo)/2 * s, center = A (lo + hi)/2 + T.
    A box whose axes are not orthogonal within `ortho_tol` is rejected (the slab test needs a rotation).

    meshes=True: an annotation stays a cuboid when its transform is orthogonal and its 8 vertices are the corners of
    their box-frame bounds; every other one becomes a mesh primitive (its triangles in world coordinates, each vertex
    transformed in float64 and rounded to fp32 once, so that the triangles sharing it share its floats), whose box is
    a cull volume - the box-frame bounds above when the transform is orthogonal, else the world AABB - padded outward
    until it contains every fp32 vertex.  A mesh without <faces>, with a face index outside [0, V), or open /
    non-manifold is refused by name.  The result then also has mesh_tri_start [B+1] int32 and mesh_tris [T,3,3]
    float32 (primitive b owns triangles [start[b], start[b+1]); cuboids own none) when there is a mesh."""
    c, h, r, sem, inst, names = [], [], [], [], [], []
    tris, start = [], [0]
    for b in boxes:
        if b.timestamp != -1 and (frame is None or b.timestamp != frame):
            continue
        A, T = b.transform[:3, :3], b.transform[:3, 3]
        s = np.linalg.norm(A, axis=0)
        if np.any(s <= 0):
            raise ValueError(f"{b.name}: degenerate transform")
        R = A / s
        ortho = bool(np.abs(R.T @ R - np.eye(3)).max() <= ortho_tol)
        mesh = meshes and not _is_cuboid(b, ortho)
        if not ortho and not mesh:
            raise ValueError(f"{b.name}: transform axes are not orthogonal (max |R^T R - I| = {np.abs(R.T @ R - np.eye(3)).max():.2e})")
        if ortho and np.linalg.det(R) < 0:
            R = R * np.array([1.0, 1.0, -1.0])
        lo, hi = b.vertices.min(0), b.vertices.max(0)
        if ortho:
            ci, hi_ = A @ ((lo + hi) * 0.5) + T, (hi - lo) * 0.5 * s
        if mesh:
            _check_closed(b)
            wv = b.world_vertices().astype(np.float32)
            if not ortho:
                wlo, whi = wv.astype(np.float64).min(0), wv.astype(np.float64).max(0)
                ci, hi_, R = (wlo + whi) * 0.5, (whi - wlo) * 0.5, np.eye(3)
            ci32 = np.asarray(ci, dtype=np.float32)
            hi_ = _pad_to_contain(ci32, np.asarray(hi_, dtype=np.float32), np.asarray(R, dtype=np.float32),
                                  wv.astype(np.float64))
            tris.append(wv[b.faces])
        c.append(ci)
        h.append(hi_)
        r.append(R)
        start.append(start[-1] + (b.faces.shape[0] if mesh else 0))
        sem.append(b.semantic_id)
        inst.append(b.instance_id)
        names.append(b.name)
    n = len(c)
    out = {"box_center": np.asarray(c, dtype=np.float32).reshape(n, 3), "box_half": np.asarray(h, dtype=np.float32).reshape(n, 3),
           "box_rot": np.asarray(r, dtype=np.float32).reshape(n, 3, 3), "box_sem": np.asarray(sem, dtype=np.int32),
           "box_inst": np.asarray(inst, dtype=np.int32), "names": names}
    if tris:
        out["mesh_tri_start"] = np.asarray(start, dtype=np.int32)
        out["mesh_tris"] = np.ascontiguousarray(np.concatenate(tris, 0), dtype=np.float32)
    return out


def sequence_primitives(boxes: Iterable[Box3D], frame_ids: Sequence[int], ortho_tol: float = 1e-3,
                        meshes: bool = False) -> Dict[str, np.ndarray]:
    """One primitive table for the rays of many frames (DESIGN 3.2): the static boxes (boxes_to_primitives(frame=None))
    at ids [0, S), then one block of dynamic boxes per distinct timestamp among `frame_ids`, in order of first
    appearance.  Adds static_boxes = S and frame_boxes [F,2] int32, row f = (begin, end) of frame_ids[f]'s block
    (frames of one timestamp share it; a frame without dynamic boxes has an empty range).  A ray of frame f meets
    [0, S) and its frame's block (include/pnr.h pnr_intersect_frames), which equals boxes_to_primitives(frame=
    frame_ids[f]) up to the order of the boxes.  With a FrameSet: frame_ids = [fid for _, fid in frames.names]."""
    boxes = list(boxes)
    fids = [int(f) for f in frame_ids]
    parts = [boxes_to_primitives(boxes, None, ortho_tol, meshes)]
    begin, where = {}, parts[0]["box_center"].shape[0]
    for t in fids:
        if t in begin:
            continue
        part = boxes_to_primitives([b for b in boxes if b.timestamp == t != -1], t, ortho_tol, meshes)
        begin[t] = (where, where + part["box_center"].shape[0])
        where += part["box_center"].shape[0]
        parts.append(part)
    out = {k: np.concatenate([p[k] for p in parts], 0) for k in ("box_center", "box_half", "box_rot", "box_sem", "box_inst")}
    out["names"] = [n for p in parts for n in p["names"]]
    if any("mesh_tris" in p for p in parts):
        start, tris = [0], []
        for p in parts:
            n = p["box_center"].shape[0]
            own = np.diff(p["mesh_tri_start"]) if "mesh_tris" in p else np.zeros(n, dtype=np.int64)
            start += (start[-1] + np.cumsum(own)).tolist()
            if "mesh_tris" in p:
                tris.append(p["mesh_tris"])
        out["mesh_tri_start"] = np.asarray(start, dtype=np.int32)
        out["mesh_tris"] = np.ascontiguousarray(np.concatenate(tris, 0), dtype=np.float32)
    out["static_boxes"] = int(parts[0]["box_center"].shape[0])
    out["frame_boxes"] = np.asarray([begin[t] for t in fids], dtype=np.int32).reshape(len(fids), 2)
    return out


def primitive_batch(prims: Dict[str, np.ndarray], sem_to_train: Optional[Dict[int, int]] = None,
                    inst_to_slot: Optional[Dict[int, int]] = None, device="cuda") -> Dict[str, "object"]:
    """The primitive block of a render batch (torch tensors on `device`).  `sem_to_train` maps KITTI-360 semanticIds
    to the network's class channels, `inst_to_slot` instanceIds to its instance channels; boxes whose id has no
    channel get -1 (they still bound samples, they just do not vote in the fixed maps).  The mesh table
    (mesh_tri_start, mesh_tris) and a sequence table's frame_boxes (int32 tensor) and static_boxes (int) are carried
    along when the primitives have them."""
    import torch
    sem = np.array([(sem_to_train or {}).get(int(s), int(s) if sem_to_train is None else -1) for s in prims["box_sem"]], dtype=np.int32)
    inst = np.array([(inst_to_slot or {}).get(int(s), int(s) if inst_to_slot is None else -1) for s in prims["box_inst"]], dtype=np.int32)
    t = lambda a, dt: torch.as_tensor(a, dtype=dt).to(device)
    return {"box_center": t(prims["box_center"], torch.float32), "box_half": t(prims["box_half"], torch.float32),
            "box_rot": t(prims["box_rot"], torch.float32), "box_sem": t(sem, torch.int32), "box_inst": t(inst, torch.int32),
            **({"mesh_tri_start": t(prims["mesh_tri_start"], torch.int32), "mesh_tris": t(prims["mesh_tris"], torch.float32)}
               if "mesh_tris" in prims else {}),
            **({"frame_boxes": t(prims["frame_boxes"], torch.int32), "static_boxes": int(prims["static_boxes"])}
               if "frame_boxes" in prims else {})}
