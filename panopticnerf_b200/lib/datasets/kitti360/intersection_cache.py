"""Per-frame ray / primitive intersection cache.  The reference precomputes the intersections in its dataset code
and caches them on disk (SURVEY 8(f) rank 3, "bbx_intersection"; its file layout is not in the mount).  Here the
intersection stage is a 0.2 ms kernel inside the render call, so nothing needs a cache to be fast; this module keeps
the results of `pnr_intersect` in one .npz per frame for tools that want them offline (label transfer, debugging),
keyed by what they depend on so that a stale file is refused."""
from __future__ import annotations

import hashlib
from typing import Dict

import numpy as np

_FORMAT = 1


def _key(prims: Dict[str, np.ndarray], c2w: np.ndarray, intrinsics, H: int, W: int, max_hits: int) -> str:
    h = hashlib.sha256()
    for a in (prims["box_center"], prims["box_half"], prims["box_rot"], np.asarray(c2w, dtype=np.float32),
              np.asarray(intrinsics, dtype=np.float32), np.array([H, W, max_hits, _FORMAT], dtype=np.int64)):
        h.update(np.ascontiguousarray(a).tobytes())
    if "mesh_tris" in prims:      # only then: a cache of cuboids keeps its key
        for a in (np.asarray(prims["mesh_tri_start"], dtype=np.int32), np.asarray(prims["mesh_tris"], dtype=np.float32)):
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def save_intersections(path, hit_mask, box_id, t_in, t_out, prims, c2w, intrinsics, H: int, W: int) -> None:
    """hit_mask [H*W] bool, box_id [H*W,M] int32 (-1 pad), t_in / t_out [H*W,M] float32 (numpy or torch)."""
    npy = lambda a: a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    box_id = npy(box_id)
    np.savez_compressed(path, format=np.int64(_FORMAT), key=_key(prims, c2w, intrinsics, H, W, box_id.shape[1]),
                        hit_mask=np.packbits(npy(hit_mask).astype(bool)), n_rays=np.int64(H * W),
                        box_id=box_id.astype(np.int32), t_in=npy(t_in).astype(np.float32), t_out=npy(t_out).astype(np.float32))


def load_intersections(path, prims, c2w, intrinsics, H: int, W: int) -> Dict[str, np.ndarray]:
    z = np.load(path, allow_pickle=False)
    if int(z["format"]) != _FORMAT:
        raise ValueError(f"{path}: cache format {int(z['format'])}, this build reads {_FORMAT}")
    M = z["box_id"].shape[1]
    if str(z["key"]) != _key(prims, c2w, intrinsics, H, W, M):
        raise ValueError(f"{path}: stale cache (primitives, pose, intrinsics or image size differ)")
    n = int(z["n_rays"])
    return {"hit_mask": np.unpackbits(z["hit_mask"])[:n].astype(bool), "box_id": z["box_id"], "t_in": z["t_in"], "t_out": z["t_out"]}
