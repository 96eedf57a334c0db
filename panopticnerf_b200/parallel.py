"""Ray sharding across the GPUs of one box (SURVEY.md 8(e)).

Rays are independent, so the render path shards with no data-path collective: rank r renders the
contiguous ray range [r*ceil(R/G), ...) with the same kernels, and ONE all-gather of the per-ray output
maps (the reference has no collective on this path; BASELINE.json's north_star adds this one) rebuilds
the full image on every rank.  Results are bit-identical to the single-GPU render because every kernel
is deterministic and per-ray.

torch.distributed is only plumbing here (NCCL over NVLink on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import Callable, Dict, Iterable, Optional, Tuple

import torch
import torch.distributed as dist

DEFAULT_KEYS = ("rgb_map", "depth_map", "acc_map")


def shard_range(R: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous equal ranges of ceil(R/world) rays; the last ranks may be short or empty."""
    per = (R + world - 1) // world
    lo = min(rank * per, R)
    return lo, min(lo + per, R)


def shard_batch(batch: Dict[str, torch.Tensor], rank: int, world: int) -> Dict[str, torch.Tensor]:
    """Per-ray tensors (leading dim R) are sliced; scene tensors (boxes, aabb) are replicated."""
    R = batch["rays"].shape[0]
    lo, hi = shard_range(R, rank, world)
    out = {}
    for k, v in batch.items():
        per_ray = torch.is_tensor(v) and v.dim() >= 1 and v.shape[0] == R and k in (
            "rays", "near", "far", "u", "u_fine", "ray_frame")
        out[k] = v[lo:hi].contiguous() if per_ray else v
    return out


TRAIN_RAY_KEYS = ("rays", "near", "far", "u", "u_fine", "noise", "noise_fine", "rgb", "depth", "pseudo_label",
                  "pseudo_weight")
# per-ray keys that only a batch on a sequence table (kitti360.sequence_primitives) carries: sliced with the rays too
FRAME_RAY_KEYS = ("ray_frame",)
# per-ray keys that only a weighted batch (RaySampler(weights=...)) carries: sliced with the rays too
WEIGHTED_RAY_KEYS = ("importance",)


def shard_training_batch(batch: Dict[str, torch.Tensor], rank: int, world: int) -> Dict[str, torch.Tensor]:
    """A training batch's shard for data-parallel training: the rays and every per-ray target and random draw
    (TRAIN_RAY_KEYS, FRAME_RAY_KEYS, WEIGHTED_RAY_KEYS) are sliced to `shard_range`; scene tensors (primitives,
    meshes, aabb, a sequence table's frame_boxes) are replicated.  A rank past the last ray gets an empty shard (zero
    rows)."""
    R = batch["rays"].shape[0]
    lo, hi = shard_range(R, rank, world)
    out = {}
    for k, v in batch.items():
        if (k in TRAIN_RAY_KEYS or k in FRAME_RAY_KEYS or k in WEIGHTED_RAY_KEYS) and torch.is_tensor(v):
            if v.dim() < 1 or v.shape[0] != R:
                raise ValueError(f"shard_training_batch: {k} has shape {tuple(v.shape)}, expected a leading dim of R={R}")
            out[k] = v[lo:hi].contiguous()
        else:
            out[k] = v
    return out


def all_gather_maps(local: Dict[str, torch.Tensor], R: int, keys: Iterable[str] = DEFAULT_KEYS,
                    group: Optional[dist.ProcessGroup] = None) -> Dict[str, torch.Tensor]:
    """One all_gather_into_tensor of the selected per-ray maps, packed as a single [per, F] fp32 tile
    per rank (padded to ceil(R/world) rows), then unpacked to full-image tensors on every rank."""
    world = dist.get_world_size(group)
    per = (R + world - 1) // world
    keys = [k for k in keys if k in local]
    cols = [local[k].reshape(local[k].shape[0], -1).to(torch.float32) for k in keys]
    widths = [c.shape[1] for c in cols]
    n_loc = cols[0].shape[0]
    tile = torch.zeros(per, sum(widths), dtype=torch.float32, device=cols[0].device)
    if n_loc:
        tile[:n_loc] = torch.cat(cols, 1)
    full = torch.empty(world * per, sum(widths), dtype=torch.float32, device=tile.device)
    dist.all_gather_into_tensor(full, tile, group=group)
    full = full[:R]
    out, c0 = {}, 0
    for k, w in zip(keys, widths):
        shape = (R,) + tuple(local[k].shape[1:])
        out[k] = full[:, c0:c0 + w].reshape(shape).to(local[k].dtype)
        c0 += w
    return out


class TileGather:
    """The path's one exchange step through libpnr's own NCCL entry points (pnr_comm_init / pnr_allgather_outputs,
    include/pnr.h): every rank contributes one contiguous BYTE tile of its per-ray outputs and ends with all of them.

    float tiles : the selected fp32 maps, 4*F bytes per ray (rgb|depth|acc = 20 B; + logits = 4*(5+C+K) B);
    label tiles : pnr_label_tiles first - rgb as u8, depth f32, semantic / instance argmax as i16 = 11 B per ray
                  (13 with both labels) instead of 4*(5+C+K): what a consumer of the rendered image / label tiles
                  needs (north_star), ~35x fewer bytes over NVLink than the logits at cfg3 / cfg5.
    torch.distributed is used once, to hand rank 0's NCCL unique id to the other ranks.
    Data-parallel training (lib/train/data_parallel.py) uses the same communicator: `allgather` of tensors (gradients,
    counts) and `broadcast` of the start-up state."""

    def __init__(self, device, group: Optional[dist.ProcessGroup] = None):
        import ctypes as C
        from . import _capi
        self._C, self._capi = C, _capi
        self.device = torch.device(device)
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        L = _capi.lib()
        if not L.pnr_comm_available():
            raise _capi.PnrError("TileGather: libnccl.so.2 could not be loaded by libpnr")
        uid = torch.zeros(_capi.COMM_ID_BYTES, dtype=torch.uint8)
        if self.rank == 0:
            buf = (C.c_uint8 * _capi.COMM_ID_BYTES)()
            _capi.check(L.pnr_comm_unique_id(buf), "pnr_comm_unique_id")
            uid = torch.tensor(list(buf), dtype=torch.uint8)
        uid = uid.to(self.device) if dist.get_backend(group) == "nccl" else uid
        dist.broadcast(uid, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        ub = (C.c_uint8 * _capi.COMM_ID_BYTES)(*uid.cpu().tolist())
        h = C.c_void_p()
        _capi.check(L.pnr_comm_init(C.byref(h), ub, self.rank, self.world, self.device.index), "pnr_comm_init")
        self._h = h

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._capi.lib().pnr_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _gather_bytes(self, tile: torch.Tensor) -> torch.Tensor:
        """tile: contiguous uint8 [nbytes] on self.device -> [world, nbytes]."""
        full = torch.empty(self.world, tile.numel(), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            self._capi.check(self._capi.lib().pnr_allgather_outputs(
                self._h, tile.data_ptr(), full.data_ptr(), tile.numel(), self._capi.stream_ptr()),
                "pnr_allgather_outputs")
        return full

    def allgather(self, t: torch.Tensor) -> torch.Tensor:
        """[world, *t.shape] <- every rank's t (contiguous, on self.device, any dtype), in rank order; asynchronous on
        the current stream."""
        full = self._gather_bytes(t.contiguous().reshape(-1).view(torch.uint8))
        return full.view(t.dtype).reshape((self.world,) + tuple(t.shape))

    def broadcast(self, t: torch.Tensor, root: int = 0) -> torch.Tensor:
        """t (contiguous, on self.device) <- root's t, in place (pnr_broadcast)."""
        if not t.is_contiguous() or t.device != self.device:
            raise self._capi.PnrError(f"broadcast: expected a contiguous tensor on {self.device}")
        with torch.cuda.device(self.device):
            self._capi.check(self._capi.lib().pnr_broadcast(self._h, t.data_ptr(), t.numel() * t.element_size(), root,
                                                            self._capi.stream_ptr()), "pnr_broadcast")
        return t

    def gather_maps(self, local: Dict[str, torch.Tensor], R: int, keys: Iterable[str] = DEFAULT_KEYS):
        """fp32 maps (same result as all_gather_maps, through the C ABI)."""
        per = (R + self.world - 1) // self.world
        keys = [k for k in keys if k in local]
        cols = [local[k].reshape(local[k].shape[0], -1).to(torch.float32) for k in keys]
        widths = [c.shape[1] for c in cols]
        tile = torch.zeros(per, sum(widths), dtype=torch.float32, device=self.device)
        if cols[0].shape[0]:
            tile[:cols[0].shape[0]] = torch.cat(cols, 1)
        full = self._gather_bytes(tile.view(torch.uint8).reshape(-1)).view(torch.float32)
        full = full.reshape(self.world * per, sum(widths))[:R]
        out, c0 = {}, 0
        for k, w in zip(keys, widths):
            out[k] = full[:, c0:c0 + w].reshape((R,) + tuple(local[k].shape[1:])).to(local[k].dtype)
            c0 += w
        return out

    def gather_labels(self, local: Dict[str, torch.Tensor], R: int) -> Dict[str, torch.Tensor]:
        """rgb8 [R,3] u8, depth [R] f32, sem_label / inst_label [R] i16 of the whole image on every rank."""
        C, capi = self._C, self._capi
        per = (R + self.world - 1) // self.world
        n = local["rgb_map"].shape[0]
        sem, inst = local.get("semantic_map"), local.get("instance_map")
        up = lambda b: (b + 15) // 16 * 16
        seg = {"rgb8": up(per * 3), "depth": up(per * 4), "sem": up(per * 2) if sem is not None else 0,
               "inst": up(per * 2) if inst is not None else 0}
        tile = torch.zeros(sum(seg.values()), dtype=torch.uint8, device=self.device)
        off, o = {}, 0
        for k, b in seg.items():
            off[k], o = o, o + b
        base = tile.data_ptr()
        with torch.cuda.device(self.device):
            capi.check(capi.lib().pnr_label_tiles(
                capi.ptr(local["rgb_map"]), capi.ptr(local["depth_map"]), capi.ptr(sem), capi.ptr(inst), n,
                sem.shape[1] if sem is not None else 0, inst.shape[1] if inst is not None else 0,
                base + off["rgb8"], base + off["depth"], (base + off["sem"]) if sem is not None else None,
                (base + off["inst"]) if inst is not None else None, capi.stream_ptr()), "pnr_label_tiles")
        full = self._gather_bytes(tile)                                  # [world, tile bytes]
        out = {"rgb8": full[:, off["rgb8"]:off["rgb8"] + per * 3].reshape(-1, 3)[:R],
               "depth": full[:, off["depth"]:off["depth"] + per * 4].contiguous().view(torch.float32).reshape(-1)[:R]}
        if sem is not None:
            out["sem_label"] = full[:, off["sem"]:off["sem"] + per * 2].contiguous().view(torch.int16).reshape(-1)[:R]
        if inst is not None:
            out["inst_label"] = full[:, off["inst"]:off["inst"] + per * 2].contiguous().view(torch.int16).reshape(-1)[:R]
        out["bytes_per_rank"] = tile.numel()
        return out


def render_sharded(render_fn: Callable[[Dict[str, torch.Tensor]], Dict[str, torch.Tensor]],
                   batch: Dict[str, torch.Tensor], keys: Iterable[str] = DEFAULT_KEYS,
                   group: Optional[dist.ProcessGroup] = None) -> Dict[str, torch.Tensor]:
    """Render this rank's ray shard with `render_fn` (Renderer.render) and all-gather the maps."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    R = batch["rays"].shape[0]
    local = render_fn(shard_batch(batch, rank, world))
    return all_gather_maps(local, R, keys, group)
