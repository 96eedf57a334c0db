"""Thin wrappers of the evaluation entry points of libpnr (include/pnr.h, pnr_eval_*): dtype / device / contiguity
checks, then one enqueue on the current stream.  Every accumulator is ADDED to (zero it first)."""
from __future__ import annotations

from typing import Optional

import torch

from ... import _capi

MAX_CLASSES = 64
IMAGE_SUMS = 6      # {sum (rgb - gt)^2, pixels, sum |d|, sum d^2, sum |d| / gt, depth pixels}


def workspace_bytes(n: int) -> int:
    return int(_capi.lib().pnr_eval_workspace_bytes(int(n)))


def _ids(t: torch.Tensor, name: str):
    return _capi.ptr(t, torch.int32, name), t.numel()


def eval_semantic(pred: torch.Tensor, gt: torch.Tensor, C: int, conf: torch.Tensor,
                  id_to_channel: Optional[torch.Tensor] = None) -> None:
    """conf [C, C+1] int64 (read as u64) += the frame's confusion counts."""
    p, n = _ids(pred, "pred")
    g, ng = _ids(gt, "gt")
    if n != ng:
        raise ValueError(f"eval_semantic: {n} predicted pixels, {ng} ground-truth pixels")
    if conf.shape != (C, C + 1):
        raise ValueError(f"eval_semantic: conf must be [{C}, {C + 1}], got {tuple(conf.shape)}")
    t = 0 if id_to_channel is None else id_to_channel.numel()
    with torch.cuda.device(gt.device):
        _capi.check(_capi.lib().pnr_eval_semantic(p, g, n, C, _capi.ptr(id_to_channel, torch.int32, "id_to_channel"), t,
                                                  _capi.ptr(conf, torch.int64, "conf"), _capi.stream_ptr()),
                    "pnr_eval_semantic")


def eval_panoptic(pred: torch.Tensor, gt: torch.Tensor, C: int, is_thing: torch.Tensor, workspace: torch.Tensor,
                  tp: torch.Tensor, fp: torch.Tensor, fn: torch.Tensor, iou_sum: torch.Tensor,
                  id_to_channel: Optional[torch.Tensor] = None) -> None:
    """tp, fp, fn [C] int64 (read as u64), iou_sum [C] float64 += the frame's panoptic tallies.  workspace: uint8 of at
    least workspace_bytes(n) bytes."""
    p, n = _ids(pred, "pred")
    g, ng = _ids(gt, "gt")
    if n != ng:
        raise ValueError(f"eval_panoptic: {n} predicted pixels, {ng} ground-truth pixels")
    t = 0 if id_to_channel is None else id_to_channel.numel()
    pt = _capi.ptr
    with torch.cuda.device(gt.device):
        _capi.check(_capi.lib().pnr_eval_panoptic(
            p, g, n, C, pt(id_to_channel, torch.int32, "id_to_channel"), t, pt(is_thing, torch.uint8, "is_thing"),
            pt(workspace, torch.uint8, "workspace"), workspace.numel(), pt(tp, torch.int64, "tp"),
            pt(fp, torch.int64, "fp"), pt(fn, torch.int64, "fn"), pt(iou_sum, torch.float64, "iou_sum"),
            _capi.stream_ptr()), "pnr_eval_panoptic")


def eval_image(frame_sums: torch.Tensor, workspace: torch.Tensor, rgb_map: Optional[torch.Tensor] = None,
               rgb_gt: Optional[torch.Tensor] = None, depth_map: Optional[torch.Tensor] = None,
               depth_gt: Optional[torch.Tensor] = None) -> None:
    """frame_sums [6] float64 += the frame's image / depth error sums (see IMAGE_SUMS)."""
    n = rgb_map.numel() // 3 if rgb_map is not None else (depth_map.numel() if depth_map is not None else 0)
    for name, t, per in (("rgb_map", rgb_map, 3), ("rgb_gt", rgb_gt, 3), ("depth_map", depth_map, 1),
                         ("depth_gt", depth_gt, 1)):
        if t is not None and t.numel() != n * per:
            raise ValueError(f"eval_image: {name} has {t.numel()} values for {n} pixels")
    if frame_sums.numel() != IMAGE_SUMS:
        raise ValueError(f"eval_image: frame_sums must hold {IMAGE_SUMS} doubles")
    f32 = lambda t, name: _capi.ptr(t, torch.float32, name)
    args = (f32(rgb_map, "rgb_map"), f32(rgb_gt, "rgb_gt"), f32(depth_map, "depth_map"), f32(depth_gt, "depth_gt"), n,
            _capi.ptr(frame_sums, torch.float64, "frame_sums"), _capi.ptr(workspace, torch.uint8, "workspace"),
            workspace.numel())
    with torch.cuda.device(frame_sums.device):
        _capi.check(_capi.lib().pnr_eval_image(*args, _capi.stream_ptr()), "pnr_eval_image")
