"""Evaluator of rendered frames, the reference's `lib/evaluators` plugin surface: `evaluate(output, batch)` after every
`renderer.render(batch)`, then `summarize()` once for the sequence.  All per-frame work is CUDA (pnr_eval_* of
include/pnr.h) accumulated on the device; `evaluate` only enqueues - the host reads the accumulators once, in
`summarize`.  The metric rules are chosen here (the reference's evaluator is not in the mount): include/pnr.h and
DESIGN.md 3.4.

cfg keys (all optional; read with getattr): num_classes (C, 1..64), eval_is_thing [C] (default: every class is stuff),
eval_id_to_channel [n_ids] (dataset id -> class channel or -1; default: id d < C is channel d), and the id tables of
fuse_panoptic used when the batch carries no `panoptic_pred`: eval_inst_class, eval_inst_id, eval_class_id.

Batch keys: panoptic_gt int32 [R] or [H, W] (required); panoptic_pred int32 (optional: the prediction's panoptic ids,
otherwise fused from the output's semantic / instance maps); rgb [R, 3] and depth [R] (<= 0 = no depth) as in the
training batch, compared with the output's rgb_map / depth_map when both are present."""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch

from ..visualizers import fuse_panoptic
from . import ops


def summarize_counts(conf, tp, fp, fn, iou_sum, is_thing, frame_sums) -> Dict[str, object]:
    """The sequence's metrics from host copies of the accumulators (conf [C, C+1], tp / fp / fn / iou_sum [C],
    frame_sums [F, 6]).  A metric with nothing to average over is NaN."""
    conf = np.asarray(conf, dtype=np.float64)
    C = conf.shape[0]
    inter = np.diag(conf[:, :C])
    den = conf.sum(axis=1) + conf[:, :C].sum(axis=0) - inter
    iou = np.full(C, np.nan)
    np.divide(inter, den, out=iou, where=den > 0)
    tp, fp, fn, iou_sum = (np.asarray(x, dtype=np.float64) for x in (tp, fp, fn, iou_sum))
    seen = tp + fp + fn > 0
    pq, rq, sq = np.full(C, np.nan), np.full(C, np.nan), np.zeros(C)
    np.divide(iou_sum, tp + 0.5 * fp + 0.5 * fn, out=pq, where=seen)
    np.divide(tp, tp + 0.5 * fp + 0.5 * fn, out=rq, where=seen)
    np.divide(iou_sum, tp, out=sq, where=tp > 0)
    mean = lambda v, m: float(v[m].mean()) if m.any() else math.nan
    thing = np.asarray(is_thing, dtype=bool)
    res = {"miou": mean(iou, den > 0), "acc": float(inter.sum() / conf.sum()) if conf.sum() > 0 else math.nan,
           "iou": iou.tolist(), "pq_per_class": pq.tolist()}
    for suffix, m in (("", seen), ("_th", seen & thing), ("_st", seen & ~thing)):
        res["pq" + suffix], res["sq" + suffix], res["rq" + suffix] = mean(pq, m), mean(sq, m), mean(rq, m)
    fs = np.asarray(frame_sums, dtype=np.float64).reshape(-1, ops.IMAGE_SUMS)
    rgb = fs[fs[:, 1] > 0]
    with np.errstate(divide="ignore"):
        psnr = -10.0 * np.log10(rgb[:, 0] / (3.0 * rgb[:, 1]))          # per frame (NeRF convention), then averaged
    res["psnr"] = float(psnr.mean()) if len(psnr) else math.nan
    s = fs.sum(axis=0)
    n = s[5]
    res["depth_mae"] = float(s[2] / n) if n > 0 else math.nan
    res["depth_rmse"] = math.sqrt(s[3] / n) if n > 0 else math.nan
    res["depth_absrel"] = float(s[4] / n) if n > 0 else math.nan
    res["frames"] = int(fs.shape[0])
    return res


class Evaluator:
    def __init__(self, cfg=None, num_classes: Optional[int] = None, is_thing=None, id_to_channel=None,
                 inst_class=None, inst_id=None, class_id=None):
        get = lambda v, key: v if v is not None else getattr(cfg, key, None)
        C = int(get(num_classes, "num_classes") or 0)
        if not 1 <= C <= ops.MAX_CLASSES:
            raise ValueError(f"Evaluator: num_classes={C} outside [1, {ops.MAX_CLASSES}]")
        self.C = C
        thing = get(is_thing, "eval_is_thing")
        self.is_thing = torch.zeros(C, dtype=torch.uint8) if thing is None else torch.as_tensor(thing, dtype=torch.uint8).reshape(-1)
        if self.is_thing.numel() != C:
            raise ValueError(f"Evaluator: is_thing has {self.is_thing.numel()} entries for {C} classes")
        t = get(id_to_channel, "eval_id_to_channel")
        self.id_to_channel = None if t is None else torch.as_tensor(t, dtype=torch.int32).reshape(-1)
        if self.id_to_channel is not None and self.id_to_channel.numel() == 0:
            raise ValueError("Evaluator: id_to_channel is empty")
        as_i32 = lambda v: None if v is None else torch.as_tensor(v, dtype=torch.int32).reshape(-1)
        self._fuse_tables = [as_i32(get(inst_class, "eval_inst_class")), as_i32(get(inst_id, "eval_inst_id")),
                             as_i32(get(class_id, "eval_class_id"))]
        self.device = None
        self.frames = 0

    # device state, made on the device of the first frame
    def _on(self, dev: torch.device) -> None:
        if self.device == dev:
            return
        if self.device is not None:
            raise ValueError(f"Evaluator: frames on {dev} after frames on {self.device}")
        self.device = dev
        to = lambda t: None if t is None else t.to(dev)
        self._thing, self._map = to(self.is_thing), to(self.id_to_channel)
        self._fuse_dev = [to(t) for t in self._fuse_tables]
        C = self.C
        self.conf = torch.zeros(C, C + 1, dtype=torch.int64, device=dev)
        self.tp, self.fp, self.fn = (torch.zeros(C, dtype=torch.int64, device=dev) for _ in range(3))
        self.iou_sum = torch.zeros(C, dtype=torch.float64, device=dev)
        self.frame_sums = torch.zeros(64, ops.IMAGE_SUMS, dtype=torch.float64, device=dev)
        self._ws = torch.empty(0, dtype=torch.uint8, device=dev)

    def reset(self) -> None:
        if self.device is not None:
            for t in (self.conf, self.tp, self.fp, self.fn, self.iou_sum, self.frame_sums):
                t.zero_()
        self.frames = 0

    def evaluate(self, output: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor]) -> None:
        """Accumulate one frame.  Enqueues work on the current stream; never waits for the device."""
        gt = batch["panoptic_gt"]
        if not gt.is_cuda:
            raise ValueError(f"Evaluator: panoptic_gt is on {gt.device} - the evaluator runs on CUDA tensors only (no CPU path)")
        self._on(gt.device)
        gt = gt.reshape(-1)
        pred = batch.get("panoptic_pred")
        if pred is None:
            ic, ii, ci = self._fuse_dev
            pred = fuse_panoptic(output, self._thing, ic, ii, ci)["panoptic"]
        pred = pred.reshape(-1)
        n = gt.numel()
        need = ops.workspace_bytes(n)
        if self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        ops.eval_semantic(pred, gt, self.C, self.conf, self._map)
        ops.eval_panoptic(pred, gt, self.C, self._thing, self._ws, self.tp, self.fp, self.fn, self.iou_sum, self._map)
        if self.frames == self.frame_sums.shape[0]:
            self.frame_sums = torch.cat([self.frame_sums, torch.zeros_like(self.frame_sums)])
        rgb = (output.get("rgb_map"), batch.get("rgb")) if "rgb" in batch and "rgb_map" in output else (None, None)
        depth = (output.get("depth_map"), batch.get("depth")) if "depth" in batch and "depth_map" in output else (None, None)
        if rgb[0] is not None or depth[0] is not None:
            ops.eval_image(self.frame_sums[self.frames], self._ws, rgb[0], rgb[1], depth[0], depth[1])
        self.frames += 1

    def summarize(self) -> Dict[str, object]:
        """Copies the accumulators to the host (once) and returns the sequence's metrics: miou, acc, iou [C],
        pq / sq / rq (+ _th / _st), pq_per_class [C], psnr, depth_mae / depth_rmse / depth_absrel, frames."""
        if self.device is None:
            raise ValueError("Evaluator.summarize: no frame was evaluated")
        host = [t.cpu().numpy() for t in (self.conf, self.tp, self.fp, self.fn, self.iou_sum,
                                          self.frame_sums[:self.frames])]
        return summarize_counts(*host[:5], self.is_thing.numpy(), host[5])
