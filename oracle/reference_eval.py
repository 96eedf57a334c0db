"""CPU reference of the frame evaluation (pnr_eval_semantic / pnr_eval_panoptic / pnr_eval_image of include/pnr.h and
lib/evaluators).  TEST INFRASTRUCTURE ONLY (same rule as reference_renderer.py: only tests/ and tools/ may import it).

PARITY UNPINNED: the reference's evaluator is not in the mount.  The rules below are chosen in this repository
(DESIGN.md 3.4) and restated here from their definitions, in numpy / plain Python, one frame at a time:
  - ids are panoptic ids id*1000 + n; a negative id is void; dataset id d = id // 1000 maps to id_to_channel[d]
    (void past the table or for an entry outside [0, C)), or to d itself when d < C without a table;
  - semantic: conf[C, C+1] over the pixels whose gt channel is not void, column C = prediction without a channel;
  - panoptic quality (Kirillov et al. 2019) with the void / crowd handling of the COCO / Cityscapes panoptic tools:
    a gt segment of a thing class with n == 0 is a crowd region; same-channel pairs match when IoU > 0.5 with
    union = area_p + area_g - inter - |p ∩ void|; unmatched non-crowd gt -> FN; an unmatched prediction is an FP
    unless (|p ∩ void| + |p ∩ crowd of its class|) / area_p > 0.5; a frame's matched IoUs are summed with math.fsum;
  - image: per frame sum of squared rgb error and the pixel count (PSNR per frame, averaged over frames); depth: sums
    of |d|, d^2 and |d| / gt over depth_gt > 0.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import numpy as np


def channels(ids, C: int, id_to_channel: Optional[Sequence[int]] = None) -> np.ndarray:
    ids = np.asarray(ids, dtype=np.int64)
    d = np.where(ids >= 0, ids // 1000, -1)
    if id_to_channel is None:
        return np.where((d >= 0) & (d < C), d, -1)
    t = np.asarray(id_to_channel, dtype=np.int64)
    ok = (d >= 0) & (d < len(t))
    ch = np.where(ok, t[np.clip(d, 0, len(t) - 1)], -1)
    return np.where((ch >= 0) & (ch < C), ch, -1)


def semantic_confusion(pred, gt, C: int, id_to_channel=None) -> np.ndarray:
    g = channels(np.ravel(gt), C, id_to_channel)
    p = channels(np.ravel(pred), C, id_to_channel)
    keep = g >= 0
    p = np.where(p < 0, C, p)
    return np.bincount(g[keep] * (C + 1) + p[keep], minlength=C * (C + 1)).reshape(C, C + 1).astype(np.uint64)


def panoptic_frame(pred, gt, C: int, is_thing, id_to_channel=None):
    """One frame -> (tp, fp, fn int64 [C], iou_sum float64 [C])."""
    pred = np.ravel(np.asarray(pred, dtype=np.int64))
    gt = np.ravel(np.asarray(gt, dtype=np.int64))
    thing = np.asarray(is_thing, dtype=bool)
    ch = lambda i: int(channels(np.array([i]), C, id_to_channel)[0])
    gk = np.where(channels(gt, C, id_to_channel) >= 0, gt, -1)          # -1 = void
    pk = np.where(channels(pred, C, id_to_channel) >= 0, pred, -1)
    keep = (gk >= 0) | (pk >= 0)
    pairs, counts = np.unique(np.stack([gk[keep], pk[keep]], 1), axis=0, return_counts=True)

    def crowd(g):
        c = ch(g)
        return c >= 0 and bool(thing[c]) and g % 1000 == 0

    gt_area, pr_area, pr_void, pr_crowd = {}, {}, {}, {}
    for (g, p), n in zip(pairs.tolist(), counts.tolist()):
        if g >= 0:
            gt_area[g] = gt_area.get(g, 0) + n
        if p >= 0:
            pr_area[p] = pr_area.get(p, 0) + n
            if g < 0:
                pr_void[p] = pr_void.get(p, 0) + n
            elif crowd(g) and ch(g) == ch(p):
                pr_crowd[p] = pr_crowd.get(p, 0) + n
    tp, fp, fn = (np.zeros(C, dtype=np.int64) for _ in range(3))
    ious = [[] for _ in range(C)]
    matched_g, matched_p = set(), set()
    for (g, p), n in zip(pairs.tolist(), counts.tolist()):
        if g < 0 or p < 0 or ch(g) != ch(p) or crowd(g):
            continue
        union = pr_area[p] + gt_area[g] - n - pr_void.get(p, 0)
        iou = n / union
        if iou > 0.5:
            c = ch(g)
            tp[c] += 1
            ious[c].append(iou)
            matched_g.add(g)
            matched_p.add(p)
    for g in gt_area:
        if g not in matched_g and not crowd(g):
            fn[ch(g)] += 1
    for p, area in pr_area.items():
        if p in matched_p:
            continue
        if (pr_void.get(p, 0) + pr_crowd.get(p, 0)) / area > 0.5:
            continue
        fp[ch(p)] += 1
    return tp, fp, fn, np.array([math.fsum(v) for v in ious], dtype=np.float64)


def image_sums(rgb=None, rgb_gt=None, depth=None, depth_gt=None) -> np.ndarray:
    """One frame -> float64 [6] = {sum (rgb - gt)^2, pixels, sum |d|, sum d^2, sum |d| / gt, depth pixels}."""
    s = np.zeros(6, dtype=np.float64)
    if rgb is not None:
        d = np.asarray(rgb, np.float64).reshape(-1, 3) - np.asarray(rgb_gt, np.float64).reshape(-1, 3)
        s[0], s[1] = (d * d).sum(), d.shape[0]
    if depth is not None:
        g = np.ravel(np.asarray(depth_gt, np.float64))
        ok = g > 0
        d = np.ravel(np.asarray(depth, np.float64))[ok] - g[ok]
        s[2], s[3], s[4], s[5] = np.abs(d).sum(), (d * d).sum(), (np.abs(d) / g[ok]).sum(), ok.sum()
    return s


def _mean(v, m):
    return float(np.mean(v[m])) if m.any() else float("nan")


def summarize(conf, tp, fp, fn, iou_sum, is_thing, frame_sums) -> Dict[str, object]:
    """The metrics of accumulated counts (the same keys as Evaluator.summarize)."""
    conf = np.asarray(conf, np.float64)
    C = conf.shape[0]
    inter = np.diag(conf[:, :C])
    den = conf.sum(1) + conf[:, :C].sum(0) - inter
    iou = np.where(den > 0, inter / np.where(den > 0, den, 1), np.nan)
    tp, fp, fn = (np.asarray(x, np.float64) for x in (tp, fp, fn))
    iou_sum = np.asarray(iou_sum, np.float64)
    seen = tp + fp + fn > 0
    d = np.where(seen, tp + 0.5 * fp + 0.5 * fn, 1.0)
    pq = np.where(seen, iou_sum / d, np.nan)
    sq = np.where(tp > 0, iou_sum / np.where(tp > 0, tp, 1.0), 0.0)
    rq = np.where(seen, tp / d, np.nan)
    th = np.asarray(is_thing, bool)
    fs = np.asarray(frame_sums, np.float64).reshape(-1, 6)
    with np.errstate(divide="ignore"):
        psnr = [-10.0 * math.log10(r[0] / (3.0 * r[1])) if r[0] > 0 else math.inf for r in fs if r[1] > 0]
    tot = fs.sum(0)
    out = {"miou": _mean(iou, den > 0), "acc": float(inter.sum() / conf.sum()) if conf.sum() > 0 else float("nan"),
           "iou": iou.tolist(), "pq_per_class": pq.tolist(), "frames": int(fs.shape[0])}
    for name, m in (("", seen), ("_th", seen & th), ("_st", seen & ~th)):
        out["pq" + name], out["sq" + name], out["rq" + name] = _mean(pq, m), _mean(sq, m), _mean(rq, m)
    out["psnr"] = float(np.mean(psnr)) if psnr else float("nan")
    n = tot[5]
    out["depth_mae"] = tot[2] / n if n > 0 else float("nan")
    out["depth_rmse"] = math.sqrt(tot[3] / n) if n > 0 else float("nan")
    out["depth_absrel"] = tot[4] / n if n > 0 else float("nan")
    return out
