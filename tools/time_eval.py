"""Device time of Evaluator.evaluate (pnr_eval_semantic + pnr_eval_panoptic + pnr_eval_image) per frame, CUDA events,
on a cfg2-sized frame (376 x 1408) and a cfg5-sized one (1024 x 2048), with the CPU reference's time on the same
frame beside it.  Frames: blocky panoptic ids of a few hundred segments (45 classes, every other one a thing class;
some void, unmapped and crowd blocks), the prediction shifted by a few pixels with 15 % of its blocks relabelled and
3 % of its pixels given the id of a random pixel of the frame - KITTI-360-like segment counts with boundary noise.

    python tools/time_eval.py [--iters 50] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import reference_eval as RE                       # noqa: E402
from panopticnerf_b200.lib.evaluators import Evaluator        # noqa: E402

C = 45
IS_THING = np.arange(C) % 2 == 0


def frame(H, W, block, seed):
    g = np.random.default_rng(seed)
    bh, bw = block
    nby, nbx = -(-H // bh), -(-W // bw)
    d = g.integers(0, C, (nby, nbx))
    thing = IS_THING[d]
    n = np.where(thing, np.where(g.random(d.shape) < 0.1, 0, g.integers(1, 1000, d.shape)), 0)
    ids = np.where(g.random(d.shape) < 0.05, -1, d * 1000 + n)
    ids = np.where(g.random(d.shape) < 0.02, 60000, ids)
    gt = np.repeat(np.repeat(ids, bh, 0), bw, 1)[:H, :W]
    rel = np.where(g.random(d.shape) < 0.15, g.integers(0, C, d.shape) * 1000 + g.integers(0, 1000, d.shape), ids)
    pred = np.roll(np.repeat(np.repeat(rel, bh, 0), bw, 1)[:H, :W], (bh // 8, bw // 6), (0, 1))
    noise = g.random((H, W)) < 0.03                   # take the id of a random pixel: no new segments
    pred = np.where(noise, pred.ravel()[g.integers(0, H * W, (H, W))], pred)
    rgb, rgb_gt = g.random((H * W, 3), dtype=np.float32), g.random((H * W, 3), dtype=np.float32)
    depth, depth_gt = (g.random(H * W, dtype=np.float32) * 80 for _ in range(2))
    return pred.astype(np.int32), gt.astype(np.int32), rgb, rgb_gt, depth, depth_gt


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_eval.py needs a CUDA device")
    dev = "cuda:0"
    print(json.dumps({"gpu": gpu_info()}))
    for name, H, W, block in (("cfg2", 376, 1408, (24, 48)), ("cfg5", 1024, 2048, (64, 96))):
        pred, gt, rgb, rgb_gt, depth, depth_gt = frame(H, W, block, seed=H)
        out = {"rgb_map": torch.from_numpy(rgb).to(dev), "depth_map": torch.from_numpy(depth).to(dev)}
        batch = {"panoptic_pred": torch.from_numpy(pred).to(dev), "panoptic_gt": torch.from_numpy(gt).to(dev),
                 "rgb": torch.from_numpy(rgb_gt).to(dev), "depth": torch.from_numpy(depth_gt).to(dev)}
        ev = Evaluator(num_classes=C, is_thing=IS_THING)
        for _ in range(args.warmup):
            ev.evaluate(out, batch)
        torch.cuda.synchronize()
        ev.reset()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            ev.evaluate(out, batch)
        t1.record()
        torch.cuda.synchronize()
        dev_ms = t0.elapsed_time(t1) / args.iters
        s = ev.summarize()
        c0 = time.perf_counter()
        conf = RE.semantic_confusion(pred, gt, C)
        tal = RE.panoptic_frame(pred, gt, C, IS_THING)
        sums = RE.image_sums(rgb, rgb_gt, depth, depth_gt)
        cpu_ms = (time.perf_counter() - c0) * 1e3
        ref = RE.summarize(conf, *tal, IS_THING, sums[None])
        segs = len(np.unique(gt))
        print(json.dumps({"frame": name, "pixels": H * W, "gt_segments": segs, "device_ms_per_frame": round(dev_ms, 4),
                          "cpu_reference_ms_per_frame": round(cpu_ms, 1), "pq": s["pq"], "pq_reference": ref["pq"],
                          "miou": s["miou"], "miou_reference": ref["miou"], "frames_timed": s["frames"]}))


if __name__ == "__main__":
    main()
