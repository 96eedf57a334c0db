"""Time pnr_sample_ray_batch and what it adds to a training iteration.

1. The kernel alone: CUDA events around R = 2048 .. 2^20 rays (64 + 128 jitter words per ray, cfg3's N and Ni) drawn
   from a 64-frame set of cfg2-sized frames (376 x 1408 pinhole, rgb8 + label + depth: 33.9 M pixels), median of
   repeated launches after a warm-up, with the bytes written per launch and the rate they make.
2. One cfg3 NetworkWrapper + FusedAdam iteration (separate fine network, 2048 rays, 64 + 128 samples, 64 primitives)
   fed by RaySampler.batch(step, ...), alternated step by step with the same iteration on a batch built before the
   loop; medians of both.
Prints the card and its power limit with the numbers, and one JSON line (also written to --out FILE when given).
    python tools/time_ray_batch.py [--steps 30] [--out FILE]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN
from panopticnerf_b200 import synthetic as S
from panopticnerf_b200.lib.datasets.ray_batch import Camera, FrameSet, RaySampler, sample_ray_batch
from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper

DEV = "cuda:0"


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


def frame_set(cfg, F=64) -> FrameSet:
    H, W = int(cfg.H), int(cfg.W_img)
    P = F * H * W
    g = torch.Generator(device=DEV).manual_seed(0)
    c2w = torch.zeros(F, 3, 4)
    c2w[:, :3, :3] = torch.eye(3)
    c2w[:, 2, 3] = torch.arange(F) * 0.25              # a camera driving forward through the synthetic scene
    c2w[:, 1, 3] = 1.0
    return FrameSet([Camera("pinhole", H, W, (cfg.fx, cfg.fy, cfg.cx, cfg.cy))], c2w.reshape(F, 12).to(DEV),
                    torch.zeros(F, dtype=torch.int32, device=DEV),
                    torch.arange(F + 1, dtype=torch.int64, device=DEV) * (H * W),
                    torch.randint(0, 256, (P, 3), dtype=torch.uint8, device=DEV, generator=g),
                    torch.randint(-1, int(cfg.num_classes), (P,), device=DEV, generator=g).to(torch.int16),
                    torch.rand(P, device=DEV, generator=g) * 60)


def time_kernel(fs, R, N, Ni, reps):
    for _ in range(3):
        sample_ray_batch(fs, 1, 0, 0, R, N, Ni)
    times = []
    for i in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        sample_ray_batch(fs, 1, i, 0, R, N, Ni)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cfg = PN.make_cfg("cfg3", perturb=1.0, bound_by_primitives=True)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    fs = frame_set(PN.make_cfg("cfg2", num_classes=45))
    who = card()
    result = {"card": who, "frames": fs.num_frames, "pixels": fs.num_pixels, "N": N, "Ni": Ni, "kernel": []}
    print(f"[{who}] pnr_sample_ray_batch over {fs.num_frames} frames, {fs.num_pixels / 1e6:.1f} M pixels, "
          f"N = {N}, Ni = {Ni}")
    for R in [2048 << k for k in range(10)]:
        ms = time_kernel(fs, R, N, Ni, reps=50 if R <= 1 << 17 else 20)
        nbytes = R * 4 * (6 + 3 + 1 + 1 + N + Ni)     # rays, rgb, depth, pseudo_label, u, u_fine
        result["kernel"].append({"R": R, "ms": ms, "GB_per_s_written": nbytes / ms / 1e6})
        print(f"  R = {R:8d}: {ms * 1e3:9.1f} us  ({R / ms / 1e6:7.2f} G rays/s, {nbytes / ms / 1e6:7.1f} GB/s written)")
    sys.stdout.flush()

    net = S.init_network_weights(PN.make_network(cfg), seed=0).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
    wrapper = NetworkWrapper(cfg, net, fine)
    opt = FusedAdam(list(net.parameters()) + list(fine.parameters()), lr=5e-4)
    scene = {k: v.to(DEV) for k, v in S.make_boxes(64, 45, 64, seed=0).items()}
    scene["scene_aabb"] = torch.tensor(S.SCENE_AABB, dtype=torch.float32, device=DEV)
    sampler = RaySampler(fs, seed=0, scene=scene)
    R = 2048
    fixed = {k: v.clone() for k, v in sampler.batch(10 ** 6, R, N, Ni).items()}
    times = {"sampled": [], "prebuilt": []}
    for i in range(5 + 2 * args.steps):
        kind = "sampled" if i % 2 == 0 else "prebuilt"
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        batch = sampler.batch(i, R, N, Ni) if kind == "sampled" else fixed
        opt.zero_grad()
        _, loss, _, _ = wrapper(batch)
        loss.backward()
        opt.step()
        b.record()
        torch.cuda.synchronize()
        if i >= 5:
            times[kind].append(a.elapsed_time(b))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    result["iteration_ms"] = med
    print(f"[{who}] cfg3 NetworkWrapper + FusedAdam iteration, {R} rays, alternated over {args.steps} steps each: "
          f"sampled batch median {med['sampled']:.2f} ms, pre-built batch median {med['prebuilt']:.2f} ms "
          f"(difference {med['sampled'] - med['prebuilt']:+.2f} ms)")
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
