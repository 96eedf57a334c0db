"""Time the weighted draws: building a weight table and drawing from it.

1. pnr_pixel_weights (frame balance + class balance, labels read) and pnr_pixel_cdf on time_ray_batch.py's 64-frame
   set of cfg2-sized frames (33.9 M pixels), and pnr_pixel_cdf alone on P = 2^31 + 3 pixels when the card has the
   memory: CUDA events, median of repeated calls, with the bytes each call needs to move (weights: label 2 B read +
   weight 2 B written per pixel; cdf: weight 2 B read twice + group sums 0.25 B written per pixel) and the rate they
   make against 3.35 TB/s.
2. pnr_sample_ray_batch, weighted against uniform, alternated, at R = 2048 .. 2^20 rays (64 + 128 jitter words).
3. One cfg3 NetworkWrapper + FusedAdam iteration (2048 rays) fed by a weighted and by a uniform RaySampler, alternated.
Prints the card and its power limit with the numbers, and one JSON line (also written to --out FILE when given).
    python tools/time_pixel_weights.py [--steps 30] [--out FILE]"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import panopticnerf_b200 as PN
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.datasets.ray_batch import RaySampler, fill_frame_store, pixel_weights, sample_ray_batch
from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper
from time_ray_batch import card, frame_set

DEV = "cuda:0"
HBM = 3.35e12


def events(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def cdf_call(weight):
    P = weight.numel()
    L = _capi.lib()
    cum = torch.empty((P + 31) // 32, dtype=torch.uint64, device=DEV)
    tot = torch.empty(2, dtype=torch.uint64, device=DEV)
    ws = torch.empty(L.pnr_pixel_cdf_workspace_bytes(P), dtype=torch.uint8, device=DEV)

    def run():
        _capi.check(L.pnr_pixel_cdf(weight.data_ptr(), P, cum.data_ptr(), tot.data_ptr(), ws.data_ptr(), ws.numel(),
                                    _capi.stream_ptr()), "pnr_pixel_cdf")
    return run


def weights_call(pw_args):
    L = _capi.lib()
    return lambda: _capi.check(L.pnr_pixel_weights(C.byref(pw_args), _capi.stream_ptr()), "pnr_pixel_weights")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cfg = PN.make_cfg("cfg3", perturb=1.0, bound_by_primitives=True)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    fs = frame_set(PN.make_cfg("cfg2", num_classes=45))
    P = fs.num_pixels
    who = card()
    result = {"card": who, "frames": fs.num_frames, "pixels": P, "N": N, "Ni": Ni}
    print(f"[{who}] weight tables over {fs.num_frames} frames, {P / 1e6:.1f} M pixels")

    # 1. the builders: a table with frame and class balance, timed through the C entry points with fixed arguments
    pw = pixel_weights(fs, balance_frames=True, class_alpha=0.5)
    a = _capi.PnrPixelWeightsArgs()
    fill_frame_store(a, fs, "time")
    ff = torch.ones(fs.num_frames, device=DEV)
    cf = torch.rand(int(fs.label.max()) + 2, device=DEV) + 0.5
    a.label, a.C, a.frame_factor, a.class_factor, a.scale = fs.label.data_ptr(), cf.numel() - 1, ff.data_ptr(), cf.data_ptr(), 30000.0
    out = torch.empty(P, dtype=torch.uint16, device=DEV)
    a.weight = out.data_ptr()
    ms_w = events(weights_call(a), 50)
    ms_c = events(cdf_call(pw.weight), 50)
    bw, bc = 4 * P, 4 * P + 8 * ((P + 31) // 32)
    result["pixel_weights"] = {"ms": ms_w, "bytes": bw, "TB_per_s": bw / ms_w / 1e9, "of_peak": bw / ms_w / 1e-3 / HBM}
    result["pixel_cdf"] = {"ms": ms_c, "bytes": bc, "TB_per_s": bc / ms_c / 1e9, "of_peak": bc / ms_c / 1e-3 / HBM}
    for k, ms, b in (("pnr_pixel_weights", ms_w, bw), ("pnr_pixel_cdf", ms_c, bc)):
        print(f"  {k:18s}: {ms * 1e3:8.1f} us, {b / 1e6:6.1f} MB moved, {b / ms / 1e9:5.2f} TB/s "
              f"({100 * b / ms / 1e-3 / HBM:4.1f} % of 3.35 TB/s)")
    Pbig = (1 << 31) + 3
    if torch.cuda.mem_get_info(DEV)[0] > 2 * Pbig + Pbig // 4 + (4 << 30):
        big = torch.zeros(Pbig, dtype=torch.int16, device=DEV)
        big[:: 977] = 3
        big = big.view(torch.uint16)
        ms_b = events(cdf_call(big), 10)
        bb = 4 * Pbig + 8 * ((Pbig + 31) // 32)
        result["pixel_cdf_2e31"] = {"ms": ms_b, "bytes": bb, "TB_per_s": bb / ms_b / 1e9, "of_peak": bb / ms_b / 1e-3 / HBM}
        print(f"  pnr_pixel_cdf at P = 2^31 + 3: {ms_b:8.2f} ms, {bb / ms_b / 1e9:5.2f} TB/s "
              f"({100 * bb / ms_b / 1e-3 / HBM:4.1f} % of 3.35 TB/s)")
        del big
        torch.cuda.empty_cache()
    sys.stdout.flush()

    # 2. the draw, weighted against uniform, alternated
    result["draw"] = []
    for R in [2048 << k for k in range(10)]:
        reps = 40 if R <= 1 << 17 else 16
        times = {"weighted": [], "uniform": []}
        for i in range(3 + 2 * reps):
            kind = "weighted" if i % 2 == 0 else "uniform"
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            sample_ray_batch(fs, 1, i, 0, R, N, Ni, weights=pw if kind == "weighted" else None)
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                times[kind].append(e0.elapsed_time(e1))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        result["draw"].append({"R": R, "weighted_ms": med["weighted"], "uniform_ms": med["uniform"]})
        print(f"  draw R = {R:8d}: weighted {med['weighted'] * 1e3:9.1f} us, uniform {med['uniform'] * 1e3:9.1f} us")
    sys.stdout.flush()

    # 3. one cfg3 iteration fed by each sampler
    net = S.init_network_weights(PN.make_network(cfg), seed=0).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
    wrapper = NetworkWrapper(cfg, net, fine)
    opt = FusedAdam(list(net.parameters()) + list(fine.parameters()), lr=5e-4)
    scene = {k: v.to(DEV) for k, v in S.make_boxes(64, 45, 64, seed=0).items()}
    scene["scene_aabb"] = torch.tensor(S.SCENE_AABB, dtype=torch.float32, device=DEV)
    samplers = {"weighted": RaySampler(fs, seed=0, scene=scene, weights=pw), "uniform": RaySampler(fs, seed=0, scene=scene)}
    R = 2048
    times = {"weighted": [], "uniform": []}
    for i in range(5 + 2 * args.steps):
        kind = "weighted" if i % 2 == 0 else "uniform"
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        batch = samplers[kind].batch(i, R, N, Ni)
        opt.zero_grad()
        _, loss, _, _ = wrapper(batch)
        loss.backward()
        opt.step()
        e1.record()
        torch.cuda.synchronize()
        if i >= 5:
            times[kind].append(e0.elapsed_time(e1))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    result["iteration_ms"] = med
    print(f"[{who}] cfg3 NetworkWrapper + FusedAdam iteration, {R} rays, alternated over {args.steps} steps each: "
          f"weighted draw median {med['weighted']:.2f} ms, uniform draw median {med['uniform']:.2f} ms")
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
