"""Time the fused MLP kernel on 64- and 128-sample tiles, alternated, on one cfg frame's samples:
python tools/time_mlp_rows.py [preset] [precision ...] [--runs N] [key=value ...].

Both kernels run on the same context and inputs (pnr_set_mlp_rows picks the tile), one call each per round, the L2
flushed before every call; CUDA events; the median and the min .. max of N rounds (default 9) after two warm-up rounds.
The raw rows of the two kernels are compared bit for bit once.  The GPU's name, power limit and SM clock (sampled
around the timed rounds) are printed with the times.  Run it with PNR_LIB set to an ablation build of the library
(_build.build(out=..., extra_flags=["-DPNR_ABL_STREAM_ONLY"]), or -DPNR_ABL_NO_PROLOGUE, -DPNR_ABL_NO_TRUNK_EPILOGUE;
DESIGN 3.1) to take the table of where the time goes; an ablation's outputs are garbage and are not compared."""
import ast
import os
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN  # noqa: E402
from panopticnerf_b200 import _capi, synthetic as S  # noqa: E402
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P  # noqa: E402

DEV = "cuda:0"


def gpu_info():
    q = "name,power.limit,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def main():
    argv = sys.argv[1:]
    runs = 9
    if "--runs" in argv:
        i = argv.index("--runs")
        runs = int(argv[i + 1])
        del argv[i:i + 2]
    args = [a for a in argv if "=" not in a]
    over = {}
    for a in argv:
        if "=" in a:
            k, v = a.split("=", 1)
            try:
                over[k] = ast.literal_eval(v)
            except (ValueError, SyntaxError):
                over[k] = v
    if over.get("xyz_encoding") == "hashgrid":
        over.setdefault("hash_aabb", [c for corner in S.SCENE_AABB for c in corner])
    preset = args[0] if args else "cfg2"
    precs = args[1:] or ["fp16x3"]
    ablation = "PNR_LIB" in os.environ
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    print(f"gpu: {gpu_info()}  library: {os.environ.get('PNR_LIB', 'product')}", flush=True)
    for prec in precs:
        cfg = PN.make_cfg(preset, precision=prec, **over)
        net = S.init_network_weights(PN.make_network(cfg)).to(DEV)
        batch = {k: v.to(DEV) for k, v in S.make_batch(cfg).items()}
        rays = batch["rays"]
        near, far = P.scene_near_far(rays, batch["scene_aabb"], cfg.near, cfg.far)
        z = P.stratified_z(near, far, torch.linspace(0, 1, cfg.N_samples).to(DEV))
        ctx = net.pack()
        times = {64: [], 128: []}
        outs = {}
        clocks = []
        for r in range(runs + 2):
            for rows in (64, 128):
                _capi.set_mlp_rows(ctx, rows)
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                out = net.forward_rays(rays, z)
                b.record()
                torch.cuda.synchronize()
                if r >= 2:
                    times[rows].append(a.elapsed_time(b))
                if r == 0:
                    outs[rows] = out
                del out
            if r >= 2 and r % 3 == 0:
                clocks.append(gpu_info().split(",")[-1].strip())
        _capi.set_mlp_rows(ctx, 0)
        same = "not compared (ablation build)" if ablation else \
            ("bit-identical" if torch.equal(outs[64].view(torch.int32), outs[128].view(torch.int32)) else "DIFFERENT")
        tag = "" if not over else " " + " ".join(f"{k}={v}" for k, v in over.items() if k != "hash_aabb")
        for rows in (64, 128):
            t = sorted(times[rows])
            print(f"{preset}{tag} {prec:7s} {rows:3d} rows: median {t[len(t) // 2]:8.3f} ms  "
                  f"min {t[0]:8.3f}  max {t[-1]:8.3f}  ({len(t)} runs)", flush=True)
        m64, m128 = sorted(times[64])[runs // 2], sorted(times[128])[runs // 2]
        print(f"{preset}{tag} {prec:7s} 128 / 64 rows: {m128 / m64:.3f}; raw rows {same}; SM clocks sampled: "
              f"{', '.join(clocks)}", flush=True)


if __name__ == "__main__":
    main()
