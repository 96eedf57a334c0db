"""Time pnr_stereo_depth on KITTI-360-sized stereo pairs.

Pairs: 376 x 1408 (KITTI-360's rectified perspective size), ray-cast from textured fronto-parallel layers (a plane at
30 m, boxes at 6 m and 2.5 m) with KITTI-360's fx = 552.554 px and b = 0.6 m, written into a frame store.  For
D = 128 and 256 and n = 1 and 8 pairs per call: the ms per pair of one call, timed with CUDA events after a warm-up
(median of --reps calls); the per-kernel split of one call from torch.profiler; the HBM bytes the chosen layout moves
per pair (S accumulated by direction: 2 N D stored by the first direction, 4 N D loaded and stored by each of the
other seven, 2 N D read by the left-right pass and again by the selection, plus the census words and the images) and
their rate against the H100 SXM's 3.35 TB/s, with the card and its power limit read in the same run, and one JSON
line (also to --out FILE).
    python tools/time_stereo.py [--reps 20] [--out FILE]"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
from panopticnerf_b200 import _capi  # noqa: E402
from oracle_stereo import render_pair  # noqa: E402

DEV = "cuda:0"
H, W, FX, B = 376, 1408, 552.554, 0.6
HBM = 3.35e12


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


def layout_bytes(D: int) -> int:
    """HBM bytes per pair of the chosen layout (module docstring)."""
    N = H * W
    images = 2 * 3 * N
    census = 2 * 8 * N + 8 * 2 * 8 * N            # written once, both words read once per direction
    S = 2 * N * D + 7 * 4 * N * D + 2 * 2 * N * D
    rest = 2 * N + 2 * N + 4 * N + 2 * N          # d_R written and read, depth and disparity written
    return images + census + S + rest


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_stereo: needs a CUDA device")
    pairs = [render_pair(H, W, FX, 682.049, 238.77, B, [(30.0, None, 1 + i), (6.0, (500, 800, 100, 300), 20 + i),
                                                         (2.5, (1000, 1200, 150, 330), 40 + i)]) for i in range(8)]
    rgb8 = torch.from_numpy(np.concatenate([p[0].reshape(-1, 3) for p in pairs])).to(DEV)
    off = torch.arange(9, dtype=torch.int64, device=DEV) * (H * W)
    right = torch.from_numpy(np.stack([p[1] for p in pairs])).to(DEV)
    depth = torch.zeros(8 * H * W, dtype=torch.float32, device=DEV)
    results = []
    for D in (128, 256):
        for n in (1, 8):
            frames = np.arange(n, dtype=np.int32)
            args = _capi.PnrStereoArgs()
            args.rgb8, args.pix_offset, args.P, args.F = rgb8.data_ptr(), off.data_ptr(), rgb8.shape[0], 8
            args.frames, args.n, args.H, args.W = frames.ctypes.data, n, H, W
            args.right, args.D, args.P1, args.P2, args.U = right.data_ptr(), D, 10, 120, 10
            args.B16, args.min_depth, args.max_depth = float(np.float32(16 * FX * B)), 0.1, 40.0
            args.depth = depth.data_ptr()
            need = _capi.lib().pnr_stereo_workspace_bytes(n, H, W, D)
            ws = torch.empty(need, dtype=torch.uint8, device=DEV)
            args.workspace, args.workspace_bytes = ws.data_ptr(), need
            call = lambda: _capi.check(_capi.lib().pnr_stereo_depth(C.byref(args), _capi.stream_ptr()),
                                       "pnr_stereo_depth")
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            ms = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            call_ms = float(np.median(ms))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                call()
                torch.cuda.synchronize()
            split = {}
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA and "stereo_" in ev.name:
                    k = ev.name.split("(")[0].split("<")[0].replace("void ", "").replace("pnr::", "")
                    split[k] = split.get(k, 0.0) + ev.device_time / 1000.0
            per_pair = call_ms / n
            nb = layout_bytes(D)
            r = {"D": D, "n": n, "ms_per_call": round(call_ms, 4), "ms_per_pair": round(per_pair, 4),
                 "kernel_ms_per_call": {k: round(v, 4) for k, v in sorted(split.items())},
                 "layout_bytes_per_pair": nb, "bytes_per_s": nb / (per_pair * 1e-3),
                 "share_of_3_35_TBps": round(nb / (per_pair * 1e-3) / HBM, 3)}
            results.append(r)
            print(f"D={D:3d} n={n}: {per_pair:.3f} ms per pair ({call_ms:.3f} ms per call); layout moves "
                  f"{nb / 1e9:.2f} GB per pair = {r['bytes_per_s'] / 1e12:.2f} TB/s ({100 * r['share_of_3_35_TBps']:.0f}% "
                  f"of 3.35 TB/s); kernels per call: " + ", ".join(f"{k} {v:.3f} ms" for k, v in sorted(split.items())))
            del ws
    c = card()
    print(f"card: {c}")
    line = json.dumps({"tool": "time_stereo", "card": c, "H": H, "W": W, "results": results})
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
