"""Time pnr_project_depth on KITTI-360-sized synthetic scans.

Scans: 1.2e5 points each, laid out like a Velodyne HDL-64E sweep (azimuth all around, elevation -24.8 .. +2 degrees,
range 2 .. 80 m), the sensor 1 m further along the drive per frame.  Frame sets of F = 100 frames of the 1408 x 376
perspective camera and of the 1400 x 1400 fisheye (KITTI-360's image_00 and image_02 intrinsics).  Per set, the window
w = 0 and 5 (Q = F (2w + 1) pairs) with the occlusion filter off and at r = 2: one call over the whole set, timed with
CUDA events after a warm-up, median of --reps calls.  Reports ms, points projected per second and the bytes per second
of the point reads (16 B per point and pair, as the scatter issues them; a scan shared by 2w + 1 frames is read that
many times), with the card and its power limit read in the same run, and one JSON line (also to --out FILE).
    python tools/time_project_depth.py [--reps 20] [--out FILE]"""
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
from panopticnerf_b200 import _capi  # noqa: E402

DEV = "cuda:0"
NPTS = 120000
PINHOLE = (0, 376, 1408, (552.554, 552.554, 682.049, 238.77))
FISHEYE = (2, 1400, 1400, (1336.9, 1335.6, 716.9, 705.8, 2.2134, 0.01647, 1.6035))
VELO_TO_CAM = np.array([[0, -1, 0, 0], [0, 0, -1, -0.3], [1, 0, 0, -0.8]], np.float64)   # x fwd, z up -> z fwd, y down


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


def scans(S: int, seed=0) -> torch.Tensor:
    g = torch.Generator(device=DEV).manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, device=DEV)
    az = u(S, NPTS) * 2 * np.pi
    el = np.radians(-24.8) + u(S, NPTS) * np.radians(26.8)
    r = 2 + u(S, NPTS) * 78
    pts = torch.stack([r * el.cos() * az.cos(), r * el.cos() * az.sin(), r * el.sin(), u(S, NPTS)], -1)
    return pts.reshape(-1, 4).contiguous()


def args_for(cam, F: int, w: int, radius: int, points: torch.Tensor, keep: list):
    S = F + 2 * w
    pf, ps, pm = [], [], []
    for f in range(F):
        for d in range(-w, w + 1):
            M = VELO_TO_CAM.copy()
            M[2, 3] += d * 1.0   # scan f + d was taken d metres further along the drive
            pf.append(f), ps.append(f + w + d), pm.append(M.astype(np.float32).reshape(12))
    host = [np.arange(S + 1, dtype=np.int64) * NPTS, np.array(pf, np.int32), np.array(ps, np.int32),
            np.stack(pm).astype(np.float32)]
    H, W = cam[1], cam[2]
    P = F * H * W
    fc = torch.zeros(F, dtype=torch.int32, device=DEV)
    po = torch.arange(F + 1, dtype=torch.int64, device=DEV) * (H * W)
    depth = torch.zeros(P, dtype=torch.float32, device=DEV)
    a = _capi.PnrProjectDepthArgs()
    a.points, a.Npts = points.data_ptr(), points.shape[0]
    a.scan_offset, a.S = host[0].ctypes.data, S
    a.pair_frame, a.pair_scan, a.pair_M, a.Q = host[1].ctypes.data, host[2].ctypes.data, host[3].ctypes.data, len(pf)
    a.frame_cam, a.pix_offset, a.F, a.P = fc.data_ptr(), po.data_ptr(), F, P
    a.cams[0].model, a.cams[0].H, a.cams[0].W = cam[0], H, W
    for i, x in enumerate(cam[3]):
        a.cams[0].intr[i] = x
    a.num_cameras, a.min_depth, a.max_depth = 1, 0.1, 80.0
    a.occlusion_radius, a.occlusion_margin = radius, 0.1
    a.depth = depth.data_ptr()
    need = int(_capi.lib().pnr_project_depth_workspace_bytes(P, radius))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = (ws.data_ptr(), need) if need else (None, 0)
    keep += [host, fc, po, depth, ws]
    return a, depth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_project_depth needs a GPU"
    lib = _capi.lib()
    F = args.frames
    points = scans(F + 10)
    result = {"card": card(), "points_per_scan": NPTS, "frames": F, "rows": []}
    print(f"# {result['card']}")
    print(f"{'camera':>8} {'w':>2} {'r':>2} {'pairs':>6} {'ms':>9} {'Gpts/s':>8} {'GB/s read':>10} {'covered':>8}")
    for name, cam in (("pinhole", PINHOLE), ("fisheye", FISHEYE)):
        for w in (0, 5):
            for radius in (0, 2):
                keep = []
                a, depth = args_for(cam, F, w, radius, points, keep)
                st = torch.cuda.current_stream()
                call = lambda: _capi.check(lib.pnr_project_depth(C.byref(a), st.cuda_stream), "pnr_project_depth")
                for _ in range(3):
                    call()
                times = []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    call()
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1))
                ms = float(np.median(times))
                n = a.Q * NPTS
                row = {"camera": name, "w": w, "r": radius, "pairs": a.Q, "ms": ms, "points_per_s": n / ms * 1e3,
                       "read_bytes_per_s": 16 * n / ms * 1e3, "covered": float((depth > 0).float().mean()),
                       "ms_min": float(min(times)), "ms_max": float(max(times))}
                result["rows"].append(row)
                print(f"{name:>8} {w:>2} {radius:>2} {a.Q:>6} {ms:>9.3f} {row['points_per_s'] / 1e9:>8.2f} "
                      f"{row['read_bytes_per_s'] / 1e9:>10.1f} {row['covered']:>8.3f}")
                del keep, depth
                torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
