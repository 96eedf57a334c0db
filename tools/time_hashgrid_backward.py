"""Time the hash-grid table gradient on both paths: pnr_hashgrid_backward (fp32 atomics) and pnr_hashgrid_backward_fixed
(fixed-point sums; with the warp combining of the product library and without it, from a variant library built with
-DPNR_HASH_FIXED_COMBINE=0 under build/), on the same points, alternated call by call:
  * 2048 x 256 coherent training samples, the cfg2 frame's 33.9 M samples along rays, and as many random points;
  * T = 2^19 and 2^22 (L = 16, F = 2);
then the cfg3 hash-grid NetworkWrapper + FusedAdam iteration with cfg.hash_grad = "atomic" and "fixed", alternated step
by step.  CUDA events around each call, after warm-up; median, min and max.  The card and its power limit are read in
the same run.  The fixed path's outputs of the two libraries are checked to be identical bit for bit.
    python tools/time_hashgrid_backward.py [reps]"""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN                                          # noqa: E402
from panopticnerf_b200 import _build, _capi, synthetic as S             # noqa: E402
from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper      # noqa: E402

DEV = "cuda:0"
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 15
WARMUP = 3
FRAME = 33_882_112                     # the samples of one cfg2 frame (1408 x 376 rays x 64)
NOCOMBINE = ROOT / "build" / "libpnr_hashfixed_nocombine.so"


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


def variant_lib():
    """The same sources with the warp combining compiled out (built once; delete the file to rebuild)."""
    if not NOCOMBINE.exists():
        _build.build(out=NOCOMBINE, extra_flags=["-DPNR_HASH_FIXED_COMBINE=0"])
    lib = C.CDLL(str(NOCOMBINE))
    for name in ("pnr_hashgrid_backward_fixed", "pnr_hashgrid_fixed_workspace_bytes", "pnr_last_error"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = _capi.SIGNATURES[name]
    return lib


def stats(ts):
    ts = sorted(ts)
    return ts[len(ts) // 2], ts[0], ts[-1]


def fmt(name, ts, n):
    med, lo, hi = stats(ts)
    return f"    {name:<22} median {med:8.3f} ms  (min {lo:8.3f}, max {hi:8.3f})  {n / med / 1e3:8.1f} M points/s"


def alternate(fns, reps):
    """Each function once per round, in turn; CUDA events around each call; the first WARMUP rounds are dropped."""
    times = {k: [] for k in fns}
    for r in range(WARMUP + reps):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            if r >= WARMUP:
                times[k].append(a.elapsed_time(b))
    return times


def ray_points(n, seed, per_ray):
    g = torch.Generator(device=DEV).manual_seed(seed)
    R = n // per_ray
    o = torch.rand(R, 1, 3, device=DEV, generator=g) * 0.2 + 0.4
    d = torch.nn.functional.normalize(torch.randn(R, 1, 3, device=DEV, generator=g), dim=-1) * 0.4
    t = torch.linspace(0, 1, per_ray, device=DEV)
    return (o + d * t[None, :, None]).reshape(-1, 3).clamp(0, 1).contiguous()


def kernels(nc_lib):
    L, F, base, scale = 16, 2, 16.0, 1.3819
    main = _capi.lib()
    for T_log2 in (19, 22):
        for what, n, mk in (("training batch 2048 x 256 rays", 2048 * 256, lambda n: ray_points(n, 1, 256)),
                            ("cfg2 frame 33.9 M along rays", FRAME, lambda n: ray_points(n, 2, 64)),
                            ("cfg2 frame 33.9 M random", FRAME, lambda n: torch.rand(n, 3, device=DEV))):
            x = mk(n)
            n = x.shape[0]
            g = torch.randn(n, L * F, device=DEV) * 1e-4
            gt = torch.zeros(L, 1 << T_log2, F, device=DEV)
            nb = main.pnr_hashgrid_fixed_workspace_bytes(L, F, T_log2)
            ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
            args = (x.data_ptr(), n, None, g.data_ptr(), L, F, T_log2, base, scale, gt.data_ptr())
            st = _capi.stream_ptr()
            fns = {"atomic": lambda: _capi.check(main.pnr_hashgrid_backward(*args, st)),
                   "fixed (combining)": lambda: _capi.check(main.pnr_hashgrid_backward_fixed(*args, ws.data_ptr(), nb, st)),
                   "fixed (no combining)": lambda: _capi.check(nc_lib.pnr_hashgrid_backward_fixed(*args, ws.data_ptr(), nb, st))}
            outs = []
            for k in ("fixed (combining)", "fixed (no combining)"):
                gt.zero_()
                fns[k]()
                outs.append(gt.clone())
            assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "the two fixed builds differ"
            times = alternate(fns, REPS)
            print(f"  T=2^{T_log2} ({gt.numel() * 4 / 2**20:.0f} MB table, {nb / 2**20:.0f} MB workspace), {what}:")
            for k, ts in times.items():
                print(fmt(k, ts, n))
            del x, g, gt, ws, outs
            torch.cuda.empty_cache()


def training(steps):
    R = 2048
    runs = {}
    for mode in ("atomic", "fixed"):
        cfg = PN.make_cfg("cfg3", xyz_encoding="hashgrid", hash_aabb=[*S.SCENE_AABB[0], *S.SCENE_AABB[1]],
                          render_path="staged", bound_by_primitives=True, perturb=1.0, hash_grad=mode)
        net = S.init_network_weights(PN.make_network(cfg), seed=0).to(DEV)
        fine = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
        w = NetworkWrapper(cfg, net, fine)
        opt = FusedAdam(list(net.parameters()) + list(fine.parameters()), lr=5e-4)
        runs[mode] = (w, opt)
    rows = (R + int(cfg.W_img) - 1) // int(cfg.W_img)
    batch = S.make_batch(cfg, seed=0, row0=150, rows=rows)
    batch["rays"] = batch["rays"][:R].contiguous()
    g = torch.Generator().manual_seed(0)
    batch.update(rgb=torch.rand(R, 3, generator=g), depth=torch.rand(R, generator=g) * 40 + 5,
                 pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    batch = {k: v.to(DEV) for k, v in batch.items()}

    def step(mode):
        w, opt = runs[mode]
        opt.zero_grad()
        _, loss, _, _ = w(batch)
        loss.backward()
        opt.step()

    times = alternate({m: (lambda m=m: step(m)) for m in runs}, steps)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    print(f"  cfg3 hash-grid NetworkWrapper + FusedAdam iteration, separate fine network, {R} rays x ({N} + {N}+{Ni}) "
          f"samples, T=2^{int(cfg.hash_log2_size)}:")
    for k, ts in times.items():
        med, lo, hi = stats(ts)
        print(f"    hash_grad={k!r:<9} median {med:8.2f} ms  (min {lo:8.2f}, max {hi:8.2f}) over {len(ts)} steps")


if __name__ == "__main__":
    nc = variant_lib()
    print(f"[{card()}] hash-grid table gradient, L=16 F=2, {REPS} alternated calls per path after {WARMUP} warm-up rounds")
    kernels(nc)
    training(max(REPS, 20))
    print(f"[{card()}] end")
