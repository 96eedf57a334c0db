"""One launch of every HBM-bound stage at the cfg2 frame size (for captures of achieved DRAM throughput with torch.profiler)."""
import sys
from pathlib import Path
import torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN
from panopticnerf_b200 import synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
dev = "cuda:0"
cfg = PN.make_cfg("cfg2")
batch = {k: v.to(dev) for k, v in S.make_batch(cfg).items()}
rays = batch["rays"]
R, N = rays.shape[0], cfg.N_samples
for it in range(2):
    rays2 = P.generate_rays(cfg.H, cfg.W_img, (cfg.fx, cfg.fy, cfg.cx, cfg.cy), torch.eye(4)[:3], device=dev)
    near, far = P.scene_near_far(rays, batch["scene_aabb"], cfg.near, cfg.far)
    hit, bid, tin, tout = P.intersect(rays, batch["box_center"], batch["box_half"], batch["box_rot"], 4)
    z, sb = P.stratified_z(near, far, torch.linspace(0, 1, N).to(dev), 0.0, None, bid, tin, tout, want_tags=True)
    raw = torch.randn(R, N, 4, device=dev)
    out = P.raw2outputs(raw, z, rays)
    w = out["weights"]
    zf, zall = P.sample_pdf(z, w, 128)
    x = torch.rand(4_000_000, 3, device=dev) * 60
    e = P.embed(x, 10)
    raw113 = torch.randn(100_000, N, 113, device=dev)
    o2 = P.raw2outputs(raw113, z[:100_000].contiguous(), rays[:100_000].contiguous(), num_classes=45, num_instances=64)
    torch.cuda.synchronize()
print("ok")
