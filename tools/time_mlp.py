"""Time only the fused MLP kernel on a cfg frame: python tools/time_mlp.py [preset] [precision ...] [key=value ...].

key=value pairs override cfg entries (values parsed as Python literals, else kept as strings), e.g.
`xyz_encoding=hashgrid hash_levels=16 hash_features=2 hash_log2_size=19`; a hash-grid network without `hash_aabb`
gets the synthetic scene's box.  For a hash-grid network the standalone encoder (pnr_hashgrid_encode) on the same
points is timed as well."""
import ast
import sys
from pathlib import Path
import torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN
from panopticnerf_b200 import synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P

DEV = "cuda:0"
args = [a for a in sys.argv[1:] if "=" not in a]
over = {}
for a in sys.argv[1:]:
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
flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)


def timed(fn):
    ts = []
    for i in range(9):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= 2:
            ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


for prec in precs:
    cfg = PN.make_cfg(preset, precision=prec, **over)
    net = S.init_network_weights(PN.make_network(cfg)).to(DEV)
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg).items()}
    rays = batch["rays"]
    near, far = P.scene_near_far(rays, batch["scene_aabb"], cfg.near, cfg.far)
    z = P.stratified_z(near, far, torch.linspace(0, 1, cfg.N_samples).to(DEV))
    med, best = timed(lambda: net.forward_rays(rays, z))
    tag = "" if not over else " " + " ".join(f"{k}={v}" for k, v in over.items() if k != "hash_aabb")
    print(f"{preset}{tag} mlp {prec:7s}: median {med:8.3f} ms  best {best:8.3f} ms  "
          f"{rays.shape[0] / med / 1e3:6.2f} Mrays/s", flush=True)
    if net.hashgrid:
        pts = (rays[:, None, :3] + rays[:, None, 3:] * z[..., None]).reshape(-1, 3).contiguous()
        with torch.no_grad():
            med, best = timed(lambda: net.xyz_encoder(pts))
        print(f"{preset}{tag} pnr_hashgrid_encode alone, same {pts.shape[0] / 1e6:.1f} M points: median {med:8.3f} ms  "
              f"best {best:8.3f} ms", flush=True)
