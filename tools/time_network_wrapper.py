"""Time one full training iteration through NetworkWrapper: coarse pass (64 perturbed samples) -> fine pass (64 + 128
importance samples) -> five loss terms -> backward into both networks -> Adam step, on cfg3 networks with a separate
fine network and 2048 rays of a synthetic frame with its primitives.  CUDA events around each step, median over the
timed steps after warm-up.  Prints the card and its power limit with the number, then runs tools/time_train_step.py
(one pass of 192 given depths, no sampler) in the same call for comparison.
    python tools/time_network_wrapper.py [n_rays] [timed_steps]"""
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN
from panopticnerf_b200 import synthetic as S
from panopticnerf_b200.lib.train import make_network_wrapper

DEV = "cuda:0"
R = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
STEPS = max(20, int(sys.argv[2]) if len(sys.argv) > 2 else 30)
WARMUP = 5


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


cfg = PN.make_cfg("cfg3", perturb=1.0, bound_by_primitives=True)
net = S.init_network_weights(PN.make_network(cfg), seed=0).to(DEV)
fine = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
wrapper = make_network_wrapper(cfg, net, fine)
opt = torch.optim.Adam(wrapper.parameters(), lr=5e-4)
rows = (R + int(cfg.W_img) - 1) // int(cfg.W_img)
batch = S.make_batch(cfg, seed=0, row0=150, rows=rows)
batch["rays"] = batch["rays"][:R].contiguous()
g = torch.Generator().manual_seed(0)
batch.update(rgb=torch.rand(R, 3, generator=g), depth=torch.rand(R, generator=g) * 40 + 5,
             pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
batch = {k: v.to(DEV) for k, v in batch.items()}

times = []
for i in range(WARMUP + STEPS):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    opt.zero_grad(set_to_none=True)
    output, loss, stats, _ = wrapper(batch)
    loss.backward()
    opt.step()
    b.record()
    torch.cuda.synchronize()
    if i >= WARMUP:
        times.append(a.elapsed_time(b))
med = sorted(times)[len(times) // 2]
N, Ni = int(cfg.N_samples), int(cfg.N_importance)
print(f"[{card()}] cfg3 NetworkWrapper iteration (separate fine net), {R} rays x ({N} + {N}+{Ni}) samples, Adam "
      f"included: median {med:.2f} ms over {STEPS} steps (min {min(times):.2f}, max {max(times):.2f}); "
      f"{R / med:.1f} k rays/s; loss {float(loss.detach()):.4f}, n_inst {int(stats['n_inst'])}")
sys.stdout.flush()
subprocess.run([sys.executable, str(ROOT / "tools" / "time_train_step.py")], check=True)
