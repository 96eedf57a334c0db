"""Time the pieces of data-parallel training, with the card's name and power limit printed in the same run:

  1. pnr_adam_step alone (CUDA events, median of 50 launches after warm-up) at P = 1.35 M (the cfg3 coarse + fine
     networks) and P = 1.35 M + 16.8 M (plus a T = 2^19, L = 16, F = 2 hash table), for G = 1, 2, 4 and 8 gradient
     slices simulated on one GPU, with the achieved HBM bytes/s ((G + 3) reads + 3 writes of 4P) against 3.35 TB/s;
  2. one cfg3 NetworkWrapper iteration (separate fine network, 2048 rays, 64 + 128 samples) with torch.optim.Adam and
     with FusedAdam, alternated step by step within the run (median of each);
  3. with >= 2 visible GPUs, a torchrun child over every visible GPU: DataParallelWrapper + FusedAdam, the step time
     per rank and the gradient all-gather time (median over steps, per rank).
    python tools/time_data_parallel.py [--steps N] [--out FILE]"""
import argparse
import json
import os
import socket
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import panopticnerf_b200 as PN                                                # noqa: E402
from panopticnerf_b200 import synthetic as S                                  # noqa: E402
from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper             # noqa: E402
from panopticnerf_b200 import _capi                                            # noqa: E402

HBM_PEAK = 3.35e12            # H100 SXM data sheet, HBM3
R = 2048


def card(dev: int = 0) -> str:
    q = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(dev) + ", power limit unknown"


def median(xs):
    return sorted(xs)[len(xs) // 2]


def time_adam(P: int, G: int, reps: int = 50) -> dict:
    import ctypes as C
    dev = "cuda:0"
    grads = torch.randn(G, P, device=dev)
    p, m, v = torch.randn(P, device=dev), torch.zeros(P, device=dev), torch.zeros(P, device=dev)
    a = _capi.PnrAdamArgs()
    a.P, a.ld_grad, a.G, a.beta1, a.beta2, a.eps, a.weight_decay, a.step_size, a.bc2_sqrt = \
        P, P, G, 0.9, 0.999, 1e-8, 0.0, 1e-3, 0.03
    L = _capi.lib()

    def launch():
        _capi.check(L.pnr_adam_step(grads.data_ptr(), p.data_ptr(), m.data_ptr(), v.data_ptr(), C.byref(a), None,
                                    _capi.stream_ptr()), "pnr_adam_step")
    for _ in range(5):
        launch()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3)
    t = median(times)
    nbytes = (G + 3 + 3) * 4 * P
    return {"P": P, "G": G, "ms": t * 1e3, "bytes": nbytes, "TB_s": nbytes / t / 1e12, "of_peak": nbytes / t / HBM_PEAK}


def batch(cfg, seed: int):
    b = S.make_batch(cfg, seed=0, row0=150, rows=(R + int(cfg.W_img) - 1) // int(cfg.W_img))
    b["rays"] = b["rays"][:R].contiguous()
    g = torch.Generator().manual_seed(seed)
    b.update(rgb=torch.rand(R, 3, generator=g), depth=torch.rand(R, generator=g) * 40 + 5,
             pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    return b


def time_wrapper(steps: int) -> dict:
    dev = "cuda:0"
    cfg = PN.make_cfg("cfg3", perturb=1.0, bound_by_primitives=True)
    runs = {}
    for name in ("torch.optim.Adam", "FusedAdam"):
        net = S.init_network_weights(PN.make_network(cfg), seed=0).to(dev)
        fine = S.init_network_weights(PN.make_network(cfg), seed=1).to(dev)
        w = NetworkWrapper(cfg, net, fine)
        opt = (torch.optim.Adam(w.parameters(), lr=5e-4) if name == "torch.optim.Adam"
               else FusedAdam(w.parameters(), lr=5e-4))
        runs[name] = (w, opt, [])
    b = {k: v.to(dev) for k, v in batch(cfg, 0).items()}
    for i in range(5 + steps):
        for name, (w, opt, times) in runs.items():           # alternated step by step
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            opt.zero_grad()
            _, loss, _, _ = w(b)
            loss.backward()
            opt.step()
            e1.record()
            torch.cuda.synchronize()
            if i >= 5:
                times.append(e0.elapsed_time(e1))
    return {name: median(t) for name, (_, _, t) in runs.items()}


def child(steps: int):
    """One rank of the multi-GPU measurement (run under torch.distributed.run)."""
    import torch.distributed as dist
    from panopticnerf_b200 import parallel
    from panopticnerf_b200.lib.train import DataParallelWrapper
    rank, lr = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    tg = parallel.TileGather(dev)
    cfg = PN.make_cfg("cfg3", perturb=1.0, bound_by_primitives=True)
    net = S.init_network_weights(PN.make_network(cfg), seed=0).to(dev)
    fine = S.init_network_weights(PN.make_network(cfg), seed=1).to(dev)
    w = DataParallelWrapper(cfg, net, fine, comm=tg)
    opt = FusedAdam(w.parameters(), lr=5e-4, comm=tg)
    b = {k: v.to(dev) for k, v in batch(cfg, 0).items()}
    step_t, gather_t = [], []
    for i in range(5 + steps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        opt.zero_grad()
        _, loss, _, _ = w(b)
        loss.backward()
        opt.step()
        e1.record()
        torch.cuda.synchronize()
        g0, g1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g0.record()
        tg.allgather(opt.flat_grads()[0])
        g1.record()
        torch.cuda.synchronize()
        if i >= 5:
            step_t.append(e0.elapsed_time(e1))
            gather_t.append(g0.elapsed_time(g1))
    res = torch.tensor([median(step_t), median(gather_t)], device=dev)
    allr = tg.allgather(res).cpu().tolist()
    if rank == 0:
        print("DPRESULT " + json.dumps({"world": tg.world, "card": card(lr), "global_rays": R,
                                         "per_rank_ms": [{"step": s, "grad_allgather": g} for s, g in allr],
                                         "grad_bytes_received_per_rank": (tg.world - 1) * 4 * opt._flat[0]["P"]}))
    tg.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.steps)
    if not torch.cuda.is_available():
        raise SystemExit("time_data_parallel.py needs a CUDA device")
    result = {"card": card(0)}
    print(f"[{result['card']}]")
    result["adam"] = []
    for P in (1_351_394, 1_351_394 + 16 * (1 << 19) * 2):
        for G in (1, 2, 4, 8):
            r = time_adam(P, G)
            result["adam"].append(r)
            print(f"pnr_adam_step P={P} G={G}: {r['ms']:.3f} ms, {r['TB_s']:.2f} TB/s = {100 * r['of_peak']:.1f} % "
                  f"of 3.35 TB/s")
    result["wrapper_ms"] = time_wrapper(args.steps)
    print("cfg3 NetworkWrapper iteration (2048 rays, 64 + 128 samples), median ms: " +
          ", ".join(f"{k} {v:.2f}" for k, v in result["wrapper_ms"].items()))
    n = torch.cuda.device_count()
    if n >= 2:
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
                            "--master-addr", "127.0.0.1", "--master-port", str(port), __file__, "--child",
                            "--steps", str(args.steps)], capture_output=True, text=True, timeout=1800)
        line = [ln for ln in r.stdout.splitlines() if ln.startswith("DPRESULT ")]
        if r.returncode != 0 or not line:
            raise SystemExit(r.stdout[-2000:] + r.stderr[-4000:])
        result["multi_gpu"] = json.loads(line[0][len("DPRESULT "):])
        print(f"{n} GPUs: " + json.dumps(result["multi_gpu"]))
    else:
        result["multi_gpu"] = None
        print("one visible GPU: the multi-GPU step and exchange were not measured")
    print(json.dumps(result))
    if args.out:
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
