"""Worker of tests/test_gpu_hashgrid_fixed.py::test_two_ranks_equal_the_one_process_simulation (run under
torch.distributed.run, one rank per GPU).  Two ranks train the hash-grid network with cfg.hash_grad = "fixed" for 5 steps
of FusedAdam over libpnr's NCCL exchange; every step's loss, and in the end every parameter and moment, equal the
one-process simulation of the same two shards bit for bit (with the fixed-point table gradient the hash-grid network
makes the claim tests/dp2_worker.py makes for the frequency network)."""
import copy
import os
import sys
from pathlib import Path

import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import panopticnerf_b200 as PN                                               # noqa: E402
from panopticnerf_b200 import parallel, synthetic as S                       # noqa: E402
from panopticnerf_b200.lib.train import DataParallelWrapper, FusedAdam       # noqa: E402
from test_gpu_data_parallel import cfg3, simulate_shards, train_batch      # noqa: E402


def run(tg, dev, rank):
    cfg = cfg3("hashgrid")
    cfg.hash_grad = "fixed"
    net = S.init_network_weights(PN.make_network(cfg), seed=100 + rank).to(dev)
    fine = S.init_network_weights(PN.make_network(cfg), seed=200 + rank).to(dev)
    params = lambda n, f: list(n.parameters()) + list(f.parameters())
    w = DataParallelWrapper(cfg, net, fine, device=dev, comm=tg)
    sim_net, sim_fine = copy.deepcopy(net), copy.deepcopy(fine)
    opt = FusedAdam(params(net, fine), lr=1e-3, comm=tg)
    sim_opt = FusedAdam(params(sim_net, sim_fine), lr=1e-3)
    for s in range(5):
        batch = {k: v.to(dev) for k, v in train_batch(cfg, 301, seed=40 + s, step=4).items()}
        opt.zero_grad()
        _, loss, _, _ = w(batch)
        loss.backward()
        opt.step()
        results, stacks = simulate_shards(cfg, sim_net, sim_fine, batch, 2, sim_opt, device=dev)
        sim_opt.step_gathered(stacks)
        assert torch.equal(results[rank][1], loss.detach()), f"step {s}: loss differs from the simulation"
    for f, g in zip(opt._flat, sim_opt._flat):
        for k in ("param", "exp_avg", "exp_avg_sq"):
            assert torch.equal(f[k].view(torch.int32), g[k].view(torch.int32)), f"{k} differs from the one-process simulation"


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    tg = parallel.TileGather(dev)
    run(tg, dev, rank)
    torch.cuda.synchronize()
    tg.close()
    dist.barrier()
    if rank == 0:
        print(f"DP2 HASHFIXED OK world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
