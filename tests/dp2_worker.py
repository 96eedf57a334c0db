"""Worker of tests/test_gpu_data_parallel.py::test_two_ranks_hold_identical_replicas (run under torch.distributed.run,
one rank per GPU).  Each rank builds its networks from a different seed; DataParallelWrapper's broadcast must leave
identical replicas.  After 5 steps of FusedAdam over libpnr's NCCL exchange both ranks hold identical parameters and
moments.  For the frequency network they also equal, bit for bit, the one-process simulation of the same two shards.
The hash-grid table gradient is accumulated with fp32 atomics, whose order varies from run to run, so for the hash-grid
network only replica identity is asserted."""
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


def _same_on_all_ranks(tg, t):
    g = tg.allgather(t.detach().contiguous())
    return all(torch.equal(g[0].view(torch.int32), g[r].view(torch.int32)) for r in range(1, g.shape[0]))


def run(kind, tg, dev, rank):
    cfg = cfg3(kind)
    net = S.init_network_weights(PN.make_network(cfg), seed=100 + rank).to(dev)
    fine = S.init_network_weights(PN.make_network(cfg), seed=200 + rank).to(dev)
    params = lambda n, f: list(n.parameters()) + list(f.parameters())
    assert not _same_on_all_ranks(tg, params(net, fine)[0])             # seeded differently
    w = DataParallelWrapper(cfg, net, fine, device=dev, comm=tg)
    for p in params(net, fine):
        assert _same_on_all_ranks(tg, p), "the broadcast left different replicas"
    sim_net, sim_fine = copy.deepcopy(net), copy.deepcopy(fine)
    opt = FusedAdam(params(net, fine), lr=1e-3, comm=tg)
    sim_opt = FusedAdam(params(sim_net, sim_fine), lr=1e-3)
    for s in range(5):
        batch = {k: v.to(dev) for k, v in train_batch(cfg, 301, seed=40 + s, step=4).items()}
        opt.zero_grad()
        _, loss, stats, _ = w(batch)
        loss.backward()
        opt.step()
        assert _same_on_all_ranks(tg, loss) and _same_on_all_ranks(tg, stats["n_inst"])
        if kind == "frequency":
            results, stacks = simulate_shards(cfg, sim_net, sim_fine, batch, 2, sim_opt, device=dev)
            sim_opt.step_gathered(stacks)
            assert torch.equal(results[rank][1], loss.detach()), f"step {s}: loss differs from the simulation"
    for f in opt._flat:
        for k in ("param", "exp_avg", "exp_avg_sq"):
            assert _same_on_all_ranks(tg, f[k]), f"{kind}: {k} differs between the replicas"
    if kind == "frequency":
        for f, g in zip(opt._flat, sim_opt._flat):
            for k in ("param", "exp_avg", "exp_avg_sq"):
                assert torch.equal(f[k], g[k]), f"{k} differs from the one-process simulation"


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    tg = parallel.TileGather(dev)
    for kind in ("frequency", "hashgrid"):
        run(kind, tg, dev, rank)
    torch.cuda.synchronize()
    tg.close()
    dist.barrier()
    if rank == 0:
        print(f"DP2 OK world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
