"""DataParallelWrapper: data-parallel training whose step is the gradient of the GLOBAL batch's loss.

The loss terms are means over counted rays (colour values, rays with depth, labelled rays, rays whose dominant primitive
holds inst_min_weight of their weight), and those counts differ from shard to shard.  Averaging each rank's mean loss,
as DistributedDataParallel does, weights the rays of sparsely labelled shards more.  Here every shard normalises by the
global counts instead, so the sum of the ranks' gradients is the gradient of the whole batch's mean loss:

  1. local counts: 3R, n_depth and n_sem come from the targets alone and are all-gathered before the render;
  2. forward and losses with the global normalisers (inv_n_*); n_inst exists only after the label pass, so it is
     all-gathered on the device with the loss partials, and the instance map's gradient is scaled by
     n_inst_local / n_inst_global before the backward;
  3. backward into the flat gradient of FusedAdam;
  4. FusedAdam.step(): all-gather of the flat gradients and one pnr_adam_step per group, which sums the G slices in
     rank order, so every replica holds the same bits and a G-rank step equals its G shards run one after another.

The exchanges go through libpnr's NCCL entry points (parallel.TileGather).  Each phase is a method of its own, so a
test can run G shards in one process and stack their results itself."""
from __future__ import annotations

from typing import Dict, Sequence

import torch

from ... import parallel
from ..networks.renderer.panopticnerf_renderer import Renderer
from .losses import panoptic_losses

_TERMS = ("rgb", "depth", "sem", "fix", "inst")
# exchange vector of one rank (int32): n_inst, then the fp32 bits of the four terms' global partials, the instance term
# normalised by this shard's n_inst, and the squared colour error over the global colour count
_EXCHANGE = 7


class DataParallelWrapper(torch.nn.Module):
    """forward(batch) -> (output, loss, scalar_stats, image_stats), the call shape of NetworkWrapper, on this rank's
    contiguous shard of the global batch (parallel.shard_training_batch).  `loss`, its terms, psnr and n_inst in
    scalar_stats are the global batch's, identical on every rank; `loss.backward()` leaves this shard's part of the
    global gradient; `output` holds this shard's maps.  Train with
    FusedAdam(wrapper.parameters(), comm=wrapper.comm), whose step() sums the ranks' gradients.

    comm: parallel.TileGather (made on `device` when None; torch.distributed must be up) or an object with rank, world,
    allgather(t) -> [world, *t.shape] and broadcast(t).  At construction every replica takes rank 0's parameters."""

    def __init__(self, cfg, net, net_fine=None, device=None, comm=None):
        super().__init__()
        self.cfg, self.net, self.net_fine = cfg, net, net_fine
        self.device = torch.device(device) if device is not None else next(net.parameters()).device
        self.comm = comm if comm is not None else parallel.TileGather(self.device)
        self.rank, self.world = int(self.comm.rank), int(self.comm.world)
        self.renderer = Renderer(cfg, net, net_fine)
        self.weights = tuple(float(getattr(cfg, k)) for k in ("w_rgb", "w_depth", "w_sem", "w_fix", "w_inst"))
        self.inst_min_weight = float(cfg.inst_min_weight)
        self.sem_is_prob = str(getattr(cfg, "sem_activation", "none")) == "softmax"
        self.num_classes = (net_fine if net_fine is not None else net).C
        with torch.no_grad():
            for p in self.parameters():
                self.comm.broadcast(p.data)
                # written through data_ptr(): a network packed before the broadcast must repack from rank 0's values
                torch.autograd.graph.increment_version(p)

    # ---------------------------------------------------------------------------------------------- phases
    def shard(self, batch: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        return parallel.shard_training_batch(batch, self.rank, self.world)

    def instance_term_on(self, shard: Dict[str, torch.Tensor]) -> bool:
        """The renderer's rule for the instance maps, read from the configuration and the replicated primitives, so
        that every rank, an empty shard's included, decides the same: instance slots (cfg.num_instances > 0) and
        primitives (a non-empty box_center) that carry box_inst."""
        has_boxes = "box_center" in shard and shard["box_center"].shape[0] > 0
        return int(getattr(self.cfg, "num_instances", 0)) > 0 and has_boxes and shard.get("box_inst") is not None

    def local_counts(self, shard: Dict[str, torch.Tensor]) -> torch.Tensor:
        """[3R, n_depth, n_sem] of a shard (int32, on the device): the normalisers that the targets alone decide."""
        R = shard["rays"].shape[0]
        c = torch.zeros(3, dtype=torch.int32, device=self.device)
        c[0] = 3 * R
        if "depth" in shard:
            c[1] = (shard["depth"].to(self.device) > 0).sum()
        if "pseudo_label" in shard:
            lab = shard["pseudo_label"].to(self.device)
            c[2] = ((lab >= 0) & (lab < self.num_classes)).sum()
        return c

    def forward_local(self, shard: Dict[str, torch.Tensor], counts: Sequence[int]) -> dict:
        """Render and losses of a shard normalised by the global counts [3R, n_depth, n_sem] (host ints).  Returns the
        step's state: 'output', 'total' (differentiable, this shard's part of the global objective up to the instance
        scale that `finish` sets), 'inst' (whether the instance term is on) and 'exchange' (int32 [_EXCHANGE], this
        rank's row of the exchange)."""
        inv_n = (1.0 / max(int(counts[0]), 1), 1.0 / max(int(counts[1]), 1), 1.0 / max(int(counts[2]), 1))
        ex = torch.zeros(_EXCHANGE, dtype=torch.int32, device=self.device)
        step = {"inst_scale": torch.ones(1, dtype=torch.float32, device=self.device), "exchange": ex}
        inst = self.instance_term_on(shard)
        if shard["rays"].shape[0] == 0:       # an empty shard takes part with zero counts, partials and gradients
            step.update(output={}, total=None, inst=inst)
            return step
        output = self.renderer.render_train(shard)
        if inst != ("instance_map" in output and "fixed_instance_map" in output):
            raise RuntimeError("DataParallelWrapper: the render's instance maps disagree with instance_term_on()")
        coarse = {"rgb_map": output["rgb_map_0"]} if "rgb_map_0" in output else None
        total, terms = panoptic_losses(output, shard, self.weights if inst else self.weights[:4], self.sem_is_prob,
                                       out_coarse=coarse, inst_min_weight=self.inst_min_weight, inv_n=inv_n,
                                       inst_scale=step["inst_scale"])
        sq = ((output["rgb_map"].detach() - shard["rgb"].to(output["rgb_map"].dtype)) ** 2).sum() * inv_n[0]
        vals = [terms[k] for k in _TERMS[:4]] + [terms["inst"] if inst else sq.new_zeros(()), sq]
        ex[1:].view(torch.float32).copy_(torch.stack([v.to(torch.float32) for v in vals]))
        if inst:
            ex[0] = terms["n_inst"]
            output["inst_label"] = terms["inst_label"]
        step.update(output=output, total=total, inst=inst)
        return step

    def finish(self, step: dict, gathered: torch.Tensor):
        """(loss, scalar_stats) of a step from every rank's exchange row stacked in rank order (int32 [G, _EXCHANGE]):
        sets the instance scale n_inst_local / n_inst_global and forms the global values, identical on every rank."""
        n = gathered[:, 0]
        n_global = n.sum().to(torch.int32)
        nf = n.to(torch.float32)
        ng = n_global.to(torch.float32).clamp(min=1.0)
        step["inst_scale"].copy_((step["exchange"][0].to(torch.float32) / ng).reshape(1))
        part = gathered[:, 1:].contiguous().view(torch.float32)              # [G, 6]
        terms = part[:, :4].sum(0)
        inst_term = (part[:, 4] * (nf / ng)).sum()
        w = self.weights if step["inst"] else self.weights[:4]
        allt = torch.cat([terms, inst_term.reshape(1)])[:len(w)]
        total = (allt * torch.tensor(w, dtype=torch.float32, device=self.device)).sum()
        mse = part[:, 5].sum()
        if step["total"] is not None:        # the value is the global total; the gradient is this shard's part of it
            loss = step["total"] - step["total"].detach() + total
        else:
            loss = total.clone().requires_grad_(True)
        stats = {"loss": total}
        stats.update({k + "_loss": v for k, v in zip(_TERMS, allt.unbind(0))})
        stats["psnr"] = -10.0 * torch.log10(mse)
        if step["inst"]:
            stats["n_inst"] = n_global
        return loss, stats

    # ---------------------------------------------------------------------------------------------- the step
    def forward(self, batch: Dict[str, torch.Tensor]):
        shard = self.shard(batch)
        counts = self.comm.allgather(self.local_counts(shard)).sum(0).tolist()
        step = self.forward_local(shard, counts)
        loss, stats = self.finish(step, self.comm.allgather(step["exchange"]))
        return step["output"], loss, stats, {}


def is_data_parallel(cfg) -> bool:
    """cfg.distributed is set and the torch.distributed process group is up."""
    import torch.distributed as dist
    return bool(getattr(cfg, "distributed", False)) and dist.is_available() and dist.is_initialized()


__all__ = ["DataParallelWrapper", "is_data_parallel"]
