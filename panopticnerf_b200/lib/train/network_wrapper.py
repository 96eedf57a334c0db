"""NetworkWrapper(cfg, net, net_fine=None): one training iteration of the coarse and fine networks from a batch of rays,
in the call shape of the reference trainer (`output, loss, scalar_stats, image_stats = network_wrapper(batch);
loss.backward()`; the reference's lib/train/trainers is not in the mount).

  render_train (perturbed coarse samples -> coarse maps -> fine samples from the detached coarse weights -> fine maps,
  all with gradients) -> PanopticLoss: photometric on the fine and coarse colours, depth, 2D pseudo-label
  cross-entropy, fixed-semantic NLL and the instance term on the fine maps.

`loss.backward()` then runs pnr_losses' map gradients through pnr_composite_backward and network_backward of each
pass, so both networks (or the one shared network, twice) receive their parameter gradients."""
from __future__ import annotations

import importlib
from typing import Dict

import torch

from ..networks.renderer.panopticnerf_renderer import Renderer
from .losses import panoptic_losses

DEFAULT_MODULE = "panopticnerf_b200.lib.train.network_wrapper"


class NetworkWrapper(torch.nn.Module):
    """forward(batch) -> (output, loss, scalar_stats, image_stats).  batch: the rays and primitives `Renderer.render`
    takes, plus the targets rgb [R,3], depth [R] (<= 0 = invalid) and pseudo_label [R] (-1 = ignore; optional
    pseudo_weight [R]).  Weights cfg.w_rgb, w_depth, w_sem, w_fix, w_inst; cfg.inst_min_weight: the share of a ray's
    rendering weight its dominant primitive must hold for the ray to supervise the instance head.  The instance term
    is on when the network has instance slots and the batch carries primitives with box_inst."""

    def __init__(self, cfg, net, net_fine=None):
        super().__init__()
        self.cfg, self.net, self.net_fine = cfg, net, net_fine
        self.renderer = Renderer(cfg, net, net_fine)
        self.weights = tuple(float(getattr(cfg, k)) for k in ("w_rgb", "w_depth", "w_sem", "w_fix", "w_inst"))
        self.inst_min_weight = float(cfg.inst_min_weight)
        self.sem_is_prob = str(getattr(cfg, "sem_activation", "none")) == "softmax"

    def forward(self, batch: Dict[str, torch.Tensor]):
        output = self.renderer.render_train(batch)
        inst = "instance_map" in output and "fixed_instance_map" in output
        coarse = {"rgb_map": output["rgb_map_0"]} if "rgb_map_0" in output else None
        loss, terms = panoptic_losses(output, batch, self.weights if inst else self.weights[:4], self.sem_is_prob,
                                      out_coarse=coarse, inst_min_weight=self.inst_min_weight)
        scalar_stats = {"loss": loss.detach()}
        scalar_stats.update({k + "_loss": v.detach() for k, v in terms.items() if k not in ("n_inst", "inst_label")})
        mse = ((output["rgb_map"].detach() - batch["rgb"].to(output["rgb_map"].dtype)) ** 2).mean()
        scalar_stats["psnr"] = -10.0 * torch.log10(mse)
        if inst:
            scalar_stats["n_inst"] = terms["n_inst"]
            output["inst_label"] = terms["inst_label"]
        return output, loss, scalar_stats, {}


def make_network_wrapper(cfg, net, net_fine=None):
    """The NetworkWrapper of cfg.trainer_module (the reference's make_trainer resolves its wrapper the same way); with
    cfg.distributed set and the torch.distributed process group up, the DataParallelWrapper of this rank (train it
    with FusedAdam(wrapper.parameters(), comm=wrapper.comm))."""
    from .data_parallel import DataParallelWrapper, is_data_parallel
    if is_data_parallel(cfg) and not getattr(cfg, "trainer_module", None):
        return DataParallelWrapper(cfg, net, net_fine)
    module = importlib.import_module(getattr(cfg, "trainer_module", None) or DEFAULT_MODULE)
    return module.NetworkWrapper(cfg, net, net_fine)
