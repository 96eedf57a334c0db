"""Float64 oracle of the instance term `pnr_losses` computes (rule chosen here, DESIGN 3.4; the reference's instance
supervision is not in the mount), written with plain torch ops so that autograd provides the reference gradient.
CPU PyTorch, test infrastructure only."""
from __future__ import annotations

import torch


def instance_labels(fixed_instance_map, inst_min_weight: float = 0.5):
    """Target slot of every ray: the lowest slot k whose fixed_instance_map[r,k] equals the row maximum, when that
    maximum is >= inst_min_weight; -1 otherwise (a NaN in the row makes the maximum NaN, a ray without primitives has
    maximum 0: neither counts)."""
    m = fixed_instance_map.max(1).values                                    # NaN propagates
    k = (fixed_instance_map == m[:, None]).to(torch.int64).argmax(1)        # first slot holding the maximum
    return torch.where(m >= inst_min_weight, k, torch.full_like(k, -1))


def instance_loss(instance_map, fixed_instance_map, inst_min_weight: float = 0.5):
    """Mean over the counted rays of lse(instance_map[r]) - instance_map[r, k].  No gradient reaches
    fixed_instance_map (the target is piecewise constant).  Returns (mean, per_ray [R] (0 where not counted),
    label [R], n counted)."""
    label = instance_labels(fixed_instance_map.detach(), inst_min_weight)
    ok = label >= 0
    n = int(ok.sum())
    ce = torch.logsumexp(instance_map, 1) - instance_map.gather(1, label.clamp(min=0)[:, None])[:, 0]
    per_ray = torch.where(ok, ce, torch.zeros_like(ce))
    return per_ray.sum() / max(n, 1), per_ray, label, n
