"""CPU oracle of the loss terms `pnr_losses` computes (SURVEY 8(f) rank 2).  TEST INFRASTRUCTURE ONLY.
PARITY UNPINNED: the reference's NetworkWrapper is not in the mount; the terms are the paper's (photometric MSE on the
fine and coarse colours, L1 depth on valid stereo depth, cross-entropy of the rendered semantics against 2D pseudo
labels, negative log-likelihood of the fixed bounding-primitive semantics), written with plain torch ops so that
autograd provides the reference gradients."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F


def losses(rgb_map, rgb_map0, depth_map, semantic_map, fixed_semantic_map, rgb_gt, depth_gt, label, label_weight=None,
           weights=(1.0, 0.1, 1.0, 1.0), sem_is_prob: bool = False, eps: float = 1e-8):
    """Returns (total, terms[4]) with terms = (rgb, depth, sem, fix) means."""
    ref = next(t for t in (rgb_map, depth_map, semantic_map, fixed_semantic_map) if t is not None)
    R, dt = ref.shape[0], ref.dtype
    zero = torch.zeros((), dtype=dt)
    l_rgb = zero
    if rgb_map is not None:
        l_rgb = l_rgb + ((rgb_map - rgb_gt) ** 2).sum() / (3 * R)
    if rgb_map0 is not None:
        l_rgb = l_rgb + ((rgb_map0 - rgb_gt) ** 2).sum() / (3 * R)
    l_depth = zero
    if depth_map is not None and depth_gt is not None:
        ok = depth_gt > 0
        l_depth = (torch.abs(depth_map - depth_gt) * ok).sum() / max(int(ok.sum()), 1)
    l_sem = l_fix = zero
    Cn = semantic_map.shape[1] if semantic_map is not None else (fixed_semantic_map.shape[1] if fixed_semantic_map is not None else 0)
    if label is not None and Cn > 0:
        has = (label >= 0) & (label < Cn)
        n = max(int(has.sum()), 1)
        lab = label.clamp(0, Cn - 1).long()
        conf = label_weight if label_weight is not None else torch.ones(R, dtype=dt)
        if semantic_map is not None:
            if sem_is_prob:
                p = semantic_map.gather(1, lab[:, None])[:, 0]
                l_sem = (-torch.log(torch.clamp_min(p, eps)) * conf * has).sum() / n
            else:
                l_sem = (F.cross_entropy(semantic_map, lab, reduction="none") * conf * has).sum() / n
        if fixed_semantic_map is not None:
            p = fixed_semantic_map.gather(1, lab[:, None])[:, 0]
            l_fix = (-torch.log(torch.clamp_min(p, eps)) * conf * has).sum() / n
    terms = torch.stack([l_rgb, l_depth, l_sem, l_fix])
    return (terms * torch.tensor(weights, dtype=dt)).sum(), terms
