"""Oracle of the hash-grid Network (cfg.xyz_encoding = "hashgrid"; rule chosen here, the reference's 360 architecture is
not in the mount): the oracle's Network with h(x) = oracle/reference_panoptic.hashgrid_encode of the sample point in
place of gamma(x) in layer 0 and in the skip concatenation; the view branch keeps gamma(d).  Same state_dict keys and
shapes as the product network (`xyz_encoder.table` [L, 2^T, F], `xyz_encoder.aabb` [6]).  CPU PyTorch, test
infrastructure only."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import reference_panoptic as OP
from oracle import reference_renderer as O

# a small hash grid for the CPU tier (table of 2^12 entries per level) and the scene box of the synthetic rays
SCENE_AABB = [-16.0, -4.0, 0.0, 16.0, 12.0, 64.0]


def hash_cfg(preset: str = "cfg2", **over):
    from panopticnerf_b200 import make_cfg
    kw = dict(xyz_encoding="hashgrid", hash_aabb=SCENE_AABB)
    kw.update(over)
    return make_cfg(preset, **kw)


class HashGridEncoder(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.L, self.F, self.T_log2 = int(cfg.hash_levels), int(cfg.hash_features), int(cfg.hash_log2_size)
        self.base, self.scale = float(cfg.hash_base_resolution), float(cfg.hash_per_level_scale)
        self.table = nn.Parameter(torch.zeros(self.L, 1 << self.T_log2, self.F))
        self.register_buffer("aabb", torch.as_tensor(cfg.hash_aabb, dtype=torch.float32).reshape(6).clone())

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        out = OP.hashgrid_encode(x.reshape(-1, 3), self.aabb, self.table, self.base, self.scale)
        return out.reshape(*x.shape[:-1], self.L * self.F)


class Network(O.Network):
    def __init__(self, cfg):
        super().__init__(cfg)
        E, W = int(cfg.hash_levels) * int(cfg.hash_features), self.W
        self.in_dim = E
        self.pts_linears[0] = nn.Linear(E, W)
        self.pts_linears[self.skip + 1] = nn.Linear(W + E, W)
        self.xyz_encoder = HashGridEncoder(cfg)

    def forward(self, pts: torch.Tensor, viewdirs: torch.Tensor) -> torch.Tensor:
        ex = self.xyz_encoder(pts)
        ed = O.embed(viewdirs, self.Ld).to(ex.dtype)
        h = ex
        for i, lin in enumerate(self.pts_linears):
            h = F.relu(lin(h))
            if i == self.skip:
                h = torch.cat([ex, h], -1)
        sigma = self.alpha_linear(h)
        feat = self.feature_linear(h)
        g = F.relu(self.views_linears[0](torch.cat([feat, ed], -1)))
        outs = [self.rgb_linear(g), sigma]
        if self.C > 0:
            outs.append(self.semantic_linears[1](F.relu(self.semantic_linears[0](h))))
        if self.K > 0:
            outs.append(self.instance_linears[1](F.relu(self.instance_linears[0](h))))
        return torch.cat(outs, -1)


def mlp_flops_per_sample(cfg) -> int:
    """2 x the multiply-adds of the network's linears per sample, layer 0 with K = E."""
    net = Network(cfg)
    return 2 * sum(p.numel() for n, p in net.named_parameters() if n.endswith("weight"))


def oracle_like(net, cfg, dtype=torch.float32) -> Network:
    """The oracle network with the product network's parameters (on the CPU, in `dtype`)."""
    onet = Network(cfg).to(dtype)
    onet.load_state_dict({k: v.detach().cpu().to(dtype) if v.is_floating_point() and k != "xyz_encoder.aabb" else v.detach().cpu()
                          for k, v in net.state_dict().items()})
    return onet
