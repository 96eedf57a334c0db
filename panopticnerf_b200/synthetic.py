"""Seeded synthetic inputs of KITTI-360 shape (SURVEY.md section 8(d)): pinhole / equirect rays,
a scene AABB, B oriented bounding primitives, and network weights.  Pure CPU torch, deterministic;
both bench arms and the tests draw their inputs from here so they see identical data.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

SCENE_AABB = ((-16.0, -4.0, 0.0), (16.0, 12.0, 64.0))


def make_rays(cfg, seed: int = 0, row0: int = 0, rows: Optional[int] = None) -> torch.Tensor:
    """[rows*W, 6] fp32 = origin || unnormalised direction, row-major over (v, u)."""
    H, W = int(cfg.H), int(cfg.W_img)
    rows = H - row0 if rows is None else rows
    g = torch.Generator().manual_seed(seed)
    yaw = (torch.rand((), generator=g).item() - 0.5) * 0.1
    v, u = torch.meshgrid(torch.arange(row0, row0 + rows, dtype=torch.float32),
                          torch.arange(W, dtype=torch.float32), indexing="ij")
    if getattr(cfg, "camera", "pinhole") == "equirect":
        lon = (u / W - 0.5) * (2.0 * math.pi)
        lat = (0.5 - v / H) * math.pi
        d = torch.stack([torch.cos(lat) * torch.sin(lon), -torch.sin(lat),
                         torch.cos(lat) * torch.cos(lon)], -1)
        origin = torch.tensor([0.0, 4.0, 32.0])          # panorama taken inside the scene
    else:
        d = torch.stack([(u - cfg.cx) / cfg.fx, (v - cfg.cy) / cfg.fy, torch.ones_like(u)], -1)
        origin = torch.tensor([0.0, 0.0, 0.0])
    c, s = math.cos(yaw), math.sin(yaw)
    rot = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
    d = (d.reshape(-1, 3) @ rot.T).contiguous()
    o = origin[None].expand_as(d)
    return torch.cat([o, d], -1).contiguous()


def make_boxes(num_boxes: int = 64, num_classes: int = 45, num_instances: int = 64,
               seed: int = 0) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed + 1)
    lo = torch.tensor(SCENE_AABB[0])
    hi = torch.tensor(SCENE_AABB[1])
    center = lo + (hi - lo) * torch.rand(num_boxes, 3, generator=g)
    half = 0.5 + 3.5 * torch.rand(num_boxes, 3, generator=g)
    yaw = 2.0 * math.pi * torch.rand(num_boxes, generator=g)
    c, s = torch.cos(yaw), torch.sin(yaw)
    z, one = torch.zeros_like(c), torch.ones_like(c)
    rot = torch.stack([torch.stack([c, z, s], -1), torch.stack([z, one, z], -1),
                       torch.stack([-s, z, c], -1)], -2)       # [B,3,3], columns = box axes
    sem = torch.randint(0, max(num_classes, 1), (num_boxes,), generator=g, dtype=torch.int32)
    inst = torch.randint(0, max(num_instances, 1), (num_boxes,), generator=g, dtype=torch.int32)
    return dict(box_center=center.contiguous(), box_half=half.contiguous(), box_rot=rot.contiguous(),
                box_sem=sem, box_inst=inst)


def make_batch(cfg, seed: int = 0, row0: int = 0, rows: Optional[int] = None, num_boxes: int = 64,
               with_boxes: bool = True) -> Dict[str, torch.Tensor]:
    batch = {"rays": make_rays(cfg, seed, row0, rows),
             "scene_aabb": torch.tensor(SCENE_AABB, dtype=torch.float32)}
    if with_boxes and num_boxes > 0:
        batch.update(make_boxes(num_boxes, int(cfg.num_classes), int(cfg.num_instances), seed))
    return batch


def init_network_weights(net: torch.nn.Module, seed: int = 0) -> torch.nn.Module:
    """Re-draws every nn.Linear with PyTorch's default init from a fixed seed, then shifts the sigma
    bias so that accumulated opacity is non-trivial on the synthetic scene.  A hash-grid network's table is drawn
    U(-1, 1) after the linears (features of O(1)); the linears get the same values as without it."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(net.named_parameters()):
            if name.startswith("xyz_encoder."):
                continue
            if p.dim() == 2:
                bound = 1.0 / math.sqrt(p.shape[1])
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * bound)
            else:
                w = dict(net.named_parameters())[name.replace("bias", "weight")]
                bound = 1.0 / math.sqrt(w.shape[1])
                p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * bound)
        net.alpha_linear.bias.add_(0.1)
        enc = getattr(net, "xyz_encoder", None)
        if enc is not None:
            enc.table.copy_(torch.rand(enc.table.shape, generator=g) * 2 - 1)
    return net
