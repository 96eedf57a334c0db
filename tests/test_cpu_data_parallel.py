"""CPU tier of data-parallel training: the normalisation rule on the float64 loss oracles (the sum over shards of
per-shard gradients normalised by the global counts is the whole batch's gradient; averaging the ranks' means, as DDP
does, is not), the training-batch sharder, and the refusals of pnr_adam_step and FusedAdam by name before any device
call."""
import ctypes as C

import pytest
import torch

from oracle import reference_losses as OL
import oracle_instance as OI
from panopticnerf_b200 import parallel

W = (1.0, 0.1, 1.0, 1.0, 0.7)
THR = 0.5


def _maps(R, Cn, K, seed, no_depth=(), no_label=(), no_inst=()):
    """Rendered maps (float64 leaves) and targets of R rays; rays in the given index sets carry no valid depth, no
    pseudo label or no counted instance target."""
    g = torch.Generator().manual_seed(seed)
    maps = {"rgb_map": torch.rand(R, 3, generator=g, dtype=torch.float64),
            "rgb_map0": torch.rand(R, 3, generator=g, dtype=torch.float64),
            "depth_map": torch.rand(R, generator=g, dtype=torch.float64) * 40,
            "semantic_map": torch.randn(R, Cn, generator=g, dtype=torch.float64) * 2,
            "fixed_semantic_map": torch.rand(R, Cn, generator=g, dtype=torch.float64) * 0.9 + 0.05,
            "instance_map": torch.randn(R, K, generator=g, dtype=torch.float64) * 2}
    tg = {"rgb": torch.rand(R, 3, generator=g, dtype=torch.float64),
          "depth": torch.where(torch.rand(R, generator=g) < 0.7, torch.rand(R, generator=g, dtype=torch.float64) * 40 + 1,
                               torch.zeros(R, dtype=torch.float64)),
          "label": torch.randint(-1, Cn, (R,), generator=g),
          "conf": torch.rand(R, generator=g, dtype=torch.float64),
          "fim": torch.rand(R, K, generator=g, dtype=torch.float64) * 0.4}
    dom = torch.rand(R, generator=g) < 0.6
    tg["fim"][dom, torch.randint(0, K, (int(dom.sum()),), generator=g)] = 0.9
    idx = lambda s: torch.tensor(sorted(s), dtype=torch.long)
    if no_depth:
        tg["depth"][idx(no_depth)] = 0.0
    if no_label:
        tg["label"][idx(no_label)] = -1
    if no_inst:
        tg["fim"][idx(no_inst)] = 0.1
    return maps, tg


def _counts(tg, Cn):
    """Colour values, rays with depth, labelled rays, counted instance rays."""
    R = tg["rgb"].shape[0]
    return (3 * R, int((tg["depth"] > 0).sum()), int(((tg["label"] >= 0) & (tg["label"] < Cn)).sum()),
            int((OI.instance_labels(tg["fim"], THR) >= 0).sum()))


def _terms(maps, tg):
    """The five means of one batch by the oracles (each normalised by the batch's own count)."""
    _, t4 = OL.losses(maps["rgb_map"], maps["rgb_map0"], maps["depth_map"], maps["semantic_map"],
                      maps["fixed_semantic_map"], tg["rgb"], tg["depth"], tg["label"], tg["conf"], (1.0,) * 4)
    inst, _, _, _ = OI.instance_loss(maps["instance_map"], tg["fim"], THR)
    return torch.cat([t4, inst.reshape(1)])


def _shard_grads(maps, tg, Cn, G, rule):
    """Per-shard map gradients stacked back into whole-batch order.  rule 'global': each shard's terms rescaled to the
    global counts (local mean * n_local / n_global); rule 'ddp': the mean over ranks of each shard's own weighted loss."""
    R = tg["rgb"].shape[0]
    n_glob = _counts(tg, Cn)
    out = {k: torch.zeros_like(v) for k, v in maps.items()}
    for r in range(G):
        lo, hi = parallel.shard_range(R, r, G)
        if hi == lo:                              # an empty shard contributes nothing
            continue
        leaf = {k: v[lo:hi].detach().clone().requires_grad_(True) for k, v in maps.items()}
        sub = {k: v[lo:hi] for k, v in tg.items()}
        t = _terms(leaf, sub)
        if rule == "global":
            n_loc = _counts(sub, Cn)
            per_term = (0, 1, 2, 2, 3)                   # fix shares the semantic count
            scale = torch.tensor([n_loc[i] / max(n_glob[i], 1) for i in per_term], dtype=torch.float64)
            loss = (t * scale * torch.tensor(W, dtype=torch.float64)).sum()
        else:
            loss = (t * torch.tensor(W, dtype=torch.float64)).sum() / G
        loss.backward()
        for k in maps:
            out[k][lo:hi] = leaf[k].grad
    return out


CASES = [  # (G, R, rays without depth, without labels, without counted instances) - each shard index set in [lo, hi)
    (1, 37, (), (), ()),
    (2, 37, (), (), ()),
    (3, 40, set(range(0, 14)), (), ()),                 # shard 0 has no valid depth
    (4, 41, (), set(range(11, 22)), ()),                # shard 1 has no labels
    (5, 42, (), (), set(range(27, 36))),                # shard 3 has no counted instance rays
    (5, 19, set(range(0, 4)), (), set(range(16, 19))),  # ceil(19/5) = 4 rays per shard: shard 4 is empty
]


@pytest.mark.parametrize("G,R,nd,nl,ni", CASES)
def test_global_normalisation_gives_the_whole_batch_gradient(G, R, nd, nl, ni):
    Cn, K = 7, 5
    maps, tg = _maps(R, Cn, K, seed=G * 100 + R, no_depth=nd, no_label=nl, no_inst=ni)
    whole = {k: v.detach().clone().requires_grad_(True) for k, v in maps.items()}
    (_terms(whole, tg) * torch.tensor(W, dtype=torch.float64)).sum().backward()
    got = _shard_grads(maps, tg, Cn, G, "global")
    for k in maps:
        ref = whole[k].grad
        err = float((got[k] - ref).abs().max() / ref.abs().max())
        assert err <= 1e-12, f"{k}: {err:.2e}"
    if G >= 2:
        counts = [_counts({k: v[slice(*parallel.shard_range(R, r, G))] for k, v in tg.items()}, Cn) for r in range(G)]
        unequal = any(len({c[i] for c in counts}) > 1 for i in range(1, 4))
        assert unequal
        ddp = _shard_grads(maps, tg, Cn, G, "ddp")
        worst = max(float((ddp[k] - whole[k].grad).abs().max() / whole[k].grad.abs().max()) for k in maps)
        assert worst > 1e-3, "averaging the ranks' means should not give the whole batch's gradient here"


# ------------------------------------------------------------------------------------------------ the sharder
def _train_batch(R):
    b = {k: torch.arange(R * w, dtype=torch.float32).reshape(R, w) if w > 1 else torch.arange(R, dtype=torch.float32)
         for k, w in (("rays", 6), ("near", 1), ("far", 1), ("u", 64), ("u_fine", 128), ("noise", 64),
                      ("noise_fine", 192), ("rgb", 3), ("depth", 1), ("pseudo_weight", 1))}
    b["pseudo_label"] = torch.arange(R, dtype=torch.int64)
    b.update(box_center=torch.zeros(R, 3), box_sem=torch.zeros(R, dtype=torch.int32), scene_aabb=torch.zeros(6))
    return b


@pytest.mark.parametrize("R,world", [(10, 1), (10, 3), (11, 4), (5, 8), (0, 2), (64, 8)])
def test_training_batch_sharder_slices_every_ray_key(R, world):
    b = _train_batch(R)
    seen = {k: [] for k in parallel.TRAIN_RAY_KEYS}
    for r in range(world):
        s = parallel.shard_training_batch(b, r, world)
        lo, hi = parallel.shard_range(R, r, world)
        for k in parallel.TRAIN_RAY_KEYS:
            assert s[k].shape[0] == hi - lo and s[k].is_contiguous(), k
            seen[k].append(s[k])
        for k in ("box_center", "box_sem", "scene_aabb"):     # scene tensors are replicated, even when R matches
            assert s[k] is b[k], k
    for k in parallel.TRAIN_RAY_KEYS:
        assert torch.equal(torch.cat(seen[k]), b[k]), k
    assert parallel.shard_batch(b, 0, max(world, 1))["rgb"] is b["rgb"]      # shard_batch keeps its render keys only


def test_training_batch_sharder_refuses_a_ray_key_of_another_length():
    b = _train_batch(10)
    b["u"] = b["u"][:9]
    with pytest.raises(ValueError, match="u"):
        parallel.shard_training_batch(b, 0, 2)


# ------------------------------------------------------------------------------------------------ refusals
def _adam_args(**over):
    from panopticnerf_b200 import _capi
    a = _capi.PnrAdamArgs()
    a.P, a.ld_grad, a.G, a.beta1, a.beta2, a.eps, a.weight_decay, a.step_size, a.bc2_sqrt = 8, 8, 2, 0.9, 0.999, 1e-8, 0.0, 1e-3, 0.03
    for k, v in over.items():
        setattr(a, k, v)
    return a


BAD_ADAM = [
    (dict(G=0), "G=0"), (dict(P=-1), "P=-1"), (dict(ld_grad=7), "ld_grad=7 < P=8"),
    (dict(G=1 << 30, ld_grad=1 << 40), "overflows"),
    (dict(beta1=1.0), "beta1"), (dict(beta1=-0.1), "beta1"), (dict(beta1=float("nan")), "beta1"),
    (dict(beta2=1.0), "beta2"), (dict(beta2=float("inf")), "beta2"),
    (dict(eps=float("nan")), "eps"), (dict(eps=-1.0), "eps"),
    (dict(weight_decay=float("inf")), "weight_decay"), (dict(weight_decay=-0.01), "weight_decay"),
    (dict(step_size=float("nan")), "step_size"), (dict(step_size=-1.0), "step_size"),
    (dict(bc2_sqrt=0.0), "bc2_sqrt"), (dict(bc2_sqrt=float("inf")), "bc2_sqrt"),
]


@pytest.mark.parametrize("over,msg", BAD_ADAM)
def test_adam_step_refuses_each_argument_by_name(over, msg):
    from panopticnerf_b200 import _capi
    L = _capi.lib()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    assert L.pnr_adam_step(p, p, p, p, C.byref(_adam_args(**over)), None, None) == -1
    assert msg in L.pnr_last_error().decode()


@pytest.mark.parametrize("which", range(4))
def test_adam_step_refuses_a_null_buffer_by_name(which):
    from panopticnerf_b200 import _capi
    L = _capi.lib()
    buf = (C.c_float * 64)()
    ptrs = [C.addressof(buf)] * 4
    ptrs[which] = None
    assert L.pnr_adam_step(*ptrs, C.byref(_adam_args()), None, None) == -1
    assert ("grads", "param", "exp_avg", "exp_avg_sq")[which] in L.pnr_last_error().decode()
    assert L.pnr_adam_step(None, None, None, None, C.byref(_adam_args(P=0, ld_grad=0)), None, None) == 0   # P = 0: no-op


def test_broadcast_refuses_a_null_communicator():
    from panopticnerf_b200 import _capi
    L = _capi.lib()
    assert L.pnr_broadcast(None, None, 4, 0, None) == -1
    assert "pnr_broadcast" in L.pnr_last_error().decode()


@pytest.mark.parametrize("opt,msg", [(dict(amsgrad=True), "amsgrad"), (dict(maximize=True), "maximize"),
                                     (dict(capturable=True), "capturable"), (dict(differentiable=True), "differentiable"),
                                     (dict(betas=(0.9, 1.0)), "betas"), (dict(lr=-1.0), "lr"), (dict(eps=-1.0), "eps"),
                                     (dict(weight_decay=-1.0), "weight_decay")])
def test_fused_adam_refuses_options_by_name(opt, msg):
    from panopticnerf_b200.lib.train import FusedAdam
    with pytest.raises(ValueError, match=msg):
        FusedAdam([torch.nn.Parameter(torch.zeros(3))], **opt)


def test_fused_adam_refuses_non_fp32_and_cpu_parameters():
    from panopticnerf_b200.lib.train import FusedAdam
    with pytest.raises(ValueError, match="float32"):
        FusedAdam([torch.nn.Parameter(torch.zeros(3, dtype=torch.float64))])
    with pytest.raises(ValueError, match="CUDA"):
        FusedAdam([torch.nn.Parameter(torch.zeros(3))])


class _OneRank:
    rank, world = 0, 1

    def broadcast(self, t):
        return t


@pytest.mark.parametrize("K,boxes,box_inst,on", [(6, 3, True, True), (0, 3, True, False), (6, 0, True, False),
                                                 (6, 3, False, False)])
def test_every_rank_decides_the_instance_term_by_the_renderers_rule(K, boxes, box_inst, on):
    """An empty shard renders nothing, so it decides from the configuration and the replicated primitives, as the
    renderer does: instance slots, a non-empty box_center and box_inst."""
    import panopticnerf_b200 as PN
    from panopticnerf_b200.lib.train import DataParallelWrapper
    cfg = PN.make_cfg("cfg1", num_classes=5, num_instances=K)
    w = DataParallelWrapper(cfg, PN.make_network(cfg), device="cpu", comm=_OneRank())
    shard = {"rays": torch.zeros(0, 6), "box_center": torch.zeros(boxes, 3)}
    if box_inst:
        shard["box_inst"] = torch.zeros(boxes, dtype=torch.int32)
    assert w.instance_term_on(shard) is on
