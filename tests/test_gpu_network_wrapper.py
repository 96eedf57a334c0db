"""GPU tier of the training iteration: the instance term of `pnr_losses` per ray against the float64 oracle, its labels,
count and graph capture; `Renderer.render_train` against the staged `render`; one `NetworkWrapper` iteration (both
passes, all five terms, separate and shared fine network) against the oracle chain; and a few Adam steps that train
the coarse, fine and instance heads, of a frequency and a hash-grid network."""
import ctypes as C

import numpy as np
import pytest
import torch

import panopticnerf_b200 as PN
import oracle_instance as OI
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.train import NetworkWrapper, make_network_wrapper
from test_gpu_train_chain import record_d_raw, run_chain  # noqa: F401 (record_d_raw: a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
THR = 0.5


# ------------------------------------------------------------------------------------------------ the loss kernel
def _loss_call(maps, K=0, im=None, fim=None, w_inst=1.0, thr=THR):
    """pnr_losses through the C ABI: maps holds the existing inputs (any subset, device tensors); im / fim turn the
    instance term on.  Returns (per_ray [R,4], {d_<map>}, and with the term per_ray_inst, inst_label, n_inst)."""
    ref = next(v for v in list(maps.values()) + [im] if v is not None)
    R = ref.shape[0]
    a = _capi.PnrLossArgs()
    a.R, a.eps = R, 1e-6
    a.C = maps["semantic_map"].shape[1] if "semantic_map" in maps else 0
    a.w_rgb, a.w_depth, a.w_sem, a.w_fix = 1.0, 0.1, 0.5, 2.0
    a.inv_n_rgb, a.inv_n_depth, a.inv_n_sem = 1.0 / (3 * R), 1.0 / R, 1.0 / R
    out = {"per_ray": torch.full((R, 4), float("nan"), device=DEV)}
    a.per_ray = out["per_ray"].data_ptr()
    for k, v in maps.items():
        setattr(a, k, v.data_ptr())
        if k in ("rgb_map", "rgb_map0", "depth_map", "semantic_map", "fixed_semantic_map"):
            out["d_" + k] = torch.full_like(v, float("nan"))
            setattr(a, "d_" + k, out["d_" + k].data_ptr())
    if im is not None:
        out.update(per_ray_inst=torch.full((R,), float("nan"), device=DEV), inst_label=torch.full((R,), -7, dtype=torch.int32, device=DEV),
                   n_inst=torch.full((1,), 12345, dtype=torch.int32, device=DEV), d_instance_map=torch.full_like(im, float("nan")))
        a.K, a.w_inst, a.inst_min_weight = K, w_inst, thr
        a.instance_map, a.fixed_instance_map = im.data_ptr(), fim.data_ptr()
        for k in ("per_ray_inst", "inst_label", "n_inst", "d_instance_map"):
            setattr(a, k, out[k].data_ptr())
    _capi.check(_capi.lib().pnr_losses(C.byref(a), _capi.stream_ptr()), "pnr_losses")
    return out


def _existing_maps(R, Cn, seed):
    g = torch.Generator().manual_seed(seed)
    m = {"rgb_map": torch.rand(R, 3, generator=g), "rgb_map0": torch.rand(R, 3, generator=g), "rgb_gt": torch.rand(R, 3, generator=g),
         "depth_map": torch.rand(R, generator=g) * 40, "depth_gt": torch.rand(R, generator=g) * 40 - 5,
         "semantic_map": torch.randn(R, Cn, generator=g) * 3, "fixed_semantic_map": torch.rand(R, Cn, generator=g),
         "label": torch.randint(-1, Cn, (R,), generator=g, dtype=torch.int32), "label_weight": torch.rand(R, generator=g)}
    return {k: v.to(DEV) for k, v in m.items()}


def _instance_case(R, K, seed):
    """Instance logits and fixed maps that visit every branch of the rule: ordinary rows, rows of logits +-1e4, ties of
    the maximum, a maximum exactly at the threshold and one ulp below it, NaN rows and rows without primitives."""
    g = torch.Generator().manual_seed(seed)
    im = torch.randn(R, K, generator=g) * 3
    big = torch.rand(R, generator=g) < 0.15
    im[big] = torch.where(torch.rand(int(big.sum()), K, generator=g) < 0.5, -1e4, 1e4)
    fim = torch.rand(R, K, generator=g) * (torch.rand(R, K, generator=g) < 0.3)
    fim = fim / fim.sum(1, keepdim=True).clamp(min=1.0)
    kind = torch.randint(0, 8, (R,), generator=g)
    below = float(np.nextafter(np.float32(THR), np.float32(0)))
    for r in range(R):
        k0, k1 = int(torch.randint(0, K, (1,), generator=g)), int(torch.randint(0, K, (1,), generator=g))
        if kind[r] == 1:        # a tie of the maximum (two slots, when K > 1), at the threshold
            fim[r] = 0.0
            fim[r, k0] = fim[r, k1] = THR
        elif kind[r] == 2:      # maximum exactly at the threshold
            fim[r] = fim[r] * 0.1
            fim[r, k0] = THR
        elif kind[r] == 3:      # one ulp below
            fim[r] = fim[r] * 0.1
            fim[r, k0] = below
        elif kind[r] == 4:      # NaN in the row
            fim[r, k0] = float("nan")
            fim[r, k1] = 0.9 if k1 != k0 else fim[r, k1]
        elif kind[r] == 5:      # no primitive on the ray
            fim[r] = 0.0
        elif kind[r] == 6:      # a clear dominant primitive
            fim[r, k0] = 0.95
    return im.contiguous(), fim.contiguous()


def test_the_instance_term_leaves_the_other_terms_alone():
    R, Cn, K = 1000, 19, 33
    maps = _existing_maps(R, Cn, seed=1)
    im, fim = (t.to(DEV) for t in _instance_case(R, K, seed=2))
    off = _loss_call(maps)
    on = _loss_call(maps, K, im, fim)
    for k in off:
        assert torch.equal(off[k], on[k]), k
    assert not torch.isnan(on["per_ray"]).any()


@pytest.mark.parametrize("K", [1, 2, 31, 32, 33, 128, 1000])
@pytest.mark.parametrize("R", [1, 13, 1000])
def test_the_instance_term_per_ray_matches_float64(R, K):
    im, fim = _instance_case(R, K, seed=R * 7 + K)
    w = 0.7
    got = _loss_call({}, K, im.to(DEV), fim.to(DEV), w_inst=w)
    imd = im.double().requires_grad_(True)
    mean, per_ray, label, n = OI.instance_loss(imd, fim.double(), THR)
    (w * mean).backward()
    assert torch.equal(got["inst_label"].cpu().long(), label)
    assert int(got["n_inst"]) == n
    # each ray against its own largest |ref|; floored at 1e-2 (loss) and 1e-2 * w / n (a gradient row sums to at most
    # 2 w / n): fp32 forms 1 - p and log(1 + small) with an absolute error of a few ulp(1)
    pr = per_ray.detach()
    assert ((got["per_ray_inst"].cpu().double() - pr).abs() <= 1e-4 * pr.abs().clamp(min=1e-2)).all()
    ref = imd.grad
    scale = ref.abs().amax(1, keepdim=True).clamp(min=1e-2 * w / max(n, 1))
    err = (got["d_instance_map"].cpu().double() - ref).abs()
    assert (err <= 1e-4 * scale).all(), float((err / scale).max())


def test_instance_labels_and_count_are_exact_and_replay_under_graph_capture():
    R, K = 4099, 64
    im, fim = (t.to(DEV) for t in _instance_case(R, K, seed=9))
    eager = _loss_call({}, K, im, fim)
    label = OI.instance_labels(fim.cpu().double(), THR)
    assert torch.equal(eager["inst_label"].cpu().long(), label) and int(eager["n_inst"]) == int((label >= 0).sum())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):          # warm-up outside the capture, as torch.cuda.graph expects
        _loss_call({}, K, im, fim)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = _loss_call({}, K, im, fim)
    for t in cap.values():
        t.fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(cap[k], eager[k]), k


# ------------------------------------------------------------------------------------------------ render and wrapper
def _cfg(**over):
    kw = dict(render_path="staged", bound_by_primitives=True, perturb=1.0, check_range=True)
    kw.update(over)
    return PN.make_cfg("cfg3", **kw)


def _batch(cfg, R, seed, row0=150, step=1):
    """R rays of one synthetic frame with its primitives, seeded jitter and targets (colour, depth, pseudo labels)."""
    b = S.make_batch(cfg, seed=seed, row0=row0, rows=(R * step + int(cfg.W_img) - 1) // int(cfg.W_img))
    b["rays"] = b["rays"][::step][:R].contiguous()
    g = torch.Generator().manual_seed(seed + 100)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    b.update(u=torch.rand(R, N, generator=g), u_fine=torch.rand(R, Ni, generator=g), rgb=torch.rand(R, 3, generator=g),
             depth=torch.where(torch.rand(R, generator=g) < 0.7, torch.rand(R, generator=g) * 40 + 5, torch.zeros(R)),
             pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    return b


def _dev(b):
    return {k: v.to(DEV) for k, v in b.items()}


def test_render_train_without_grad_equals_the_staged_render():
    cfg = _cfg()
    net = S.init_network_weights(PN.make_network(cfg), seed=3).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=4).to(DEV)
    ren = PN.make_renderer(cfg, net, fine)
    b = _dev(_batch(cfg, 700, seed=5))
    ref = ren.render(b)
    with torch.no_grad():
        got = ren.render_train(b)
    assert set(got) == set(ref)
    for k in ("weights", "weights_0", "z_vals", "z_vals_0", "sample_box", "rgb_map", "rgb_map_0", "instance_map",
              "fixed_instance_map_0", "fixed_semantic_map"):
        assert k in ref, k
    for k in ref:
        assert torch.equal(got[k], ref[k]), k


@pytest.mark.parametrize("shared", [False, True])
def test_one_iteration_matches_the_oracle_chain(shared, record_d_raw):
    """cfg3-shaped networks, 64 + 128 samples, primitives, fixed maps and all five terms against the float64 oracle
    chain pinned to the iteration's own decisions (tests/test_gpu_train_chain.run_chain): maps, total and terms,
    d_raw of both passes and every parameter's gradient element by element; labels and count exact."""
    cfg = _cfg()
    net = S.init_network_weights(PN.make_network(cfg), seed=21).to(DEV)
    fine = None if shared else S.init_network_weights(PN.make_network(cfg), seed=22).to(DEV)
    b = _batch(cfg, 160, seed=7, step=8)
    mine, ref, ob, pins, output = run_chain(cfg, net, fine, b, record_d_raw, f"wrapper shared={shared}")
    label = OI.instance_labels(ref["maps"]["fine"]["fixed_instance_map"].cpu(), 0.5)
    n = int((label >= 0).sum())
    assert n >= 20 and torch.equal(output["inst_label"].cpu().long(), label)
    assert float((net if shared else fine).instance_linears[1].weight.grad.norm()) > 0.0
    if not shared:      # only its colour is supervised: the coarse network's heads get exactly nothing
        assert float(net.instance_linears[1].weight.grad.abs().max()) == 0.0


def _train(cfg, net, fine, steps, lr, seed):
    wrapper = make_network_wrapper(cfg, net, fine)
    opt = torch.optim.Adam(wrapper.parameters(), lr=lr)
    b = _dev(_batch(cfg, 2048, seed=seed, step=2))
    g = torch.Generator().manual_seed(seed)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    losses, acc = [], []
    for _ in range(steps):
        b["u"], b["u_fine"] = torch.rand(2048, N, generator=g).to(DEV), torch.rand(2048, Ni, generator=g).to(DEV)
        opt.zero_grad(set_to_none=True)
        output, loss, stats, _ = wrapper(b)
        loss.backward()
        opt.step()
        lab = output["inst_label"]
        ok = lab >= 0
        acc.append(float((output["instance_map"].detach().argmax(1)[ok] == lab[ok]).float().mean()))
        losses.append(float(loss.detach()))
    return losses, acc


def test_adam_steps_lower_the_loss_and_train_the_instance_head():
    cfg = _cfg()
    net = S.init_network_weights(PN.make_network(cfg), seed=31).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=32).to(DEV)
    losses, acc = _train(cfg, net, fine, 30, 1e-3, seed=11)
    print(f"loss {losses[0]:.4f} -> {losses[-1]:.4f}; instance accuracy {acc[0]:.3f} -> {acc[-1]:.3f}")
    # the jitter is redrawn every step, so the loss is compared over three steps at either end
    assert np.mean(losses[-3:]) < 0.95 * np.mean(losses[:3]), losses
    assert np.mean(acc[-3:]) >= acc[0] + 0.5, acc


def test_a_hash_grid_network_trains_through_the_wrapper():
    from oracle_hashgrid import hash_cfg
    cfg = hash_cfg("cfg3", render_path="staged", bound_by_primitives=True, perturb=1.0, hash_log2_size=16)
    net = S.init_network_weights(PN.make_network(cfg), seed=41).to(DEV)
    table = net.xyz_encoder.table.detach().clone()
    losses, _ = _train(cfg, net, None, 10, 1e-3, seed=12)
    assert losses[-1] < losses[0], losses
    assert not torch.equal(net.xyz_encoder.table.detach(), table)


def test_make_network_wrapper_resolves_the_module_and_refuses_cpu_tensors():
    import types
    import sys
    cfg = _cfg()
    net = S.init_network_weights(PN.make_network(cfg), seed=1)
    assert type(make_network_wrapper(cfg, net)) is NetworkWrapper
    mod = types.ModuleType("pnr_test_trainer_plugin")

    class Plugin(NetworkWrapper):
        pass
    mod.NetworkWrapper = Plugin
    sys.modules[mod.__name__] = mod
    try:
        cfg.trainer_module = mod.__name__
        assert type(make_network_wrapper(cfg, net)) is Plugin
    finally:
        del sys.modules[mod.__name__]
    wrapper = NetworkWrapper(PN.make_cfg("cfg3"), net)
    with pytest.raises(_capi.PnrError, match="CUDA"):
        wrapper(_batch(cfg, 16, seed=1))
