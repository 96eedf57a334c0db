"""GPU parity of the compositing backward pass (SURVEY 8(f) rank 2, first stage of the backward chain):
`pnr_composite_backward` through the C ABI vs torch.autograd through the oracle's raw2outputs on identical
inputs and identical upstream gradients.  Tolerance: 1e-4 relative, floor = RMS of the oracle's gradient
tensor per channel group (gradients span many orders of magnitude along a ray).
Parity is "vs in-repo oracle" - the reference source is not in the mount (parity unpinned)."""
import pytest
import torch

from oracle import reference_renderer as O
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from test_gpu_train_chain import check_single_pass, record_d_raw  # noqa: F401 (record_d_raw: a fixture)
from util import assert_close, rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _case(R, N, C, K, seed, boxes=False, far=60.0):
    g = torch.Generator().manual_seed(seed)
    raw = torch.randn(R, N, 4 + C + K, generator=g)
    raw[..., 3] = raw[..., 3] * 0.6 - 0.1           # a mix of empty (sigma_raw <= 0) and occupied samples
    z = torch.sort(torch.rand(R, N, generator=g) * (far - 2.0) + 2.0, -1).values
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1) * (0.5 + torch.rand(R, 1, generator=g))
    kw = {}
    if boxes:
        B = 9
        kw["sample_box"] = torch.randint(-1, B, (R, N), generator=g, dtype=torch.int32)
        kw["box_sem"] = torch.randint(0, max(C, 1), (B,), generator=g, dtype=torch.int32)
        kw["box_inst"] = torch.randint(0, max(K, 1), (B,), generator=g, dtype=torch.int32)
    return raw, z, d, kw


def _oracle_grad(raw, z, d, kw, ups, **opts):
    raw = raw.clone().requires_grad_(True)
    out = O.raw2outputs(raw, z, d, num_classes=opts.get("C", 0), num_instances=opts.get("K", 0),
                        white_bkgd=opts.get("white_bkgd", False), mask_outside=opts.get("mask_outside", False), **kw)
    loss = sum((out[k] * u).sum() for k, u in ups.items())
    (g,) = torch.autograd.grad(loss, raw)
    return g


def _ups(out_keys, R, N, C, K, seed):
    g = torch.Generator().manual_seed(seed + 100)
    shapes = {"rgb_map": (R, 3), "depth_map": (R,), "acc_map": (R,), "weights": (R, N), "semantic_map": (R, C),
              "instance_map": (R, K), "fixed_semantic_map": (R, C), "fixed_instance_map": (R, K)}
    return {k: torch.randn(*shapes[k], generator=g) for k in out_keys}


def _check(g_gpu, g_ref, C, K, what):
    g_gpu = g_gpu.cpu()
    assert torch.isfinite(g_ref).all()
    groups = [("rgb", slice(0, 3)), ("sigma", slice(3, 4))]
    if C:
        groups.append(("sem", slice(4, 4 + C)))
    if K:
        groups.append(("inst", slice(4 + C, 4 + C + K)))
    for name, sl in groups:
        ref = g_ref[..., sl]
        assert_close(g_gpu[..., sl], ref, max(rms(ref), 1e-12), f"{what}: d_raw[{name}]")


@pytest.mark.parametrize("R,N,C,K", [(300, 64, 0, 0), (257, 33, 7, 5), (64, 192, 45, 50), (5, 1, 3, 0), (40, 256, 0, 4)])
def test_composite_backward_matches_autograd(R, N, C, K):
    raw, z, d, kw = _case(R, N, C, K, seed=R + N)
    keys = ["rgb_map", "depth_map", "acc_map", "weights"] + (["semantic_map"] if C else []) + (["instance_map"] if K else [])
    ups = _ups(keys, R, N, C, K, seed=N)
    ref = _oracle_grad(raw, z, d, kw, ups, C=C, K=K)
    got = P.raw2outputs_backward(raw.to(DEV), z.to(DEV), d.to(DEV), {k: v.to(DEV) for k, v in ups.items()},
                                 num_classes=C, num_instances=K)
    _check(got, ref, C, K, f"R={R} N={N} C={C} K={K}")


def test_composite_backward_options_and_fixed_maps():
    """white background, density masked outside the primitives, gradients of the fixed (bounding-box) maps."""
    R, N, C, K = 200, 64, 6, 4
    raw, z, d, kw = _case(R, N, C, K, seed=11, boxes=True)
    keys = ["rgb_map", "acc_map", "semantic_map", "fixed_semantic_map", "fixed_instance_map"]
    ups = _ups(keys, R, N, C, K, seed=5)
    ref = _oracle_grad(raw, z, d, kw, ups, C=C, K=K, white_bkgd=True, mask_outside=True)
    got = P.raw2outputs_backward(raw.to(DEV), z.to(DEV), d.to(DEV), {k: v.to(DEV) for k, v in ups.items()},
                                 white_bkgd=True, mask_outside=True, num_classes=C, num_instances=K,
                                 **{k: v.to(DEV) for k, v in kw.items()})
    _check(got, ref, C, K, "options")
    outside = kw["sample_box"] < 0
    assert outside.any() and bool((got.cpu()[..., 3][outside] == 0).all())


def test_composite_backward_subset_of_maps_and_empty():
    R, N = 100, 64
    raw, z, d, kw = _case(R, N, 0, 0, seed=3)
    ups = _ups(["depth_map"], R, N, 0, 0, seed=1)
    ref = _oracle_grad(raw, z, d, kw, ups)
    got = P.raw2outputs_backward(raw.to(DEV), z.to(DEV), d.to(DEV), {"depth_map": ups["depth_map"].to(DEV)})
    _check(got, ref, 0, 0, "depth only")
    assert bool((got.cpu()[..., :3] == 0).all())          # no colour gradient was supplied
    e = P.raw2outputs_backward(raw[:0].to(DEV), z[:0].to(DEV), d[:0].to(DEV), {})
    assert e.shape == (0, N, 4)


def test_losses_backpropagate_through_the_autograd_node():
    """A torch-side photometric + cross-entropy + depth loss on the composited maps reaches `raw`."""
    R, N, C = 150, 64, 8
    raw, z, d, kw = _case(R, N, C, 0, seed=21)
    g = torch.Generator().manual_seed(2)
    rgb_gt, label, depth_gt = torch.rand(R, 3, generator=g), torch.randint(0, C, (R,), generator=g), torch.rand(R, generator=g) * 50

    def loss_fn(out):
        return (((out["rgb_map"] - rgb_gt.to(out["rgb_map"].device)) ** 2).mean()
                + 0.1 * torch.nn.functional.cross_entropy(out["semantic_map"], label.to(out["rgb_map"].device))
                + 0.01 * (out["depth_map"] - depth_gt.to(out["rgb_map"].device)).abs().mean())

    raw_c = raw.clone().requires_grad_(True)
    loss_fn(O.raw2outputs(raw_c, z, d, num_classes=C)).backward()
    raw_g = raw.to(DEV).requires_grad_(True)
    out = P.raw2outputs_autograd(raw_g, z.to(DEV), d.to(DEV), num_classes=C)
    loss_fn(out).backward()
    _check(raw_g.grad, raw_c.grad, C, 0, "loss")
    assert not out["disp_map"].requires_grad


def test_composite_backward_rejects_what_it_does_not_implement():
    raw, z, d, _ = _case(4, 8, 3, 0, seed=0)
    with pytest.raises(Exception, match="softmax"):
        P.raw2outputs_backward(raw.to(DEV), z.to(DEV), d.to(DEV), {}, num_classes=3, sem_activation="softmax")
    with pytest.raises(ValueError, match="disp_map"):
        P.raw2outputs_backward(raw.to(DEV), z.to(DEV), d.to(DEV), {"disp_map": torch.zeros(4, device=DEV)}, num_classes=3)


# ------------------------------------------------------------------------------------------------------------------
# MLP backward, first slice: dL/d(embedded xyz) through the trunk (pnr_mlp_backward_trunk) vs autograd through the
# oracle network's pts_linears (float64), 1e-4 of the gradient's RMS.  relu' is discontinuous, so rows with a
# pre-activation within rounding distance of zero are only checked for sanity (test_cpu_program.assert_grad_close).
# ------------------------------------------------------------------------------------------------------------------
from panopticnerf_b200 import make_cfg, make_network, synthetic as S       # noqa: E402
from test_cpu_program import assert_grad_close, trunk_grad_oracle          # noqa: E402


@pytest.mark.parametrize("preset,over,n", [("cfg2", {}, 1000), ("cfg2", dict(precision="bf16x3"), 517),
                                           ("cfg1", dict(D=5, W=128), 128 * 3), ("cfg1", dict(D=3, W=64, xyz_res=4), 77),
                                           ("cfg3", {}, 40000)])
def test_mlp_backward_trunk_matches_autograd(preset, over, n):
    cfg = make_cfg(preset, **over)
    net = S.init_network_weights(make_network(cfg), seed=2).to(DEV)
    g = torch.Generator().manual_seed(n)
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 4
    grad_h = torch.randn(n, cfg.W, generator=g)
    got = net.backward_trunk(grad_h.to(DEV), pts=pts.to(DEV)).cpu()
    assert net.range_status() == 0
    ref, min_z = trunk_grad_oracle(cfg, net.cpu(), pts, grad_h)
    kink = {"fp16x3": 1e-5, "bf16x3": 3e-5}[cfg.precision]
    assert_grad_close(got.double(), ref, min_z, f"{preset} {over} d_emb", 1e-4, kink)


def test_mlp_backward_trunk_rays_mode_is_deterministic_and_chunk_invariant():
    """(rays, z) addressing forms the same points as the forward kernel does; two runs agree bit for bit and a
    sample's gradient does not depend on which tile or launch it was in."""
    cfg = make_cfg("cfg2")
    net = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
    g = torch.Generator().manual_seed(1)
    R, N = 301, 64
    rays = torch.cat([torch.randn(R, 3, generator=g), torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)], -1).to(DEV)
    z = torch.sort(torch.rand(R, N, generator=g) * 20 + 1, -1).values.to(DEV)
    grad_h = torch.randn(R * N, cfg.W, generator=g).to(DEV)
    a = net.backward_trunk(grad_h, rays=rays, z=z)
    b = net.backward_trunk(grad_h, rays=rays, z=z)
    assert torch.equal(a, b)
    pts = (rays[:, None, :3] + rays[:, None, 3:] * z[..., None]).reshape(-1, 3)
    c = net.backward_trunk(grad_h, pts=pts)
    assert torch.equal(a, c)
    lo, hi = 100 * N, 187 * N                      # a chunk that starts and ends inside tiles
    d = net.backward_trunk(grad_h[lo:hi].contiguous(), rays=rays[100:187].contiguous(), z=z[100:187].contiguous())
    assert torch.equal(a[lo:hi], d)


def test_mlp_backward_trunk_small_gradients_are_scaled():
    """Gradients of a mean-reduced loss are ~1e-6: the wrapper's power-of-two scaling keeps the fp16 operand parts in
    the normal range, so the result is the O(1) result times the factor - bit for bit when the factor is a power of two."""
    cfg = make_cfg("cfg2")
    net = S.init_network_weights(make_network(cfg), seed=9).to(DEV)
    g = torch.Generator().manual_seed(4)
    pts = ((torch.rand(900, 3, generator=g) * 2 - 1) * 3).to(DEV)
    grad_h = torch.randn(900, cfg.W, generator=g).to(DEV)
    big = net.backward_trunk(grad_h, pts=pts)
    small = net.backward_trunk(grad_h * 2.0 ** -20, pts=pts)
    assert torch.equal(small * 2.0 ** 20, big)
    unscaled = net.backward_trunk(grad_h * 2.0 ** -20, pts=pts, grad_scale=1.0)      # what happens without it
    assert float((unscaled * 2.0 ** 20 - big).abs().max() / big.abs().max()) > 1e-4
    from panopticnerf_b200 import _capi
    with pytest.raises(_capi.PnrError, match="power of two"):
        net.backward_trunk(grad_h, pts=pts, grad_scale=3.0)


def test_mlp_backward_trunk_rejects_what_it_does_not_implement():
    from panopticnerf_b200 import _capi
    cfg = make_cfg("cfg2", precision="fp16")
    net = S.init_network_weights(make_network(cfg), seed=0).to(DEV)
    with pytest.raises(_capi.PnrError, match="x3"):
        net.backward_trunk(torch.zeros(128, cfg.W, device=DEV), pts=torch.zeros(128, 3, device=DEV))
    net = S.init_network_weights(make_network(make_cfg("cfg2")), seed=0).to(DEV)
    with pytest.raises(_capi.PnrError, match="CUDA tensor"):
        net.backward_trunk(torch.zeros(128, 256), pts=torch.zeros(128, 3, device=DEV))


def test_mlp_backward_trunk_unpadded_rows_match_padded():
    """ld_emb = 3 + 6*xyz_res (scalar stores) gives the same numbers as the padded rows the Python layer uses."""
    from panopticnerf_b200 import _capi
    cfg = make_cfg("cfg2")
    net = S.init_network_weights(make_network(cfg), seed=8).to(DEV)
    g = torch.Generator().manual_seed(3)
    n, Ex = 700, 3 + 6 * cfg.xyz_res
    pts = ((torch.rand(n, 3, generator=g) * 2 - 1) * 3).to(DEV)
    grad_h = torch.randn(n, cfg.W, generator=g).to(DEV)
    padded = net.backward_trunk(grad_h, pts=pts, grad_scale=256.0)
    out = torch.full((n, Ex), float("nan"), device=DEV)
    _capi.check(_capi.lib().pnr_mlp_backward_trunk(net.pack(torch.device(DEV)), pts.data_ptr(), None, None, n, 1,
                                                   grad_h.data_ptr(), 256.0, out.data_ptr(), Ex, None, None, _capi.stream_ptr()))
    assert torch.equal(out, padded)


# ------------------------------------------------------------------------------------------------------------------
# The whole Network.forward backward: every parameter's gradient vs autograd through the oracle network (float64).
# ------------------------------------------------------------------------------------------------------------------
def _oracle_net(cfg, net_cpu):
    onet = O.Network(cfg).double()
    onet.load_state_dict({k: v.double() for k, v in net_cpu.state_dict().items()})
    return onet


def _min_preactivation(onet, pts, vd):
    """Smallest |pre-activation| over every ReLU of the network, per sample (float64 oracle forward)."""
    ex, ed = O.embed(pts, onet.Lx).double(), O.embed(vd, onet.Ld).double()
    m = torch.full((pts.shape[0],), float("inf"), dtype=torch.float64)
    track = lambda t: torch.minimum(m, t.abs().min(dim=1).values)
    h = ex
    with torch.no_grad():
        for i, lin in enumerate(onet.pts_linears):
            pre = lin(h); m = track(pre); h = torch.relu(pre)
            if i == onet.skip:
                h = torch.cat([ex, h], -1)
        m = track(onet.views_linears[0](torch.cat([onet.feature_linear(h), ed], -1)))
        if onet.C > 0:
            m = track(onet.semantic_linears[0](h))
        if onet.K > 0:
            m = track(onet.instance_linears[0](h))
    return m


@pytest.mark.parametrize("preset,over,n", [("cfg2", {}, 4000), ("cfg3", {}, 3000), ("cfg1", dict(D=5, W=128, num_classes=7), 1500),
                                           ("cfg2", dict(precision="bf16x3"), 30000)])
def test_network_backward_every_parameter(preset, over, n):
    """Weight gradients are sums over samples, and relu' is discontinuous: one unit taking the other branch moves a
    whole sample's contribution (~1/sqrt(n) of the sum).  So the comparison runs on the samples whose pre-activations
    all stay clear of zero by 100x the rounding error of the mode under test (10x in bf16x3) - the same samples on both sides."""
    from panopticnerf_b200.lib.train import network_backward
    cfg = make_cfg(preset, **over)
    net = S.init_network_weights(make_network(cfg), seed=11)
    onet = _oracle_net(cfg, net)
    g = torch.Generator().manual_seed(n)
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    keep = _min_preactivation(onet, pts, vd) >= (1e-4 if cfg.precision == "bf16x3" else 3e-5)
    pts, vd = pts[keep].contiguous(), vd[keep].contiguous()
    n = pts.shape[0]
    assert n >= 600, f"only {n} samples clear of the ReLU kinks"
    d_raw = torch.randn(n, 4 + cfg.num_classes + cfg.num_instances, generator=g)
    net = net.to(DEV)
    got = network_backward(net, d_raw.to(DEV), pts=pts.to(DEV), viewdirs=vd.to(DEV), return_input_grad=True)
    assert net.range_status() == 0
    raw = onet(pts.double(), vd.double())
    raw.backward(d_raw.double())
    ref = {k: p.grad for k, p in onet.named_parameters()}
    assert set(ref) == set(got) - {"embedded_xyz"}
    tol = 2e-4 if cfg.precision == "bf16x3" else 1e-4
    for name, r in ref.items():
        assert got[name].shape == r.shape
        assert_close(got[name].cpu().double(), r, rms(r), f"{preset} {over} d/d{name}", rel=tol)
    # gradients of a mean-reduced loss are tiny: the same call with d_raw * 2^-20 gives the same gradients * 2^-20
    small = network_backward(net, (d_raw * 2.0 ** -20).to(DEV), pts=pts.to(DEV), viewdirs=vd.to(DEV))
    for name in ("pts_linears.0.weight", f"pts_linears.{cfg.D - 1}.bias", "rgb_linear.weight"):
        assert_close(small[name].cpu().double() * 2.0 ** 20, ref[name], rms(ref[name]), f"{preset} {over} small d/d{name}", rel=tol)


def test_training_step_through_the_fused_path_reduces_the_loss():
    """A few SGD steps on raw = net(pts, viewdirs) -> ||raw - target||^2, forward on the fused kernel, backward through
    network_backward: the loss goes down, and the first step's gradients equal torch autograd through the same modules."""
    from panopticnerf_b200.lib.train import network_forward_autograd
    from panopticnerf_b200.lib.train.mlp_backward import _tail
    cfg = make_cfg("cfg2", num_classes=5)
    net = S.init_network_weights(make_network(cfg), seed=4).to(DEV)
    g = torch.Generator().manual_seed(0)
    pts = ((torch.rand(4096, 3, generator=g) * 2 - 1) * 3).to(DEV)
    vd = torch.nn.functional.normalize(torch.randn(4096, 3, generator=g), dim=-1).to(DEV)
    target = torch.randn(4096, 4 + 5, generator=g).to(DEV) * 0.1
    opt = torch.optim.SGD(net.parameters(), lr=0.05)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        raw = network_forward_autograd(net, pts, vd)
        loss = ((raw - target) ** 2).mean()
        loss.backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in net.parameters())
        opt.step()
        losses.append(float(loss))
    assert all(b < a for a, b in zip(losses, losses[1:])) and losses[-1] < 0.97 * losses[0], losses


def test_training_step_end_to_end_matches_the_oracle_chain(record_d_raw):
    """rays -> MLP -> compositing -> losses and back to every parameter, all on the library's kernels, against the
    same chain of the oracle in float64 pinned to the ReLU, density and depth-sign decisions the step took
    (tests/oracle_pinned.py): every parameter's gradient element by element within 1e-4 of its RMS, the instance
    head's exactly zero."""
    from panopticnerf_b200.lib.train import training_step
    cfg = make_cfg("cfg3")
    net = S.init_network_weights(make_network(cfg), seed=21)
    g = torch.Generator().manual_seed(7)
    R, N, C = 96, 64, cfg.num_classes
    rays = torch.cat([torch.randn(R, 3, generator=g) * 0.5, torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)], -1)
    z = torch.sort(torch.rand(R, N, generator=g) * 6 + 0.5, -1).values
    batch = {"rgb": torch.rand(R, 3, generator=g), "depth": torch.rand(R, generator=g) * 6,
             "pseudo_label": torch.randint(-1, C, (R,), generator=g)}
    w = (1.0, 0.1, 0.5, 0.0)
    net = net.to(DEV)
    dbatch = {k: v.to(DEV) for k, v in batch.items()}
    total, terms = training_step(net, rays.to(DEV), z.to(DEV), dbatch, w)
    check_single_pass(cfg, net, rays.to(DEV), z.to(DEV), dbatch, w, total, record_d_raw, "training_step cfg3")
    assert float(net.instance_linears[1].weight.grad.abs().max()) == 0.0


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg3", {}), ("cfg2", dict(precision="bf16x3")), ("cfg1", dict(num_classes=5))])
def test_update_weights_equals_fresh_load(preset, over):
    """After an optimiser-like change of every parameter, the device-side refresh (pnr_update_weights: no host copy, no
    rebuild) gives bit for bit what a fresh context packed on the host gives - forward, trunk forward and trunk backward,
    whether the auxiliary programs existed before the update or are first built after it."""
    from panopticnerf_b200.lib.networks.panopticnerf.network import Network
    cfg = make_cfg(preset, **over)
    g = torch.Generator().manual_seed(1)
    n = 700
    pts = ((torch.rand(n, 3, generator=g) * 2 - 1) * 3).to(DEV)
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV)
    grad_h = torch.randn(n, cfg.W, generator=g).to(DEV)
    net = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
    late = S.init_network_weights(make_network(cfg), seed=5).to(DEV)      # its aux programs are first built AFTER the update
    net(pts, vd); net.trunk_forward(pts=pts); net.backward_trunk(grad_h, pts=pts)   # all three programs exist
    late(pts, vd)
    ctx_before = net._ctx
    with torch.no_grad():
        for k, (p, q) in enumerate(zip(net.parameters(), late.parameters())):
            d = torch.randn(p.shape, generator=torch.Generator().manual_seed(100 + k)).to(DEV) * 0.05
            p.add_(d); q.add_(d)
    got = (net(pts, vd), net.trunk_forward(pts=pts), net.backward_trunk(grad_h, pts=pts, grad_scale=64.0))
    assert net._ctx == ctx_before                           # refreshed in place
    got_late = (late(pts, vd), late.trunk_forward(pts=pts), late.backward_trunk(grad_h, pts=pts, grad_scale=64.0))
    Network._fast_update = False
    try:
        fresh = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
        fresh.load_state_dict(net.state_dict())
        ref = (fresh(pts, vd), fresh.trunk_forward(pts=pts), fresh.backward_trunk(grad_h, pts=pts, grad_scale=64.0))
    finally:
        Network._fast_update = True
    for a, b, c in zip(got, got_late, ref):
        assert torch.equal(a, c) and torch.equal(b, c)
    assert net.range_status() == 0


def test_backward_trunk_collects_the_stash_maxima():
    """The backward kernel reports the largest |value| of every stash slot (what scales the weight-gradient GEMMs):
    equal to a reduction over the stash itself up to the 11 bits of an fp16 hi part."""
    import panopticnerf_b200 as PN
    from panopticnerf_b200 import synthetic as S
    cfg = PN.make_cfg("cfg1")
    net = S.init_network_weights(PN.make_network(cfg)).to(DEV)
    g = torch.Generator().manual_seed(3)
    n = 1000
    pts = (torch.rand(n, 3, generator=g) * 2 - 1).to(DEV)
    grad_h = (torch.randn(n, net.W, generator=g) * 2e-6).to(DEV)
    _, st, mx = net.backward_trunk(grad_h, pts=pts, stash=True, absmax=True)
    ref = st.abs().amax(dim=(1, 2))
    assert mx.shape == ref.shape and torch.isfinite(mx).all()
    rel = ((mx - ref).abs() / ref.clamp(min=1e-30)).max()
    assert float(rel) <= 2.0 ** -10, f"stash maxima off by {float(rel):.2e}"
    # and the two ways of getting the GEMM scales agree
    from panopticnerf_b200.lib.train.mlp_backward import _pow2_scales, _pow2_from_max
    a, b = _pow2_scales(st[net.D - 1:]), _pow2_from_max(mx[net.D - 1:])
    assert all(float(x) in (float(y), 2 * float(y), 0.5 * float(y)) for x, y in zip(a, b))   # a rounding boundary apart at most


# ------------------------------------------------------------------------------------------------
# pnr_wgrad: the weight-gradient GEMM over the samples (csrc/wgrad_wgmma.cu) vs float64 on the CPU
# ------------------------------------------------------------------------------------------------
def _wgrad_case(S_, No, Ni, seed, gscale=1e-6):
    g = torch.Generator().manual_seed(seed)
    dz = torch.randn(S_, No, generator=g) * gscale * (0.1 + torch.rand(1, No, generator=g) * 3.0)   # gradients: tiny, uneven
    dz = dz * (torch.rand(S_, No, generator=g) < 0.6)                                              # ReLU-gated zeros
    x = torch.relu(torch.randn(S_, Ni, generator=g)) + 0.05 * torch.randn(S_, Ni, generator=g)
    return dz, x


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("S_,No,Ni", [(4096, 256, 256), (5000, 256, 63), (777, 128, 283), (33, 1, 256), (1, 3, 128),
                                      (20011, 45, 128), (148 * 32 * 3 + 5, 64, 319), (132 * 64 * 3 + 5, 64, 319),
                                      (31, 256, 16), (200, 130, 17)])
def test_wgrad_matches_float64(S_, No, Ni, prec):
    from panopticnerf_b200.lib.train.mlp_backward import wgrad, _pow2_scale
    dz, x = _wgrad_case(S_, No, Ni, seed=S_ + No + Ni)
    dzd = dz.to(DEV)
    dW, db = wgrad(dzd, x.to(DEV), precision=prec, scale=_pow2_scale(dzd) if prec == "fp16x3" else None)
    torch.cuda.synchronize()
    ref_W = dz.double().t() @ x.double()
    ref_b = dz.double().sum(0)
    eW = float((dW.cpu().double() - ref_W).abs().max() / rms(ref_W))
    eb = float((db.cpu().double() - ref_b).abs().max() / max(rms(ref_b), 1e-30))
    print(f"wgrad {prec} S={S_} No={No} Ni={Ni}: max err / rms  dW {eW:.2e}  db {eb:.2e}")
    # operand parts: fp16 ~2^-21 per product (measured model on the CPU: 5e-7 of the RMS), bf16 ~2^-17 (2.6e-5);
    # fp32 accumulation over the samples adds ~1e-6
    assert eW <= (2e-5 if prec == "fp16x3" else 1e-4), f"wgrad dW: {eW:.2e}"
    assert eb <= 1e-4, f"wgrad db: {eb:.2e}"


def test_wgrad_views_determinism_and_errors():
    from panopticnerf_b200.lib.train.mlp_backward import wgrad
    from panopticnerf_b200 import _capi
    dz, x = _wgrad_case(3000, 200, 300, seed=5)
    dzd, xd = dz.to(DEV), x.to(DEV)
    # column blocks of wider matrices are views with a row stride: no copies, same numbers as the contiguous blocks
    a_W, a_b = wgrad(dzd[:, 8:136], xd[:, 20:276])
    b_W, b_b = wgrad(dzd[:, 8:136].contiguous(), xd[:, 20:276].contiguous())
    assert torch.equal(a_W, b_W) and torch.equal(a_b, b_b)
    # deterministic: partial products are added in a fixed order
    c_W, c_b = wgrad(dzd, xd)
    d_W, d_b = wgrad(dzd, xd)
    assert torch.equal(c_W, d_W) and torch.equal(c_b, d_b)
    assert wgrad(dzd, xd, bias=False)[1] is None
    with pytest.raises(_capi.PnrError):
        wgrad(dz, x)                                  # CPU tensors: no fallback
    with pytest.raises(_capi.PnrError):
        wgrad(torch.zeros(10, 300, device=DEV), xd[:10])   # more than 256 output features
    # fp16 parts without the scale lose the ~1e-6 gradients (that is what `scale` is for); with it they beat bf16
    ref = dz.double().t() @ x.double()
    from panopticnerf_b200.lib.train.mlp_backward import _pow2_scale
    err = lambda W: float((W.cpu().double() - ref).abs().max() / rms(ref))
    e_bf, e_fp, e_raw = err(c_W), err(wgrad(dzd, xd, precision="fp16x3", scale=_pow2_scale(dzd))[0]), err(wgrad(dzd, xd, precision="fp16x3")[0])
    print(f"wgrad err/rms: bf16x3 {e_bf:.1e}  fp16x3 scaled {e_fp:.1e}  fp16x3 unscaled {e_raw:.1e}")
    assert e_fp < e_bf < 1e-4 and e_raw > 10 * e_fp
    # large magnitudes and exact zeros survive the bf16 split (fp32 exponent range)
    big = torch.full((64, 16), 3.0e30, device=DEV)
    one = torch.zeros(64, 16, device=DEV)
    one[:, 0] = 1.0e-3
    W, _ = wgrad(big, one)
    assert torch.isfinite(W).all() and abs(float(W[0, 0]) / (64 * 3.0e27) - 1.0) < 1e-4 and float(W[:, 1:].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------
# pnr_linear: y = act(x W^T + b) of the layers after the trunk on the training path (csrc/linear_wgmma.cu)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S_,K,N,relu,prec", [(4096, 256, 256, False, "fp16x3"), (1000, 283, 128, True, "fp16x3"),
                                             (130, 256, 1, False, "fp16x3"), (5000, 128, 45, False, "bf16x3"),
                                             (129, 128, 3, False, "fp16x3"), (148 * 128 * 2 + 77, 256, 128, True, "bf16x3"),
                                             (132 * 128 * 2 + 77, 256, 128, True, "bf16x3"),
                                             (7, 27, 64, False, "fp16x3"), (300, 512, 256, False, "fp16x3")])
def test_linear3x_matches_float64(S_, K, N, relu, prec):
    from panopticnerf_b200.lib.train.mlp_backward import linear3x
    g = torch.Generator().manual_seed(S_ + K + N)
    x = torch.randn(S_, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g) * 0.1
    y = linear3x(x.to(DEV), w.to(DEV), b.to(DEV), relu=relu, precision=prec)
    torch.cuda.synchronize()
    ref = x.double() @ w.double().t() + b.double()
    if relu:
        ref = ref.clamp(min=0)
    e = float((y.cpu().double() - ref).abs().max() / rms(ref))
    print(f"linear3x S={S_} K={K} N={N} relu={relu} {prec}: max err / rms {e:.2e}")
    tol_scale = 1.0 if prec == "fp16x3" else 2.0
    assert e <= 1e-4 * tol_scale, f"linear3x: {e:.2e}"


def test_linear3x_transposed_scaled_gradients_and_views():
    from panopticnerf_b200.lib.train.mlp_backward import linear3x, _pow2_scale
    from panopticnerf_b200 import _capi
    g = torch.Generator().manual_seed(11)
    S_, N, K = 3000, 128, 283                       # a layer y = x W^T with x [S, 283], W [128, 283]; gradient g [S, 128]
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    gy = (torch.randn(S_, N, generator=g) * 3e-7).to(DEV)          # a mean-reduced loss: ~1e-7
    sc = _pow2_scale(gy)
    assert float(sc) == 2.0 ** round(float(torch.log2(256.0 / gy.abs().max())))
    dx = linear3x(gy, w, transposed=True, precision="fp16x3", scale=sc)
    ref = gy.cpu().double() @ w.cpu().double()
    e = float((dx.cpu().double() - ref).abs().max() / rms(ref))
    print(f"linear3x dgrad fp16x3 scaled: max err / rms {e:.2e}")
    assert dx.shape == (S_, K) and e <= 1e-4
    # unscaled, the fp16 parts of such gradients are subnormal or zero: the scale is what keeps the product exact
    bad = linear3x(gy, w, transposed=True, precision="fp16x3")
    assert float((bad.cpu().double() - ref).abs().max() / rms(ref)) > 10 * e
    # the range-safe format needs no scale
    dxb = linear3x(gy, w, transposed=True, precision="bf16x3")
    assert float((dxb.cpu().double() - ref).abs().max() / rms(ref)) <= 2e-4
    # row-strided views (a column block of a wider matrix), deterministic
    wide = torch.randn(500, 300, generator=g).to(DEV)
    a = linear3x(wide[:, 10:266], w[:, :256].contiguous())
    b2 = linear3x(wide[:, 10:266].contiguous(), w[:, :256].contiguous())
    assert torch.equal(a, b2) and torch.equal(a, linear3x(wide[:, 10:266], w[:, :256].contiguous()))
    with pytest.raises(_capi.PnrError):
        linear3x(wide.cpu(), w.cpu())
    with pytest.raises(_capi.PnrError):
        linear3x(torch.zeros(8, 600, device=DEV), torch.zeros(16, 600, device=DEV))          # K > 512
    y300 = linear3x(wide, torch.eye(300, device=DEV))              # more than 256 outputs: column blocks
    assert float((y300 - wide).abs().max()) <= 1e-5 * float(wide.abs().max())
    assert _pow2_scale(torch.zeros(4, 4, device=DEV)).item() == 1.0
