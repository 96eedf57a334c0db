"""GPU: the hash-grid trunk input (cfg.xyz_encoding = "hashgrid"), gathered on chip by the fused MLP kernel - forward,
compositing, rendering, backward, training, table updates and errors - against the oracle hash-grid network
(tests/oracle_hashgrid.py) and the library's own two-kernel paths.  Tolerances are those of tests/util.py."""
import pytest
import torch

import panopticnerf_b200 as PN
from oracle import reference_renderer as O
from oracle_hashgrid import hash_cfg, oracle_like
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from test_cpu_program import assert_grad_close
from test_gpu_fused import _same
from test_gpu_train_chain import check_single_pass, record_d_raw  # noqa: F401 (record_d_raw: a fixture)
from util import REL, assert_close, check_render_outputs, rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _samples(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(S.SCENE_AABB[0]), torch.tensor(S.SCENE_AABB[1])
    pts = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    d = torch.randn(n, 3, generator=g)
    return pts, d / d.norm(dim=-1, keepdim=True)


def _rays(cfg, R, seed=0):
    batch = S.make_batch(cfg, row0=cfg.H // 3, rows=R // cfg.W_img + 1)
    rays = batch["rays"][:R].contiguous()
    near, far = O.scene_near_far(rays[:, :3], rays[:, 3:], torch.tensor(S.SCENE_AABB), cfg.near, cfg.far)
    z = O.stratified_z(near, far, torch.linspace(0, 1, cfg.N_samples))
    return rays, z.contiguous(), batch


def _check_raw(raw, ref, C, K, what, rel=REL):
    groups = {"rgb_raw": slice(0, 3), "sigma_raw": slice(3, 4)}
    if C:
        groups["sem"] = slice(4, 4 + C)
    if K:
        groups["inst"] = slice(4 + C, 4 + C + K)
    for name, sl in groups.items():
        assert_close(raw[..., sl].cpu(), ref[..., sl], max(rms(ref[..., sl]), 1e-6), f"{what} {name}", rel)


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("preset,over", [("cfg1", dict(hash_log2_size=14)), ("cfg2", {})], ids=["cfg1", "cfg2"])
def test_forward_matches_oracle(preset, over, precision):
    """Network.forward (points) and forward_rays (points formed in the kernel) against the oracle; two runs agree bit
    for bit; the standalone encoder equals the oracle's h(x) bit for bit, and the trunk output of the on-chip path
    equals the float64 trunk fed that h(x)."""
    cfg = hash_cfg(preset, precision=precision, **over)
    net = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
    onet = oracle_like(net, cfg)
    pts, vd = _samples(2000)
    with torch.no_grad():
        ref = onet(pts, vd)
        raw = net(pts.to(DEV), vd.to(DEV))
        raw2 = net(pts.to(DEV), vd.to(DEV))
    assert torch.equal(raw, raw2)
    assert net.range_status() == 0
    _check_raw(raw, ref, 0, 0, f"{preset} {precision} pts")
    rays, z, _ = _rays(cfg, 60)
    with torch.no_grad():
        p3 = (rays[:, None, :3] + rays[:, None, 3:] * z[..., None]).reshape(-1, 3)
        d3 = (rays[:, 3:] / rays[:, 3:].norm(dim=-1, keepdim=True))[:, None].expand(-1, z.shape[1], -1).reshape(-1, 3)
        ref_r = onet(p3, d3).reshape(rays.shape[0], z.shape[1], -1)
        got_r = net.forward_rays(rays.to(DEV), z.to(DEV))
    _check_raw(got_r, ref_r, 0, 0, f"{preset} {precision} rays")
    # the trunk output the backward path uses (pnr_mlp_trunk_forward, on chip) = the trunk fed pnr_hashgrid_encode's h(x)
    if precision == "fp16x3":
        h = net.trunk_forward(pts=pts.to(DEV))
        with torch.no_grad():
            ex = onet.xyz_encoder(pts).double()
            hx = net.xyz_encoder(pts.to(DEV)).cpu().double()
            assert torch.equal(hx, ex)                        # the standalone encoder is the oracle, bit for bit
            t = ex
            on64 = oracle_like(net, cfg, torch.float64)
            for i, lin in enumerate(on64.pts_linears):
                t = torch.relu(lin(t))
                if i == on64.skip:
                    t = torch.cat([ex, t], -1)
        assert_close(h.cpu().double(), t, rms(t), f"{preset} trunk output", REL)


def test_compositing_matches_two_kernel_path():
    """pnr_mlp_composite on a cfg3 hash-grid network (heads) against pnr_mlp_forward + pnr_composite: weights and the
    fixed maps bit for bit, the summed maps to fp32 rounding."""
    cfg = hash_cfg("cfg3", N_importance=0)
    net = S.init_network_weights(PN.make_network(cfg), seed=4).to(DEV)
    full = S.make_batch(cfg, row0=cfg.H // 3, rows=2)
    R = 1500
    rays = full["rays"][:R].contiguous().to(DEV)
    near, far = P.scene_near_far(rays, full["scene_aabb"], cfg.near, cfg.far)
    hit, bid, tin, tout = P.intersect(rays, full["box_center"].to(DEV), full["box_half"].to(DEV), full["box_rot"].to(DEV), 4)
    z, sb = P.stratified_z(near, far, torch.linspace(0, 1, cfg.N_samples).to(DEV), 0.0, None, bid, tin, tout, want_tags=True)
    kw = dict(sample_box=sb, box_sem=full["box_sem"].to(DEV), box_inst=full["box_inst"].to(DEV))
    got = net.forward_composite(rays, z, **kw)
    raw = net.forward_rays(rays, z)
    ref = P.raw2outputs(raw, z, rays, num_classes=cfg.num_classes, num_instances=cfg.num_instances, **kw)
    for k in ("weights", "fixed_semantic_map", "fixed_instance_map"):
        assert torch.equal(got[k], ref[k]), k
    _same(got, ref, summed_exact=False)
    assert float(got["weights"].sum()) > 0 and net.range_status() == 0


def test_render_fused_equals_staged_chunk_invariant_and_matches_oracle():
    cfg = hash_cfg("cfg2", N_importance=32, num_classes=5)
    net = S.init_network_weights(PN.make_network(cfg), seed=2).to(DEV)
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, rows=3).items()}
    R = batch["rays"].shape[0]
    staged = PN.make_renderer(hash_cfg("cfg2", N_importance=32, num_classes=5, render_path="staged"), net).render(batch)
    fused = PN.make_renderer(cfg, net).render(batch)
    _same(fused, staged, summed_exact=False)
    _same(PN.make_renderer(hash_cfg("cfg2", N_importance=32, num_classes=5, gpu_chunk=R // 7 + 3), net).render(batch), fused,
          "chunked: ")
    # coarse + fine on a strip against the oracle renderer
    cfo = hash_cfg("cfg3", N_samples=64, N_importance=64, hash_log2_size=15)
    netf = S.init_network_weights(PN.make_network(cfo), seed=5)
    strip = S.make_batch(cfo, row0=200, rows=1)
    strip = {k: (v[::11].contiguous() if k == "rays" else v) for k, v in strip.items()}
    ref = O.make_renderer(cfo, oracle_like(netf, cfo)).render(strip)
    out = PN.make_renderer(cfo, netf.to(DEV)).render({k: v.to(DEV) for k, v in strip.items()})
    for k in ("hit_mask", "box_id", "z_vals_0"):
        assert torch.equal(out[k].cpu().to(ref[k].dtype), ref[k]), k
    check_render_outputs(out, {k: v for k, v in ref.items() if k.endswith("_0")}, float(ref["far"].max()))


@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg1", dict(D=5, W=128, hash_levels=16, hash_features=4))])
def test_backward_trunk_and_every_parameter(preset, over):
    """dL/dh(x) from backward_trunk against float64 autograd; then every parameter's gradient, the table's included,
    against float64 autograd through the oracle network, on samples clear of the ReLU kinks."""
    from panopticnerf_b200.lib.train import network_backward
    cfg = hash_cfg(preset, hash_log2_size=15, **over)
    net = S.init_network_weights(PN.make_network(cfg), seed=11)
    onet = oracle_like(net, cfg, torch.float64)
    n = 3000
    pts, vd = _samples(n, seed=3)
    g = torch.Generator().manual_seed(8)
    # dL/dh(x) through the trunk
    grad_h = torch.randn(n, cfg.W, generator=g)
    with torch.no_grad():
        hx = onet.xyz_encoder(pts)
    ex = hx.clone().requires_grad_(True)
    h, min_z = ex, torch.full((n,), float("inf"), dtype=torch.float64)
    for i, lin in enumerate(onet.pts_linears):
        pre = lin(h)
        min_z = torch.minimum(min_z, pre.detach().abs().min(dim=1).values)
        h = torch.relu(pre)
        if i == onet.skip:
            h = torch.cat([ex, h], -1)
    h.backward(grad_h.double())
    net = net.to(DEV)
    got = net.backward_trunk(grad_h.to(DEV), pts=pts.to(DEV)).cpu()
    assert got.shape == (n, net.in_dim)
    assert_grad_close(got.double(), ex.grad, min_z, f"{preset} dL/dh(x)", 1e-4, 1e-5)
    # every parameter, on the samples whose pre-activations (trunk and view layer) stay clear of zero
    onet.zero_grad()
    with torch.no_grad():
        view_pre = onet.views_linears[0](torch.cat([onet.feature_linear(h), O.embed(vd.double(), onet.Ld)], -1))
    keep = torch.minimum(min_z, view_pre.abs().min(dim=1).values) >= 3e-5
    assert int(keep.sum()) >= 600
    pts_k, vd_k = pts[keep].contiguous(), vd[keep].contiguous()
    d_raw = torch.randn(pts_k.shape[0], 4, generator=g)
    res = network_backward(net, d_raw.to(DEV), pts=pts_k.to(DEV), viewdirs=vd_k.to(DEV))
    assert net.range_status() == 0
    onet(pts_k.double(), vd_k.double()).backward(d_raw.double())
    ref = {k: p.grad for k, p in onet.named_parameters()}
    assert set(ref) == set(res) and "xyz_encoder.table" in ref
    for name, r in ref.items():
        assert res[name].shape == r.shape, name
        assert_close(res[name].cpu().double(), r, rms(r), f"{preset} d/d{name}", rel=1e-4)


def test_training_step_matches_oracle_chain_and_sgd_reduces_the_loss(record_d_raw):
    """The training step of a hash-grid network against the float64 oracle chain pinned to the step's decisions
    (tests/oracle_pinned.py): every gradient, the table's included, element by element within 1e-4 of its RMS."""
    from panopticnerf_b200.lib.train import training_step
    cfg = hash_cfg("cfg3", hash_log2_size=15)
    net = S.init_network_weights(PN.make_network(cfg), seed=21)
    g = torch.Generator().manual_seed(7)
    R, N, C = 96, 64, cfg.num_classes
    lo = torch.tensor(S.SCENE_AABB[0])
    rays = torch.cat([lo + torch.tensor([16.0, 8.0, 4.0]) + torch.randn(R, 3, generator=g) * 0.5,
                      torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)], -1)
    z = torch.sort(torch.rand(R, N, generator=g) * 6 + 0.5, -1).values
    batch = {"rgb": torch.rand(R, 3, generator=g), "depth": torch.rand(R, generator=g) * 6,
             "pseudo_label": torch.randint(-1, C, (R,), generator=g)}
    w = (1.0, 0.1, 0.5, 0.0)
    net = net.to(DEV)
    dbatch = {k: v.to(DEV) for k, v in batch.items()}
    total, _ = training_step(net, rays.to(DEV), z.to(DEV), dbatch, w)
    check_single_pass(cfg, net, rays.to(DEV), z.to(DEV), dbatch, w, total, record_d_raw, "training_step hash grid")
    # a few SGD steps (the table updated in place between launches) reduce the loss
    opt = torch.optim.SGD(net.parameters(), lr=0.05)
    losses = []
    for _ in range(5):
        opt.zero_grad()
        total, _ = training_step(net, rays.to(DEV), z.to(DEV), dbatch, w)
        opt.step()
        losses.append(float(total))
    assert all(b < a for a, b in zip(losses, losses[1:])), losses


def test_table_updates_are_seen_by_the_next_launch():
    """After an in-place table update, and after replacing the parameter tensor, a render equals that of a freshly
    built network with the same parameters, bit for bit."""
    cfg = hash_cfg("cfg1", hash_log2_size=14, num_classes=3)
    net = S.init_network_weights(PN.make_network(cfg), seed=6).to(DEV)
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, rows=8).items()}
    ren = PN.make_renderer(cfg, net)
    before = ren.render(batch)

    def fresh_render():
        f = PN.make_network(cfg)
        f.load_state_dict(net.state_dict())
        return PN.make_renderer(cfg, f.to(DEV)).render(batch)

    with torch.no_grad():
        net.xyz_encoder.table.mul_(-0.5).add_(0.1)               # in place: same tensor, same pointer
    after = ren.render(batch)
    assert not torch.equal(after["rgb_map"], before["rgb_map"])
    _same(after, fresh_render(), "in place: ")
    net.xyz_encoder.table = torch.nn.Parameter(torch.rand_like(net.xyz_encoder.table) * 2 - 1)   # a new tensor
    replaced = ren.render(batch)
    assert not torch.equal(replaced["rgb_map"], after["rgb_map"])
    _same(replaced, fresh_render(), "replaced: ")


def test_errors_no_table_and_fp16_range():
    cfg = hash_cfg("cfg1", hash_log2_size=12)
    net = S.init_network_weights(PN.make_network(cfg), seed=0).to(DEV)
    pts, vd = _samples(300)
    pts, vd = pts.to(DEV), vd.to(DEV)
    ctx = net.pack(torch.device(DEV))
    L = _capi.lib()
    _capi.check(L.pnr_bind_hashgrid_table(ctx, None))
    raw = torch.empty(300, 4, device=DEV)
    rc = L.pnr_mlp_forward(ctx, pts.data_ptr(), vd.data_ptr(), None, None, 300, 1, raw.data_ptr(), _capi.stream_ptr())
    assert rc == -3 and b"table" in L.pnr_last_error()                  # PNR_ERR_STATE
    h = torch.empty(300, cfg.W, device=DEV)
    rc = L.pnr_mlp_trunk_forward(ctx, pts.data_ptr(), None, None, 300, 1, h.data_ptr(), _capi.stream_ptr())
    assert rc == -3
    net(pts, vd)                                                         # pack() binds the table again
    assert net.range_status() == 0
    with torch.no_grad():
        net.xyz_encoder.table.fill_(1e5)                                 # features of 1e5: outside the fp16 range
    net(pts, vd)
    with pytest.raises(_capi.PnrError, match="range"):
        net.check_range()
    plain = S.init_network_weights(PN.make_network(PN.make_cfg("cfg1")), seed=0).to(DEV)
    assert L.pnr_bind_hashgrid_table(plain.pack(torch.device(DEV)), None) == -3   # not a hash-grid context
