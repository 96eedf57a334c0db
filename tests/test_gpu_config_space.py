"""GPU: the fused MLP kernel across the configuration space `pnr_create` accepts (the matrix of
tests/test_cpu_config_space.py: D in [3, 16], W in {64, 128, 256}, heads up to C = K = 128, xyz_res / view_res at 0 and
at their maximum, the four precisions, hash grids with padded E and F = 1 .. 8).  The reference is the oracle network
in float64, fed the same fp32 weights and inputs; the compositing epilogue is held to the two-kernel path, and the
device-side weight update to a fresh load.  Tolerances are those of tests/util.py and DESIGN §4."""
import pytest
import torch

from oracle import reference_renderer as O
from oracle_hashgrid import hash_cfg, oracle_like
from panopticnerf_b200 import make_cfg, make_network, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from test_cpu_config_space import FORWARD, GRIDS, _grid_cfg, _id
from test_cpu_hashgrid_network import _points as _grid_points
from test_cpu_program import assert_grad_close
from test_gpu_fused import _same
from util import assert_close, rel_err, rms

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# sample counts that cross the 64-row tile and the CTA boundaries: the last one is more tiles than an H100 SXM has SMs
# (132), twice over, plus a tail
COUNTS = [1, 63, 64, 65, 64 * 132 * 2 + 17]
REF_STRIDE = 17                                   # every 17th sample of the largest run goes to the float64 oracle
X3_TOL = {"fp16x3": 2e-5, "bf16x3": 1e-4}
FAST_BOUND = {"fp16": 1e-2, "bf16": 6e-2}          # the operand-precision bounds of test_cpu_program


def _oracle64(cfg, net_cpu):
    onet = O.Network(cfg).double()
    onet.load_state_dict({k: v.double() for k, v in net_cpu.state_dict().items()})
    return onet


def _inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    return pts, vd


def _dyadic_rays(R, N, seed):
    """Rays and depths whose points o + d*z are exact in fp32 (few mantissa bits): the kernel forms the same points as
    the oracle, whatever the order of its multiply-add."""
    g = torch.Generator().manual_seed(seed)
    o = torch.randint(-48, 49, (R, 3), generator=g).float() / 16
    d = torch.randint(-8, 9, (R, 3), generator=g).float() / 8
    d[(d == 0).all(-1), 0] = 1.0
    z = torch.randint(1, 17, (R, N), generator=g).float() / 16
    pts = (o[:, None] + d[:, None] * z[..., None]).reshape(-1, 3)
    vd = (d.double() / d.double().norm(dim=-1, keepdim=True))[:, None].expand(-1, N, -1).reshape(-1, 3)
    return torch.cat([o, d], -1), z, pts, vd


def _groups(cfg):
    C_, K_ = cfg.num_classes, cfg.num_instances
    g = {"rgb": slice(0, 3), "sigma": slice(3, 4)}
    if C_:
        g["sem"] = slice(4, 4 + C_)
    if K_:
        g["inst"] = slice(4 + C_, 4 + C_ + K_)
    return g


def _check(got, ref, cfg, what):
    """x3 modes: every output group within the parity tolerance of its RMS.  1-pass modes: above 1e-4 (they stay
    labelled "fast") and below their operand-precision bound."""
    got = got.cpu().double()
    if cfg.precision in X3_TOL:
        for name, sl in _groups(cfg).items():
            assert_close(got[:, sl], ref[:, sl], max(rms(ref[:, sl]), 1e-6), f"{what} {name}", X3_TOL[cfg.precision])
        return
    worst = max(rel_err(got[:, sl], ref[:, sl], max(rms(ref[:, sl]), 1e-6)) for sl in _groups(cfg).values())
    assert 1e-4 < worst <= FAST_BOUND[cfg.precision], f"{what}: {cfg.precision} error {worst:.3e}"


@pytest.mark.parametrize("over", FORWARD, ids=[_id(o) for o in FORWARD])
def test_forward_points_and_rays_over_the_accepted_space(over):
    """Network.forward (points) and forward_rays (points formed in the kernel) at sample counts across tile and CTA
    boundaries: shorter runs are prefixes of the longest bit for bit, two runs agree bit for bit, and a subset of the
    longest run matches the float64 oracle."""
    cfg = make_cfg("cfg2", **over)
    net_cpu = S.init_network_weights(make_network(cfg), seed=3)
    onet = _oracle64(cfg, net_cpu)
    net = net_cpu.to(DEV)
    n = COUNTS[-1]
    pts, vd = _inputs(n, seed=11)
    gp, gv = pts.to(DEV), vd.to(DEV)
    sub = torch.arange(0, n, REF_STRIDE)
    with torch.no_grad():
        full = net(gp, gv)
        assert torch.equal(net(gp, gv), full), "two runs differ"
        for m in COUNTS[:-1]:
            assert torch.equal(net(gp[:m].contiguous(), gv[:m].contiguous()), full[:m]), f"{m} samples: not a prefix"
        ref = onet(pts[sub].double(), vd[sub].double())
    _check(full[sub], ref, cfg, f"{over} points")
    # rays mode: R * N = the same counts (N = 13: rays straddle the tiles)
    rays, z, p3, d3 = _dyadic_rays(1301, 13, seed=12)
    assert rays.shape[0] * 13 == n
    gr, gz = rays.to(DEV), z.to(DEV)
    with torch.no_grad():
        raw = net.forward_rays(gr, gz)
        assert torch.equal(net.forward_rays(gr, gz), raw), "two runs differ (rays)"
        for R in (1, 5):
            assert torch.equal(net.forward_rays(gr[:R].contiguous(), gz[:R].contiguous()), raw[:R]), f"{R} rays: not a prefix"
        ref_r = onet(p3[sub].double(), d3[sub])
    _check(raw.reshape(n, -1)[sub], ref_r, cfg, f"{over} rays")
    if cfg.precision in X3_TOL:
        assert net.range_status() == 0


@pytest.mark.parametrize("k", range(len(GRIDS)), ids=[f"L{L}F{F}" for L, F in GRIDS])
def test_hashgrid_forward_over_the_accepted_grids(k):
    """The on-chip gather at F = 1, 2, 4, 8, L = 1 .. 32 and E = 1 .. 64 (zero padding up to the next 16 columns in layer 0
    and the skip layer): prefixes and reruns bit for bit, a subset against the float64 network fed h(x) of the fp32
    oracle encoder (bit-identical to the kernel's)."""
    cfg = _grid_cfg(k, hash_log2_size=14)
    net_cpu = S.init_network_weights(make_network(cfg), seed=3)
    on64 = oracle_like(net_cpu, cfg, torch.float64)
    n = COUNTS[-1]
    pts, vd = _grid_points(n, seed=11)
    sub = torch.arange(0, n, REF_STRIDE)
    with torch.no_grad():
        hx = oracle_like(net_cpu, cfg).xyz_encoder(pts[sub]).double()
        t = hx
        for i, lin in enumerate(on64.pts_linears):
            t = torch.relu(lin(t))
            if i == on64.skip:
                t = torch.cat([hx, t], -1)
        ed = O.embed(vd[sub].double(), on64.Ld)
        outs = [on64.rgb_linear(torch.relu(on64.views_linears[0](torch.cat([on64.feature_linear(t), ed], -1)))),
                on64.alpha_linear(t)]
        if cfg.num_classes:
            outs.append(on64.semantic_linears[1](torch.relu(on64.semantic_linears[0](t))))
        if cfg.num_instances:
            outs.append(on64.instance_linears[1](torch.relu(on64.instance_linears[0](t))))
        ref = torch.cat(outs, -1)
        net = net_cpu.to(DEV)
        gp, gv = pts.to(DEV), vd.to(DEV)
        full = net(gp, gv)
        assert torch.equal(net(gp, gv), full), "two runs differ"
        for m in COUNTS[:-1]:
            assert torch.equal(net(gp[:m].contiguous(), gv[:m].contiguous()), full[:m]), f"{m} samples: not a prefix"
    _check(full[sub], ref, cfg, f"L{cfg.hash_levels} F{cfg.hash_features} points")
    if cfg.precision in X3_TOL:
        assert net.range_status() == 0


COMPOSITE = [dict(num_classes=128, num_instances=128), dict(num_classes=1, num_instances=1),
             dict(num_classes=17, num_instances=113), dict(D=4, W=64, num_classes=17, num_instances=113),
             dict(hash=(5, 2), num_classes=3, num_instances=6)]


@pytest.mark.parametrize("N", [32, 96, 224])
@pytest.mark.parametrize("over", COMPOSITE, ids=[_id(o) for o in COMPOSITE])
def test_compositing_epilogue_matches_two_kernel_path(over, N):
    """pnr_mlp_composite against pnr_mlp_forward + pnr_composite with the largest composited channel count (5 + 128 +
    128), single channels, unequal merged heads, the separate-heads path (W = 64) and a hash grid with padded E:
    weights and the fixed maps bit for bit, the summed maps to fp32 rounding."""
    over = dict(over, N_samples=N, N_importance=0)
    grid = over.pop("hash", None)
    cfg = (hash_cfg("cfg2", hash_levels=grid[0], hash_features=grid[1], hash_log2_size=14, **over) if grid
           else make_cfg("cfg2", **over))
    net = S.init_network_weights(make_network(cfg), seed=4).to(DEV)
    R = 301
    full = S.make_batch(cfg, row0=cfg.H // 3, rows=1)
    rays = full["rays"][:R].contiguous().to(DEV)
    near, far = P.scene_near_far(rays, full["scene_aabb"], cfg.near, cfg.far)
    hit, bid, tin, tout = P.intersect(rays, full["box_center"].to(DEV), full["box_half"].to(DEV), full["box_rot"].to(DEV), 4)
    z, sb = P.stratified_z(near, far, torch.linspace(0, 1, N).to(DEV), 0.0, None, bid, tin, tout, want_tags=True)
    kw = dict(sample_box=sb, box_sem=full["box_sem"].to(DEV), box_inst=full["box_inst"].to(DEV))
    got = net.forward_composite(rays, z, **kw)
    raw = net.forward_rays(rays, z)
    ref = P.raw2outputs(raw, z, rays, num_classes=cfg.num_classes, num_instances=cfg.num_instances, **kw)
    assert got.keys() == ref.keys()
    for k in ("weights", "fixed_semantic_map", "fixed_instance_map"):
        assert torch.equal(got[k], ref[k]), k
    _same(got, ref, summed_exact=False)
    assert float(got["weights"].sum()) > 0 and net.range_status() == 0


TRUNK = [dict(D=9), dict(D=3), dict(D=9, W=64), dict(D=4, W=128, precision="bf16x3"),
         dict(D=9, W=256, xyz_res=0, precision="bf16x3"), dict(D=3, W=64, xyz_res=0),
         dict(hash=(5, 2)), dict(hash=(3, 8), D=3, W=64), dict(hash=(8, 1), D=9, W=128, precision="bf16x3"),
         dict(hash=(8, 8), D=5, W=256)]


def _trunk_cfg(over):
    over = dict(over)
    grid = over.pop("hash", None)
    if grid:
        return hash_cfg("cfg2", hash_levels=grid[0], hash_features=grid[1], hash_log2_size=14, **over)
    return make_cfg("cfg2", **over)


def _trunk64(cfg, net_cpu, pts, grad_h):
    """float64 trunk output h, dL/d(trunk input) by autograd and the smallest |pre-activation| per sample; the trunk input
    is gamma(x), or h(x) from the fp32 oracle encoder (bit-identical to the kernel's on-chip gather)."""
    if getattr(cfg, "xyz_encoding", "frequency") == "hashgrid":
        onet = oracle_like(net_cpu, cfg, torch.float64)
        with torch.no_grad():
            ex = oracle_like(net_cpu, cfg).xyz_encoder(pts).double()
    else:
        onet, ex = _oracle64(cfg, net_cpu), O.embed(pts, cfg.xyz_res).double()
    x = ex.clone().requires_grad_(True)
    h, min_z = x, torch.full((pts.shape[0],), float("inf"), dtype=torch.float64)
    for i, lin in enumerate(onet.pts_linears):
        pre = lin(h)
        min_z = torch.minimum(min_z, pre.detach().abs().min(dim=1).values)
        h = torch.relu(pre)
        if i == onet.skip:
            h = torch.cat([x, h], -1)
    h.backward(grad_h.double())
    return h.detach(), x.grad, min_z


@pytest.mark.parametrize("over", TRUNK, ids=[_id(o) for o in TRUNK])
def test_trunk_backward_forward_and_stash_maxima(over):
    """pnr_mlp_backward_trunk against float64 autograd, pnr_mlp_trunk_forward against the float64 trunk, and the stash
    maxima against the stash they describe: slot k holds the 16-bit hi-part bit pattern of the largest |value| the
    kernel put there, taken before the division by grad_scale for the gradient slots (k >= D-1)."""
    cfg = _trunk_cfg(over)
    net_cpu = S.init_network_weights(make_network(cfg), seed=2)
    n = 1000
    pts = _grid_points(n, seed=3)[0] if getattr(cfg, "xyz_encoding", "") == "hashgrid" else _inputs(n, seed=3)[0]
    grad_h = torch.randn(n, cfg.W, generator=torch.Generator().manual_seed(4))
    h_ref, g_ref, min_z = _trunk64(cfg, net_cpu, pts, grad_h)
    net = net_cpu.to(DEV)
    gs = 64.0
    got, stash, mx = net.backward_trunk(grad_h.to(DEV), pts=pts.to(DEV), stash=True, absmax=True, grad_scale=gs)
    h = net.trunk_forward(pts=pts.to(DEV))
    assert net.range_status() == 0
    kink = {"fp16x3": 1e-5, "bf16x3": 3e-5}[cfg.precision]
    assert_grad_close(got.cpu().double(), g_ref, min_z, f"{over} d(trunk input)", 1e-4, kink)
    assert_close(h.cpu().double(), h_ref, rms(h_ref), f"{over} trunk forward", X3_TOL[cfg.precision])
    # the stash maxima, bit for bit
    half = torch.float16 if cfg.precision.startswith("fp16") else torch.bfloat16
    scale = torch.ones(2 * cfg.D - 1, device=DEV)
    scale[cfg.D - 1:] = gs
    want = (stash.abs().amax(dim=(1, 2)) * scale).to(half).float() / scale
    assert mx.shape == want.shape and torch.equal(mx, want), (mx, want)


UPDATE = [dict(precision="fp16"), dict(D=13, W=128, precision="bf16", num_classes=17, num_instances=113),
          dict(num_classes=128, num_instances=128), dict(D=16, num_classes=128, num_instances=128),
          dict(D=9, W=64, xyz_res=0, precision="bf16x3", num_classes=1), dict(hash=(5, 2), num_classes=3),
          dict(hash=(8, 8), D=4, W=128, precision="bf16x3"), dict(hash=(3, 8), D=3, W=64, precision="bf16")]


@pytest.mark.parametrize("over", UPDATE, ids=[_id(o) for o in UPDATE])
def test_update_weights_equals_fresh_load(over):
    """After an optimiser-like change of every parameter, pnr_update_weights (no host copy, no rebuild) gives bit for bit
    what a fresh pnr_load_weights gives: forward, and, where the network has them (x3 modes, D <= 9), trunk forward and
    trunk backward - whether they existed before the update or are first built after it."""
    from panopticnerf_b200.lib.networks.panopticnerf.network import Network
    cfg = _trunk_cfg(over)
    aux = cfg.precision.endswith("x3") and cfg.D <= 9
    g = torch.Generator().manual_seed(1)
    n = 700
    pts = (_grid_points(n, seed=2)[0] if getattr(cfg, "xyz_encoding", "") == "hashgrid" else _inputs(n, seed=2)[0]).to(DEV)
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).to(DEV)
    grad_h = torch.randn(n, cfg.W, generator=g).to(DEV)

    def outputs(m):
        out = (m(pts, vd),)
        return out + ((m.trunk_forward(pts=pts), m.backward_trunk(grad_h, pts=pts, grad_scale=64.0)) if aux else ())
    net = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
    late = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
    outputs(net)                                  # every program exists before the update
    late(pts, vd)                                 # only the forward program
    ctx = net._ctx
    with torch.no_grad():
        for k, (p, q) in enumerate(zip(net.parameters(), late.parameters())):
            d = torch.randn(p.shape, generator=torch.Generator().manual_seed(100 + k)).to(DEV) * 0.05
            p.add_(d)
            q.add_(d)
    got, got_late = outputs(net), outputs(late)
    assert net._ctx == ctx
    Network._fast_update = False
    try:
        fresh = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
        fresh.load_state_dict(net.state_dict())
        ref = outputs(fresh)
    finally:
        Network._fast_update = True
    for a, b, c in zip(got, got_late, ref):
        assert torch.equal(a, c) and torch.equal(b, c)
    assert net.range_status() & 2 == 0
