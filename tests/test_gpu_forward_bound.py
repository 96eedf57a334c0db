"""GPU: the fused MLP forward element by element against the float64 bound of tests/oracle_bound.py, in the regimes of
tests/test_cpu_operand_split.py (default init; trunk layers twinned down by 2^4 .. 2^16 and up to the fp16 range;
hash tables of +-1e-4, +-1e-2, +-1; KITTI-360 world coordinates) and the four precisions.

Entry points: Network.forward (points) at sample counts across the tile and CTA tails, forward_rays (points and
directions formed in the kernel), the 128-row and the 64-row tile kernels (bit for bit the same), trunk_forward (x3
modes), and a network with heads.  Every sample of every run is compared; NaN patterns must coincide.  The worst
|err| / B per regime, entry point, precision and output group is printed (pytest -s)."""
import pytest
import torch

from oracle_bound import VIEWDIR_REL, forward_bound, view_encoding
from panopticnerf_b200 import _capi
from test_cpu_operand_split import REGIMES, apply_twin, make_regime, ratio, regime_points, trunk_input
from test_gpu_config_space import _dyadic_rays

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRECISIONS = ["fp16x3", "bf16x3", "fp16", "bf16"]
N = 64 * 132 * 2 + 17                  # more 64-row tiles than an H100 SXM has SMs, twice over, plus a tail
COUNTS = [1, 63, 64, 65, 127, 129]     # shorter runs: prefixes of the same samples


def _report(what, got, ref, B, groups):
    r = ratio(got.double(), ref, B)
    worst = {g: float(r[:, sl].max()) for g, sl in groups.items()}
    print(f"BOUND {what}: " + " ".join(f"{g}={v:.3g}" for g, v in worst.items()))
    assert max(worst.values()) <= 1.0, f"{what}: an element outside the bound: {worst}"


def _groups(C, K):
    g = {"rgb": slice(0, 3), "sigma": slice(3, 4)}
    if C:
        g["sem"] = slice(4, 4 + C)
    if K:
        g["inst"] = slice(4 + C, 4 + C + K)
    return g


def _setup(precision, regime, **over):
    cfg, net = make_regime(precision, regime, **over)
    pts, vd = regime_points(regime, N, seed=11)
    ex, e_ex = trunk_input(cfg, net, pts)
    net, k = apply_twin(net, regime, ex)
    return cfg, net, k, pts, vd, ex, e_ex


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_forward_within_the_bound(regime, precision):
    cfg, net, k, pts, vd, ex, e_ex = _setup(precision, regime)
    name = f"{regime[0]} k={k} {precision}"
    groups = _groups(0, 0)
    ed, e_ed = view_encoding(vd, cfg.view_res)
    ref, B, h_ref, h_B = forward_bound(net, precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV))
    net = net.to(DEV)
    gp, gv = pts.to(DEV), vd.to(DEV)
    with torch.no_grad():
        full = net(gp, gv)
        _report(f"{name} points", full, ref, B, groups)
        for m in COUNTS:
            assert torch.equal(net(gp[:m].contiguous(), gv[:m].contiguous()), full[:m]), f"{name}: {m} samples"
        # the 64-row kernel gives the 128-row kernel's bits
        _capi.set_mlp_rows(net.pack(), 64)
        try:
            assert torch.equal(net(gp, gv), full), f"{name}: the 64- and 128-row kernels differ"
        finally:
            _capi.set_mlp_rows(net.pack(), 0)
        if precision.endswith("x3"):
            h = net.trunk_forward(pts=gp)
            _report(f"{name} trunk_forward", h, h_ref, h_B, {"h": slice(0, cfg.W)})
    assert net.range_status() == 0, f"{name}: range check"
    # rays: points o + d z exact in fp32 (KITTI-360: origins up to 300 m), directions normalised in the kernel
    if regime[1] is None:
        rays, z, p3, d3 = _dyadic_rays(1301, 13, seed=12)
        rays[:, :3] *= regime[2] / 3.0 if regime[2] > 4 else 1.0
        rays[:, :3] = torch.round(rays[:, :3] * 16) / 16
        p3 = (rays[:, None, :3].double() + rays[:, None, 3:].double() * z[..., None].double()).reshape(-1, 3).float()
    else:
        pr, vr = regime_points(regime, 1301, seed=12)
        d = torch.round(vr * 8) / 8
        d[(d == 0).all(-1), 0] = 1.0
        z = torch.randint(1, 17, (1301, 13), generator=torch.Generator().manual_seed(13)).float() / 16
        rays = torch.cat([torch.round(pr * 16) / 16 - 2.0, d], -1)
        p3 = (rays[:, None, :3].double() + rays[:, None, 3:].double() * z[..., None].double()).reshape(-1, 3).float()
        d3 = (d.double() / d.double().norm(dim=-1, keepdim=True))[:, None].expand(-1, 13, -1).reshape(-1, 3)
    assert torch.equal(p3.double(), (rays[:, None, :3].double() + rays[:, None, 3:].double() * z[..., None].double()).reshape(-1, 3))
    ex3, e_ex3 = trunk_input(cfg, net, p3)
    ed3, e_ed3 = view_encoding(d3, cfg.view_res, rel=VIEWDIR_REL)
    ref3, B3, _, _ = forward_bound(net, precision, ex3.to(DEV), e_ex3.to(DEV), ed3.to(DEV), e_ed3.to(DEV))
    net = net.to(DEV)
    with torch.no_grad():
        raw = net.forward_rays(rays.to(DEV), z.to(DEV))
    _report(f"{name} rays", raw.reshape(-1, raw.shape[-1]), ref3, B3, groups)
    assert net.range_status() == 0


HEAD_REGIMES = [r for r in REGIMES if r[0] in ("default", "down-last-k12", "down-last-k16", "up-last", "table-0.0001")]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("regime", HEAD_REGIMES, ids=[r[0] for r in HEAD_REGIMES])
def test_forward_with_heads_within_the_bound(regime, precision):
    """Semantic and instance heads (their hidden layers merged into one step, the logits as two halves of the next)."""
    cfg, net, k, pts, vd, ex, e_ex = _setup(precision, regime, num_classes=5, num_instances=7)
    ed, e_ed = view_encoding(vd, cfg.view_res)
    ref, B, _, _ = forward_bound(net, precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV))
    net = net.to(DEV)
    with torch.no_grad():
        full = net(pts.to(DEV), vd.to(DEV))
    _report(f"heads {regime[0]} k={k} {precision} points", full, ref, B, _groups(5, 7))
    assert net.range_status() == 0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_default_network_within_the_bound(precision):
    """The library's default network (D = 8, W = 256) at the default init: the bound through eight layers."""
    regime = REGIMES[0]
    cfg, net, k, pts, vd, ex, e_ex = _setup(precision, regime, D=8)
    ed, e_ed = view_encoding(vd, cfg.view_res)
    ref, B, h_ref, h_B = forward_bound(net, precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV), chunk=256)
    net = net.to(DEV)
    with torch.no_grad():
        full = net(pts.to(DEV), vd.to(DEV))
    _report(f"D8 default {precision} points", full, ref, B, _groups(0, 0))
