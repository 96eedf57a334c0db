"""GPU: the 128-row fused MLP kernel (two consumer warpgroups on 128-sample tiles, forward programs without heads) against
the 64-row kernel on the same context and inputs: raw rows bit for bit at every tile tail, in every precision and with
the hash-grid trunk input, the range check, and a CUDA graph replay.  pnr_set_mlp_rows picks the kernel."""
import pytest
import torch

import panopticnerf_b200 as PN
from oracle_hashgrid import hash_cfg
from panopticnerf_b200 import _capi, make_cfg, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _net(cfg, seed=0):
    return S.init_network_weights(PN.make_network(cfg), seed).to(DEV)


def _samples(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(S.SCENE_AABB[0]), torch.tensor(S.SCENE_AABB[1])
    pts = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    d = torch.randn(n, 3, generator=g)
    return pts.to(DEV), (d / d.norm(dim=-1, keepdim=True)).to(DEV)


def _run(net, rows, fn):
    _capi.set_mlp_rows(net.pack(), rows)
    try:
        with torch.no_grad():
            return fn()
    finally:
        _capi.set_mlp_rows(net.pack(), 0)


def _same_bits(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), \
        f"{what}: {int((a.view(torch.int32) != b.view(torch.int32)).any(-1).sum())} rows differ"


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


CFGS = {
    "cfg2_fp16x3": lambda: make_cfg("cfg2"),
    "cfg2_bf16x3": lambda: make_cfg("cfg2", precision="bf16x3"),
    "cfg2_fp16": lambda: make_cfg("cfg2", precision="fp16"),
    "cfg2_bf16": lambda: make_cfg("cfg2", precision="bf16"),
    "hashgrid_fp16x3": lambda: hash_cfg("cfg2"),
    "hashgrid_bf16x3": lambda: hash_cfg("cfg2", precision="bf16x3"),
}


@pytest.mark.parametrize("name", list(CFGS))
def test_raw_rows_equal_the_64_row_kernel(name):
    """Every tail of the 128-sample tile (warpgroup 1 partly or not at all in the last tile), fewer tiles than SMs, and
    several tiles per CTA; the default routing takes the 128-row kernel."""
    net = _net(CFGS[name]())
    sms = _sms()
    sizes = [1, 63, 64, 65, 127, 128, 129, 128 * 5 + 40, 128 * 7 + 64, 128 * (sms // 2) + 100, 128 * 3 * sms + 77]
    pts, vd = _samples(max(sizes), seed=3)
    for n in sizes:
        a = _run(net, 64, lambda: net(pts[:n], vd[:n]))
        b = _run(net, 128, lambda: net(pts[:n], vd[:n]))
        _same_bits(b, a, f"{name} S={n}")
        assert torch.isfinite(b).all(), f"{name} S={n}"
    c = _run(net, 0, lambda: net(pts, vd))
    _same_bits(c, b, f"{name} default routing")


def test_cfg2_frame_equals_the_64_row_kernel():
    """The bench frame: 376 x 1408 rays x 64 samples, points formed in the kernel."""
    cfg = make_cfg("cfg2")
    net = _net(cfg)
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg).items()}
    rays = batch["rays"]
    near, far = P.scene_near_far(rays, batch["scene_aabb"], cfg.near, cfg.far)
    z = P.stratified_z(near, far, torch.linspace(0, 1, cfg.N_samples).to(DEV))
    a = _run(net, 64, lambda: net.forward_rays(rays, z))
    b = _run(net, 128, lambda: net.forward_rays(rays, z))
    assert b.shape[0] * b.shape[1] > 30_000_000
    _same_bits(b.reshape(-1, 4), a.reshape(-1, 4), "cfg2 frame")
    assert net.range_status() == 0


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
def test_nan_input_sets_the_status_on_both_kernels(precision):
    net = _net(make_cfg("cfg2", precision=precision))
    pts, vd = _samples(1000, seed=5)
    pts[700, 1] = float("nan")
    out = {}
    for rows in (64, 128):
        net.range_status(reset=True)
        out[rows] = _run(net, rows, lambda: net(pts, vd))
        assert net.range_status(reset=True) & 1, f"rows={rows}: NaN input not reported"
    _same_bits(out[128], out[64], precision)
    assert bool(torch.isnan(out[128][700]).all()) and bool(torch.isfinite(out[128][:700]).all())


def test_overflowing_activation_sets_the_status_on_both_kernels():
    net = _net(make_cfg("cfg2"))
    pts, vd = _samples(300, seed=6)
    for rows in (64, 128):
        net.range_status(reset=True)
        _run(net, rows, lambda: net(pts, vd))
        assert net.range_status(reset=True) == 0, f"rows={rows}"
    with torch.no_grad():
        net.pts_linears[3].bias[5] = 70000.0   # fp16: an activation >= 65520 has no hi part
    for rows in (64, 128):
        net.range_status(reset=True)
        _run(net, rows, lambda: net(pts, vd))
        assert net.range_status(reset=True) & 1, f"rows={rows}: overflow not reported"


def test_graph_replay_gives_the_same_bytes():
    net = _net(make_cfg("cfg2"))
    pts, vd = _samples(128 * 40 + 17, seed=7)
    ref = _run(net, 64, lambda: net(pts, vd))
    _capi.set_mlp_rows(net.pack(), 128)
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.no_grad(), torch.cuda.stream(s):
            net(pts, vd)                        # warm-up launch outside the capture
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(g):
            out = net(pts, vd)
        for _ in range(2):
            out.zero_()
            g.replay()
            torch.cuda.synchronize()
            _same_bits(out, ref, "graph replay")
    finally:
        _capi.set_mlp_rows(net.pack(), 0)


def test_programs_the_128_row_kernel_cannot_run_are_refused():
    """cfg3 (heads) and a 128-wide network stay on 64 rows by default and are refused when 128 rows are forced."""
    for cfg in (make_cfg("cfg3"), make_cfg("cfg2", D=5, W=128)):
        net = _net(cfg)
        pts, vd = _samples(200, seed=8)
        a = _run(net, 0, lambda: net(pts, vd))
        b = _run(net, 64, lambda: net(pts, vd))
        _same_bits(a, b, "default routing")
        with pytest.raises(_capi.PnrError, match="128-row"):
            _run(net, 128, lambda: net(pts, vd))
    with pytest.raises(_capi.PnrError, match="rows=96"):
        _capi.set_mlp_rows(net.pack(), 96)
