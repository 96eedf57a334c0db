"""GPU: the single-call frame renderer (pnr_render_fused, SURVEY 8(b)), the interval sampler (8(a) a6), the range
check of the fp16 operands, several devices driven from one process and the NCCL entry points of the C ABI."""
import ctypes as C

import pytest
import torch

import panopticnerf_b200 as PN
from oracle import reference_renderer as O
from panopticnerf_b200 import _capi, parallel, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from util import check_render_outputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# maps whose per-ray sums the compositing epilogue of the MLP kernel forms in a different (fixed) order than the
# standalone compositing kernel: equal up to fp32 rounding of a sum of N terms
SUMMED = ("rgb_map", "depth_map", "acc_map", "disp_map", "semantic_map", "instance_map")


def _same(a, b, what="", summed_exact=True):
    assert a.keys() == b.keys(), (sorted(a), sorted(b))
    for k in a:
        x, y = a[k], b[k]
        assert x.shape == y.shape and x.dtype == y.dtype, f"{what}{k}: {x.shape} {x.dtype} vs {y.shape} {y.dtype}"
        base = k[:-2] if k.endswith("_0") else k
        if base in SUMMED and not summed_exact:
            xs, ys = torch.nan_to_num(x.float()), torch.nan_to_num(y.float())
            scale = float(ys.abs().max()) + 1e-12
            assert float((xs - ys).abs().max()) <= 2e-6 * scale + 1e-7, f"{what}{k}: {float((xs - ys).abs().max())}"
        else:
            assert torch.equal(torch.nan_to_num(x.float()), torch.nan_to_num(y.float())), f"{what}{k} differs"


@pytest.mark.parametrize("preset,over,rows", [
    ("cfg1", {}, None), ("cfg1", dict(num_classes=5, num_instances=6, N_importance=16), None),
    ("cfg3", {}, 3), ("cfg3", dict(sample_mode="intervals", bound_by_primitives=True, mask_outside=True), 2),
    ("cfg2", dict(white_bkgd=True), 5)])
def test_fused_render_equals_staged(preset, over, rows):
    """One pnr_render_fused call == the stage-by-stage path from Python: every integer / mask / depth / per-sample
    weight bit for bit, the per-ray sums (formed in the MLP kernel's compositing epilogue there, by the standalone
    compositing kernel here) to fp32 rounding; and the fused result does not depend on its workspace (one chunk, the
    default, ~20 ragged chunks) - with and without jitter."""
    cfg = PN.make_cfg(preset, **over)
    net = S.init_network_weights(PN.make_network(cfg), seed=2).to(DEV)
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, rows=rows).items()}
    R = batch["rays"].shape[0]
    staged = PN.make_renderer(PN.make_cfg(preset, render_path="staged", **over), net).render(batch)
    fused = PN.make_renderer(cfg, net).render(batch)
    # masks, ids, depths, per-sample weights (hence the fine samples): bit for bit; per-ray sums: to fp32 rounding
    _same(fused, staged, summed_exact=False)
    # and the fused path does not depend on its chunking at all
    _same(PN.make_renderer(PN.make_cfg(preset, gpu_chunk=R // 20 + 3, **over), net).render(batch), fused, "chunked: ")
    g = torch.Generator().manual_seed(1)
    jit = dict(batch, perturb=1.0, u=torch.rand(R, cfg.N_samples, generator=g).to(DEV))
    if cfg.N_importance:
        jit["u_fine"] = torch.rand(R, cfg.N_importance, generator=g).to(DEV)
    _same(PN.make_renderer(PN.make_cfg(preset, gpu_chunk=R // 3 + 1, **over), net).render(jit),
          PN.make_renderer(PN.make_cfg(preset, render_path="staged", **over), net).render(jit), "jitter: ",
          summed_exact=False)


@pytest.mark.parametrize("N,perturb,M,B", [(64, 0.0, 4, 64), (64, 1.0, 4, 12), (192, 0.0, 8, 64), (7, 1.0, 2, 12),
                                           (256, 0.0, 1, 5)])
def test_interval_sampler_bit_exact(N, perturb, M, B):
    cfg = PN.make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=3, row0=150)
    near, far = O.scene_near_far(rays[:, :3], rays[:, 3:], torch.tensor(S.SCENE_AABB), cfg.near, cfg.far)
    far = torch.minimum(far, torch.full_like(far, 40.0))
    bx = S.make_boxes(B, 45, 64, seed=2)
    _, bid, tin, tout = O.intersect(rays[:, :3], rays[:, 3:], bx["box_center"], bx["box_half"], bx["box_rot"], M)
    t = torch.linspace(0, 1, N)
    u = torch.rand(rays.shape[0], N, generator=torch.Generator().manual_seed(0))
    z_ref = O.interval_z(near, far, t, bid, tin, tout, perturb, u)
    d = lambda x: x.to(DEV)
    z, sb = P.interval_z(d(near), d(far), d(t), d(bid), d(tin), d(tout), perturb, d(u))
    assert torch.equal(z.cpu(), z_ref) and torch.equal(sb.cpu(), O.tag_samples(z_ref, bid, tin, tout))


def test_interval_mode_render_end_to_end():
    """cfg3 (heads, coarse + fine) with the samples placed inside the primitives, against the oracle."""
    cfg = PN.make_cfg("cfg3", sample_mode="intervals", W=64, D=4)
    net = S.init_network_weights(PN.make_network(cfg), seed=3)
    batch = S.make_batch(cfg, row0=200, rows=1)
    batch["rays"] = batch["rays"][::7].contiguous()
    onet = O.Network(cfg)
    onet.load_state_dict(net.state_dict())
    ref = O.make_renderer(cfg, onet).render(batch)
    out = PN.make_renderer(cfg, net.to(DEV)).render({k: v.to(DEV) for k, v in batch.items()})
    for k in ("hit_mask", "box_id", "z_vals_0"):
        assert torch.equal(out[k].cpu().to(ref[k].dtype), ref[k]), k
    assert float((ref["sample_box"][ref["hit_mask"]] >= 0).float().mean()) > 0.9
    # the fine depths are discontinuous in the coarse weights: compare what does not depend on them
    check_render_outputs(out, {k: v for k, v in ref.items() if k.endswith("_0") or k in ("near", "far", "t_in", "t_out")},
                         float(ref["far"].max()))


def _scaled(net, s):
    with torch.no_grad():
        for lin in net.pts_linears:
            lin.weight.mul_(s)
    return net


def test_fp16_overflow_is_reported_and_bf16x3_handles_it():
    """Trunk weights x16 per layer: activations pass 65504 from the fifth layer on.  fp16x3 must flag it (status bit,
    Renderer.render raises), bf16x3 must run the same network within tolerance (per-tensor RMS floor)."""
    cfg = PN.make_cfg("cfg2")
    g = torch.Generator().manual_seed(4)
    pts = (torch.rand(3000, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(3000, 3, generator=g), dim=-1)
    base = _scaled(S.init_network_weights(PN.make_network(cfg), seed=5), 16.0)
    onet = O.Network(cfg)
    onet.load_state_dict(base.state_dict())
    with torch.no_grad():
        ref = onet(pts, vd)
    assert float(ref[:, 3].abs().max()) > 1e5                 # the scale really is out of fp16's range
    net16 = PN.make_network(cfg)
    net16.load_state_dict(base.state_dict())
    net16 = net16.to(DEV)
    assert net16.range_status() == 0
    with torch.no_grad():
        net16(pts.to(DEV), vd.to(DEV))
    assert net16.range_status(reset=False) & 1 and net16.range_status() & 1 and net16.range_status() == 0
    with pytest.raises(_capi.PnrError, match="range"):
        batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, rows=1).items()}
        PN.make_renderer(cfg, net16).render(batch)
    cfgb = PN.make_cfg("cfg2", precision="bf16x3")
    netb = PN.make_network(cfgb)
    netb.load_state_dict(base.state_dict())
    netb = netb.to(DEV)
    with torch.no_grad():
        got = netb(pts.to(DEV), vd.to(DEV)).cpu()
    assert netb.range_status() == 0
    from util import assert_close, rms
    assert_close(got[:, :3], ref[:, :3], rms(ref[:, :3]), "rgb (bf16x3, x16 weights)", rel=2e-4)
    assert_close(got[:, 3:4], ref[:, 3:4], rms(ref[:, 3:4]), "sigma (bf16x3, x16 weights)", rel=2e-4)


@pytest.mark.parametrize("scale,shift", [(2.0, -3.0), (1.5, 0.5)])
def test_trained_like_statistics_within_tolerance(scale, shift):
    """Larger-than-init weights (x1.5 / x2 per trunk layer: activations up to ~1e3) and a shifted sigma bias, the
    statistics a trained scene network has: fp16x3 stays inside 1e-4 of the per-tensor RMS and reports no overflow."""
    from util import assert_close, rms
    cfg = PN.make_cfg("cfg3")
    base = _scaled(S.init_network_weights(PN.make_network(cfg), seed=6), scale)
    with torch.no_grad():
        base.alpha_linear.bias.add_(shift)
    g = torch.Generator().manual_seed(7)
    pts = (torch.rand(2000, 3, generator=g) * 2 - 1) * 8
    vd = torch.nn.functional.normalize(torch.randn(2000, 3, generator=g), dim=-1)
    onet = O.Network(cfg)
    onet.load_state_dict(base.state_dict())
    with torch.no_grad():
        ref = onet(pts, vd)
    net = base.to(DEV)
    with torch.no_grad():
        got = net(pts.to(DEV), vd.to(DEV)).cpu()
    assert net.range_status() == 0
    for name, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4)), ("sem", slice(4, 49)), ("inst", slice(49, 113))):
        assert_close(got[:, sl], ref[:, sl], rms(ref[:, sl]), f"{name} (x{scale} weights)")


def test_bf16x3_render_end_to_end():
    cfg = PN.make_cfg("cfg1", precision="bf16x3", num_classes=5, num_instances=6)
    net = S.init_network_weights(PN.make_network(cfg), seed=8)
    batch = S.make_batch(cfg, rows=16)
    onet = O.Network(cfg)
    onet.load_state_dict(net.state_dict())
    ref = O.make_renderer(cfg, onet).render(batch)
    out = PN.make_renderer(cfg, net.to(DEV)).render({k: v.to(DEV) for k, v in batch.items()})
    check_render_outputs(out, ref, float(ref["far"].max()), rel=2e-4)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_second_device_from_one_process():
    """Contexts on two devices driven from one process and one thread (ADVICE r1): per-device kernel attributes,
    launches on the context's device whatever the current device is, and the caller's device left untouched."""
    cfg = PN.make_cfg("cfg1", num_classes=5, num_instances=6, N_importance=16)
    net = S.init_network_weights(PN.make_network(cfg), seed=2)
    batch = S.make_batch(cfg)
    import copy
    n0, n1 = copy.deepcopy(net).to("cuda:0"), copy.deepcopy(net).to("cuda:1")
    torch.cuda.set_device(0)
    a = PN.make_renderer(cfg, n0).render({k: v.to("cuda:0") for k, v in batch.items()})
    b = PN.make_renderer(cfg, n1).render({k: v.to("cuda:1") for k, v in batch.items()})
    assert torch.cuda.current_device() == 0 and b["rgb_map"].device.index == 1
    _same(a, {k: v.to("cuda:0") for k, v in b.items()})
    e = P.embed(torch.rand(1000, 3, device="cuda:1"), 10)       # > 48 KB shared-memory opt-in on the second device
    assert e.device.index == 1 and torch.isfinite(e).all()


def test_comm_single_rank_allgather():
    """pnr_comm_* through ctypes with world = 1 (the 2-rank case: tests/test_gpu_comm2.py under torchrun)."""
    L = _capi.lib()
    if not L.pnr_comm_available():
        pytest.skip("libnccl.so.2 not loadable")
    uid = (C.c_uint8 * _capi.COMM_ID_BYTES)()
    _capi.check(L.pnr_comm_unique_id(uid), "pnr_comm_unique_id")
    comm = C.c_void_p()
    _capi.check(L.pnr_comm_init(C.byref(comm), uid, 0, 1, 0), "pnr_comm_init")
    src = torch.arange(1000, dtype=torch.float32, device=DEV)
    dst = torch.zeros_like(src)
    _capi.check(L.pnr_allgather_outputs(comm, src.data_ptr(), dst.data_ptr(), src.numel() * 4, _capi.stream_ptr()),
                "pnr_allgather_outputs")
    torch.cuda.synchronize()
    assert torch.equal(src, dst)
    _capi.check(L.pnr_comm_destroy(comm), "pnr_comm_destroy")
    assert L.pnr_comm_init(C.byref(comm), uid, 3, 2, 0) != 0 and b"rank" in L.pnr_last_error()


def test_label_tiles_kernel():
    """pnr_label_tiles: rgb -> u8, argmax labels with ties to the lowest index and NaN treated as -inf."""
    g = torch.Generator().manual_seed(3)
    R, Cn, Kn = 1000, 45, 64
    rgb, depth = torch.rand(R, 3, generator=g), torch.rand(R, generator=g) * 50
    sem, inst = torch.randn(R, Cn, generator=g), torch.randn(R, Kn, generator=g)
    sem[5] = 0.25                        # all equal: label 0
    sem[6, 7] = sem[6, 30] = 9.0         # tie: lowest index
    inst[7, :10] = float("nan")
    g_rgb, g_depth, g_sem, g_inst = rgb.to(DEV), depth.to(DEV), sem.to(DEV), inst.to(DEV)   # kept alive over the call
    rgb8 = torch.empty(R, 3, dtype=torch.uint8, device=DEV)
    dep = torch.empty(R, device=DEV)
    sl = torch.empty(R, dtype=torch.int16, device=DEV)
    il = torch.empty(R, dtype=torch.int16, device=DEV)
    _capi.check(_capi.lib().pnr_label_tiles(g_rgb.data_ptr(), g_depth.data_ptr(), g_sem.data_ptr(), g_inst.data_ptr(),
                                            R, Cn, Kn, rgb8.data_ptr(), dep.data_ptr(), sl.data_ptr(), il.data_ptr(),
                                            _capi.stream_ptr()), "pnr_label_tiles")
    torch.cuda.synchronize()
    assert torch.equal(rgb8.cpu().float(), torch.round(rgb * 255)) and torch.equal(dep.cpu(), depth)
    assert torch.equal(sl.cpu().long(), sem.argmax(-1)) and int(sl[5]) == 0 and int(sl[6]) == 7
    assert torch.equal(il.cpu().long(), torch.nan_to_num(inst, nan=-float("inf")).argmax(-1))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_tile_gather():
    import socket
    import subprocess
    import sys
    from pathlib import Path
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    worker = Path(__file__).parent / "comm2_worker.py"
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(worker)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "COMM2 OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_checkpoint_load_then_render(tmp_path):
    """SURVEY 8(f) rank 1 on the GPU: a reference-layout checkpoint ({'net': wrapper-prefixed state_dict, ...} as
    the training template writes it) is loaded with net_utils.load_network into a Network that already rendered
    with other weights (the libpnr context must repack), and the render equals the oracle's with those weights."""
    from panopticnerf_b200.lib.utils import net_utils
    cfg = PN.make_cfg("cfg1", num_classes=5, num_instances=6, N_importance=8)
    trained = S.init_network_weights(O.make_network(cfg), seed=11)
    torch.save({"net": {"net." + k: v for k, v in trained.state_dict().items()}, "optim": {}, "scheduler": {},
                "recorder": {}, "epoch": 42}, tmp_path / "42.pth")
    batch = S.make_batch(cfg, rows=8)
    gb = {k: v.to(DEV) for k, v in batch.items()}
    net = S.init_network_weights(PN.make_network(cfg), seed=0).to(DEV)
    ren = PN.make_renderer(cfg, net)
    before = ren.render(gb)
    assert net_utils.load_network(net, str(tmp_path)) == 42
    after = ren.render(gb)
    assert not torch.equal(before["rgb_map"], after["rgb_map"])
    ref = O.make_renderer(cfg, trained).render(batch)
    for k in ("hit_mask", "box_id", "z_vals_0"):
        assert torch.equal(after[k].cpu().to(ref[k].dtype), ref[k]), k
    check_render_outputs(after, {k: v for k, v in ref.items() if k.endswith("_0") or k in ("near", "far")},
                         float(ref["far"].max()))


@pytest.mark.parametrize("preset,over,R,flags", [
    ("cfg1", dict(num_classes=5, num_instances=6), 1000, {}),                      # N = 32: one group per ray
    ("cfg2", {}, 3001, dict(white_bkgd=True)),                                       # N = 64, no heads, odd ray count
    ("cfg3", dict(N_samples=192, N_importance=0), 777, dict(mask_outside=True)),     # N = 192: rays span 1.5 tiles
    ("cfg3", dict(N_samples=96, N_importance=0, D=4, W=128), 50, {}),                # N = 96, fewer rays than CTAs
    ("cfg1", dict(num_classes=45), 1, {}), ("cfg2", dict(N_samples=128), 3, {})])
def test_compositing_epilogue_matches_two_kernel_path(preset, over, R, flags):
    """pnr_mlp_composite (compositing in the MLP kernel's epilogue, raw never written) against pnr_mlp_forward +
    pnr_composite on the same rays / depths: weights and the fixed (bounding-box) maps bit for bit, the summed maps to
    fp32 rounding; NaN patterns (disp of empty rays) coincide."""
    cfg = PN.make_cfg(preset, **over)
    net = S.init_network_weights(PN.make_network(cfg), seed=4).to(DEV)
    full = S.make_batch(cfg, row0=cfg.H // 3, rows=max(1, R // cfg.W_img + 1))
    rays = full["rays"][:R].contiguous().to(DEV)
    near, far = P.scene_near_far(rays, full["scene_aabb"], cfg.near, cfg.far)
    hit, bid, tin, tout = P.intersect(rays, full["box_center"].to(DEV), full["box_half"].to(DEV), full["box_rot"].to(DEV), 4)
    z, sb = P.stratified_z(near, far, torch.linspace(0, 1, cfg.N_samples).to(DEV), 0.0, None, bid, tin, tout, want_tags=True)
    kw = dict(sample_box=sb, box_sem=full["box_sem"].to(DEV), box_inst=full["box_inst"].to(DEV), **flags)
    got = net.forward_composite(rays, z, **kw)
    raw = net.forward_rays(rays, z)
    ref = P.raw2outputs(raw, z, rays, num_classes=cfg.num_classes, num_instances=cfg.num_instances, **kw)
    assert got.keys() == ref.keys()
    for k in ("weights", "fixed_semantic_map", "fixed_instance_map"):
        if k in ref:
            assert torch.equal(got[k], ref[k]), k
    _same(got, ref, summed_exact=False)
    assert float(got["weights"].sum()) > 0


def test_compositing_epilogue_needs_whole_groups():
    cfg = PN.make_cfg("cfg2", N_samples=48)
    net = S.init_network_weights(PN.make_network(cfg)).to(DEV)
    rays = S.make_rays(cfg, rows=1)[:10].to(DEV)
    z = torch.sort(torch.rand(10, 48, device=DEV) * 20 + 1, -1).values
    with pytest.raises(_capi.PnrError, match="multiple of 32"):
        net.forward_composite(rays, z)
    out = PN.make_renderer(cfg, net).render({"rays": rays})       # the renderer falls back to the two-kernel path
    assert out["rgb_map"].shape == (10, 3) and torch.isfinite(out["rgb_map"]).all()


def test_compositing_epilogue_refuses_bad_primitive_tables():
    """forward_composite takes the primitive tables as raw2outputs does: id tables of different lengths (one B bounds
    both in the kernel, so the shorter one would be read past its end) and tables on another device are refused before
    any launch."""
    cfg = PN.make_cfg("cfg1", num_classes=5, num_instances=6)
    net = S.init_network_weights(PN.make_network(cfg), seed=2).to(DEV)
    rays = S.make_rays(cfg, rows=1)[:10].to(DEV)
    z = torch.sort(torch.rand(10, 32, device=DEV) * 20 + 1, -1).values
    sb = torch.randint(-1, 10, (10, 32), dtype=torch.int32, device=DEV)
    ids = torch.arange(10, dtype=torch.int32, device=DEV) % 5
    ok = net.forward_composite(rays, z, sample_box=sb, box_sem=ids, box_inst=ids)     # packs the weights
    assert "fixed_semantic_map" in ok and "fixed_instance_map" in ok
    torch.cuda.synchronize()
    _capi.lib().pnr_launch_count(1)
    with pytest.raises(ValueError, match=r"got lengths \[3, 10\]"):
        net.forward_composite(rays, z, sample_box=sb, box_sem=ids[:3], box_inst=ids)
    with pytest.raises(_capi.PnrError, match="box_sem is on cpu, expected cuda:0"):
        net.forward_composite(rays, z, sample_box=sb, box_sem=ids.cpu(), box_inst=ids)
    assert _capi.lib().pnr_launch_count(0) == 0


def test_cuda_graph_capture_and_replay():
    """The kernels take everything they need as launch parameters (the per-tile program travels as a __grid_constant__
    argument, nothing is uploaded at launch time), so a forward or a fused MLP + compositing call can be captured in a
    CUDA graph and replayed on new inputs in the same buffers - results equal the eager calls bit for bit."""
    cfg = PN.make_cfg("cfg1", num_classes=6, num_instances=4, N_samples=64)
    net = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
    g = torch.Generator().manual_seed(0)

    def inputs(seed):
        gg = torch.Generator().manual_seed(seed)
        rays = torch.cat([torch.randn(300, 3, generator=gg), torch.nn.functional.normalize(torch.randn(300, 3, generator=gg), dim=-1)], -1)
        z = torch.sort(torch.rand(300, 64, generator=gg) * 9 + 0.5, -1).values
        return rays.to(DEV), z.to(DEV)
    rays, z = inputs(1)
    net.forward_rays(rays, z); net.forward_composite(rays, z)          # weights packed, attributes set: nothing left to do at capture
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            raw_g = net.forward_rays(rays, z)
            comp_g = net.forward_composite(rays, z)
    torch.cuda.current_stream().wait_stream(side)
    for seed in (2, 3):
        r2, z2 = inputs(seed)
        rays.copy_(r2); z.copy_(z2)
        graph.replay()
        torch.cuda.synchronize()
        raw_e = net.forward_rays(r2, z2)
        comp_e = net.forward_composite(r2, z2)
        assert torch.equal(raw_g, raw_e)
        for k in comp_e:
            assert torch.equal(comp_g[k], comp_e[k]), k
    assert net.range_status() == 0
