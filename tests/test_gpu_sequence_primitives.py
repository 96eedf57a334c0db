"""GPU tier of sequence tables (DESIGN 3.2, include/pnr.h pnr_intersect_frames): the kernel against each frame's own
table and the host build, bit for bit, around the 512-box staging chunk, with cuboids and meshes; zero frame fields are
pnr_intersect / pnr_intersect_meshes; render_train (uniform and interval sampling) and the fused render on a sequence
table equal, row for row, the same rays rendered with their frame's cat(static, block) table; the sampler's frame
output; a data-parallel step on a batch with ray_frame; and a box that moves between frames."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_ray_batch as ORB
import oracle_sequence as OS
from host_emu import emu  # noqa: F401  (fixture)
from panopticnerf_b200 import _capi, make_cfg, make_network, make_renderer, synthetic as S
from panopticnerf_b200.lib.datasets import kitti360 as K
from panopticnerf_b200.lib.datasets.kitti360.bboxes import Box3D
from panopticnerf_b200.lib.datasets.ray_batch import sample_ray_batch
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from test_cpu_sequence_primitives import emu_frames

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _dev(d):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in d.items()}


def _bits(a, b, what):
    a, b = a.detach(), b.detach()
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    bad = int((a != b).sum())
    assert bad == 0, f"{what}: {bad} elements differ"


def _gpu_one(rays, table, M):
    return P.intersect(rays, table["box_center"], table["box_half"], table["box_rot"], M, table.get("mesh_tri_start"),
                       table.get("mesh_tris"))


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("meshes", [False, True])
@pytest.mark.parametrize("S_,M", [(511, 1), (512, 4), (513, 8), (2000, 8)])
def test_kernel_equals_the_per_frame_tables_and_the_host_build(S_, M, meshes, emu):
    F, pool = 300, 1500
    prims = S.make_mesh_primitives(num_boxes=S_ + pool - 5, seed=S_) if meshes else S.make_boxes(S_ + pool, seed=S_)
    B = prims["box_center"].shape[0]
    fb = OS.random_sequence(prims, S_, F, 64, seed=S_, shared=40)
    fb[:8] = torch.tensor([B - 64, B], dtype=torch.int32)        # frames whose block holds the meshes
    fb[8] = torch.tensor([S_ - 3, S_ + 10])                       # clamped at S
    cfg = make_cfg("cfg2")
    rays = torch.cat([S.make_rays(cfg), S.make_rays(cfg, seed=1)]).to(DEV)
    R = rays.shape[0]
    rf = torch.randint(-1, F + 1, (R,), generator=torch.Generator().manual_seed(S_), dtype=torch.int32).to(DEV)
    p = _dev(prims)
    got = P.intersect(rays, p["box_center"], p["box_half"], p["box_rot"], M, p.get("mesh_tri_start"), p.get("mesh_tris"),
                      rf, fb.to(DEV), S_)
    ref = OS.per_frame(_gpu_one, rays, p, S_, fb, rf, M)
    for a, b, k in zip(got, ref, ("hit_mask", "box_id", "t_in", "t_out")):
        _bits(a, b, f"S={S_} {k}")
    assert bool((got[1] >= S_).any())
    if meshes and M > 1 and S_ < 1000:   # with one slot, or 2000 static boxes in front, the nearest hits are cuboids
        assert bool((got[1] >= B - 5).any()), "no ray reached a mesh in a dynamic block"
    sub = torch.randperm(R, generator=torch.Generator().manual_seed(1))[:8192].to(DEV)
    host = emu_frames(emu, rays[sub].cpu().contiguous(), prims, S_, fb, rf[sub].cpu().contiguous(), M)
    for a, b, k in zip(got, host, ("hit_mask", "box_id", "t_in", "t_out")):
        _bits(a[sub].cpu(), b, f"S={S_} host {k}")


@pytest.mark.parametrize("meshes", [False, True])
def test_zero_frame_fields_give_the_bytes_of_the_single_table_entry_points(meshes):
    prims = _dev(S.make_mesh_primitives(seed=4) if meshes else S.make_boxes(600, seed=4))
    rays = S.make_rays(make_cfg("cfg2"), rows=100, row0=150).to(DEV)
    R, B, M = rays.shape[0], prims["box_center"].shape[0], 4
    out = [torch.empty(R, dtype=torch.uint8, device=DEV), torch.empty(R, M, dtype=torch.int32, device=DEV),
           torch.empty(R, M, device=DEV), torch.empty(R, M, device=DEV)]
    st = prims.get("mesh_tri_start")
    tris = prims.get("mesh_tris")
    a = _capi.PnrIntersectFramesArgs(rays=rays.data_ptr(), R=R, box_center=prims["box_center"].data_ptr(),
                                     box_half=prims["box_half"].data_ptr(), box_rot=prims["box_rot"].data_ptr(), B=B,
                                     M=M, mesh_tri_start=_capi.ptr(st), mesh_tris=_capi.ptr(tris),
                                     T=tris.shape[0] if meshes else 0, hit_mask=out[0].data_ptr(),
                                     box_id=out[1].data_ptr(), t_in=out[2].data_ptr(), t_out=out[3].data_ptr())
    _capi.check(_capi.lib().pnr_intersect_frames(C.byref(a), _capi.stream_ptr()))
    ref = _gpu_one(rays, prims, M)
    _bits(out[0].bool(), ref[0], "hit_mask")
    for x, y, k in zip(out[1:], ref[1:], ("box_id", "t_in", "t_out")):
        _bits(x, y, k)


# ------------------------------------------------------------------------------------------------ render
MAP_KEYS = ("rgb_map", "depth_map", "acc_map", "disp_map", "weights", "semantic_map", "instance_map",
            "fixed_semantic_map", "fixed_instance_map")


def _seq_batch(cfg, R, seed, S_=48, F=6):
    """R rays of a synthetic frame with jitter, a sequence table of S_ static boxes and F frames' blocks, ray_frame."""
    prims = S.make_boxes(S_ + 90, int(cfg.num_classes), int(cfg.num_instances), seed=seed)
    fb = OS.random_sequence(prims, S_, F, 30, seed=seed, shared=1)
    fb[0] = torch.tensor([S_, S_])
    rays = S.make_rays(cfg, seed=seed, row0=150, rows=(R * 4 + int(cfg.W_img) - 1) // int(cfg.W_img))[::4][:R]
    g = torch.Generator().manual_seed(seed + 100)
    b = dict(prims, rays=rays.contiguous(), scene_aabb=torch.tensor(S.SCENE_AABB),
             u=torch.rand(R, int(cfg.N_samples), generator=g), u_fine=torch.rand(R, int(cfg.N_importance), generator=g),
             ray_frame=torch.randint(0, F, (R,), generator=g, dtype=torch.int32), frame_boxes=fb)
    b = _dev(b)
    b["static_boxes"] = S_
    return b


def _per_frame_render(render, batch, S_):
    """{(b0, b1): (rows, output)}: the rays of each frame rendered with that frame's own table."""
    B = batch["box_center"].shape[0]
    out = {}
    for (b0, b1), rows in OS.groups(batch["ray_frame"], batch["frame_boxes"], S_, B).items():
        rows = rows.to(DEV)
        sub = {k: batch[k][rows].contiguous() for k in ("rays", "u", "u_fine")}
        sub.update(OS.frame_table(batch, S_, b0, b1), scene_aabb=batch["scene_aabb"])
        out[(b0, b1)] = (rows, render(sub))
    return out


def _check_rows(whole, parts, S_, what):
    n = 0
    for (b0, b1), (rows, o) in parts.items():
        for k, v in o.items():
            if k in ("near", "far") or not torch.is_tensor(v):
                continue
            w = whole[k][rows]
            if k in ("box_id", "sample_box"):
                v = torch.where(v >= S_, v + (b0 - S_), v)
            _bits(w, v, f"{what} {k} block ({b0}, {b1})")
            n += 1
    assert n > 0
    assert {k for k in MAP_KEYS} <= set(whole)


@pytest.mark.parametrize("mode", ["uniform", "intervals"])
def test_render_train_equals_the_per_frame_tables(mode):
    cfg = make_cfg("cfg3", render_path="staged", bound_by_primitives=True, perturb=1.0, sample_mode=mode)
    net = S.init_network_weights(make_network(cfg), seed=3).to(DEV)
    fine = S.init_network_weights(make_network(cfg), seed=4).to(DEV)
    r = make_renderer(cfg, net, fine)
    batch = _seq_batch(cfg, 600, seed=11)
    whole = r.render_train(batch)
    assert bool((whole["box_id"] >= 48).any()), "no ray met a dynamic box"
    _check_rows(whole, _per_frame_render(r.render_train, batch, 48), 48, f"render_train {mode}")


def test_render_fused_equals_the_per_frame_tables():
    cfg = make_cfg("cfg3", perturb=1.0, sample_mode="intervals", bound_by_primitives=True)
    net = S.init_network_weights(make_network(cfg), seed=5).to(DEV)
    r = make_renderer(cfg, net)
    batch = _seq_batch(cfg, 2000, seed=12)
    whole = r.render(batch)
    assert bool((whole["box_id"] >= 48).any())
    _check_rows(whole, _per_frame_render(r.render, batch, 48), 48, "render_fused")


def test_a_whole_frame_renders_against_the_sequence_table():
    cfg = make_cfg("cfg1", num_classes=5, num_instances=6, max_hits=3, N_importance=32)
    net = S.init_network_weights(make_network(cfg), seed=6).to(DEV)
    r = make_renderer(cfg, net)
    batch = _seq_batch(cfg, 1024, seed=13, S_=20, F=4)
    for f in range(4):
        b = dict(batch, ray_frame=torch.full_like(batch["ray_frame"], f))
        b.pop("u"), b.pop("u_fine")
        got = r.render(b)
        b0, b1 = map(int, batch["frame_boxes"][f].tolist())
        one = dict(OS.frame_table(batch, 20, b0, b1), rays=batch["rays"], scene_aabb=batch["scene_aabb"])
        ref = r.render(one)
        for k in ("rgb_map", "fixed_semantic_map", "z_vals", "hit_mask"):
            _bits(got[k], ref[k], f"frame {f} {k}")
        _bits(got["box_id"], torch.where(ref["box_id"] >= 20, ref["box_id"] + (b0 - 20), ref["box_id"]), "box_id")


# ------------------------------------------------------------------------------------------------ sampler
def test_sampled_frame_is_the_frame_of_the_pixel():
    from test_gpu_ray_batch import device_set
    rng = np.random.default_rng(21)
    fs = ORB.random_frame_set(rng, 37, ORB.random_cameras(rng, 3, tiny=True))
    d = device_set(fs)
    a = sample_ray_batch(d, 5, 9, 0, 20000, 16, 8, want_pixel=True, want_frame=True)
    b = sample_ray_batch(d, 5, 9, 0, 20000, 16, 8, want_pixel=True)
    assert set(a) == set(b) | {"frame"} and a["frame"].dtype == torch.int32
    for k in b:
        _bits(a[k], b[k], k)
    want = ORB.frame_of(fs["pix_offset"], a["pixel"].cpu().numpy())
    assert np.array_equal(a["frame"].cpu().numpy(), want.astype(np.int32))
    assert len(np.unique(want)) >= 30              # the tiny cameras' frames hold few pixels


def test_ray_sampler_adds_ray_frame_with_a_sequence_table():
    from test_gpu_ray_batch import device_set
    from panopticnerf_b200.lib.datasets.ray_batch import RaySampler
    rng = np.random.default_rng(22)
    fs = ORB.random_frame_set(rng, 5, ORB.random_cameras(rng, 2))
    d = device_set(fs)
    plain = _dev(S.make_boxes(32, seed=1))
    seq = dict(plain, frame_boxes=torch.tensor([[20, 24]] * 5, dtype=torch.int32, device=DEV), static_boxes=20)
    a = RaySampler(d, 3, plain).batch(2, 500, 16, 8)
    b = RaySampler(d, 3, seq).batch(2, 500, 16, 8)
    assert "ray_frame" not in a and set(b) == set(a) | {"ray_frame", "frame_boxes", "static_boxes"}
    for k in a:
        _bits(a[k], b[k], k)
    with pytest.raises(ValueError, match="one .begin, end. row per frame"):
        RaySampler(d, 3, dict(seq, frame_boxes=seq["frame_boxes"][:4]))


# ------------------------------------------------------------------------------------------------ training
def test_two_shard_step_equals_the_one_gpu_step_with_ray_frame():
    from test_gpu_data_parallel import _nets, _params, cfg3, simulate_shards
    from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper
    cfg = cfg3("frequency")
    net, fine = _nets(cfg, False, seed=61)
    batch = _seq_batch(cfg, 300, seed=14)
    g = torch.Generator().manual_seed(3)
    R = batch["rays"].shape[0]
    batch.update(rgb=torch.rand(R, 3, generator=g).to(DEV),
                 pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g).to(DEV))
    opt = FusedAdam(_params(net, fine))
    opt.zero_grad()
    out_w, loss_w, _, _ = NetworkWrapper(cfg, net, fine)(batch)
    loss_w.backward()
    g_whole = opt.flat_grads()[0].clone()
    assert bool((out_w["box_id"] >= 48).any())
    results, stacks = simulate_shards(cfg, net, fine, batch, 2, opt)
    lo = 0
    for out, loss, _ in results:
        n = out["box_id"].shape[0]
        _bits(out["box_id"], out_w["box_id"][lo:lo + n], "shard box_id")
        _bits(out["rgb_map"], out_w["rgb_map"][lo:lo + n], "shard rgb_map")
        lo += n
    assert lo == R
    assert float(results[-1][1]) == pytest.approx(float(loss_w.detach()), rel=1e-5)
    g_sum = stacks[0].sum(0)
    assert float((g_whole - g_sum).abs().max() / g_whole.pow(2).mean().sqrt()) < 1e-4


# ------------------------------------------------------------------------------------------------ a moving box
def _cuboid(name, center, half, sem, inst, ts):
    T = np.eye(4)
    T[:3, :3] = np.diag(2.0 * np.asarray(half))
    T[:3, 3] = center
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
    return Box3D(name, T, v, sem, inst, ts, int(ts != -1))


def test_a_moving_box_is_seen_where_it_is_in_each_frame():
    cfg = make_cfg("cfg1", num_classes=5, num_instances=6, max_hits=3, N_importance=32, perturb=0.0)
    net = S.init_network_weights(make_network(cfg), seed=7).to(DEV)
    car = 3
    boxes = [_cuboid("object1", (-6.0, 0.0, 25.0), (1.0, 1.0, 1.0), 1, 1, -1)]
    for ts, x in ((100, 0.0), (101, 8.0), (102, 16.0)):
        boxes.append(_cuboid(f"object{ts}", (x, 0.0, 20.0), (1.5, 1.0, 2.0), car, 2, ts))
    seq = K.sequence_primitives(boxes, [100, 101, 102])
    batch = K.primitive_batch(seq, device=DEV)
    g = torch.Generator().manual_seed(0)
    tgt = torch.tensor([0.0, 0.0, 20.0]) + (torch.rand(256, 3, generator=g) - 0.5) * torch.tensor([1.0, 1.0, 0.0])
    rays = torch.cat([torch.zeros(256, 3), tgt], 1).to(DEV)       # through the car where it is at timestamp 100
    batch.update(rays=rays, scene_aabb=torch.tensor(S.SCENE_AABB, device=DEV))
    seen = []
    for f in range(3):
        b = dict(batch, ray_frame=torch.full((256,), f, dtype=torch.int32, device=DEV))
        fused = make_renderer(cfg, net).render(b)
        train = make_renderer(make_cfg("cfg1", num_classes=5, num_instances=6, max_hits=3, N_importance=32,
                                       perturb=0.0, render_path="staged"), net).render_train(b)
        for out in (fused, train):
            seen.append(bool((out["fixed_semantic_map"][:, car] > 0).all()) if f == 0 else
                        bool((out["fixed_semantic_map"][:, car] == 0).all()))
        assert bool((fused["box_id"] == 1 + f).any(1).all()) == (f == 0)
    assert all(seen), seen
