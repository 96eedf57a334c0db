"""CPU: the per-ray arithmetic the CUDA kernels use (csrc/ray_math.h, compiled for the host with
-ffp-contract=off) reproduces the oracle bit for bit: hit masks, M-nearest box ids, entry/exit depths,
stratified depths, per-sample ids and sample_pdf indices.  No GPU needed; the GPU tests repeat these
comparisons through the C ABI."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from host_emu import emu  # noqa: F401  (fixture)
from oracle import reference_renderer as O
from panopticnerf_b200 import make_cfg, synthetic as S


def _p(t):
    return C.c_void_p(t.data_ptr())


@pytest.mark.parametrize("B,M", [(64, 4), (5, 1), (300, 8)])
def test_intersect_order(emu, B, M):
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=6, row0=120)
    bx = S.make_boxes(B, 45, 64, seed=3)
    ref = O.intersect(rays[:, :3], rays[:, 3:], bx["box_center"], bx["box_half"], bx["box_rot"], M)
    R = rays.shape[0]
    hit = torch.zeros(R, dtype=torch.uint8)
    bid = torch.zeros(R, M, dtype=torch.int32)
    tin, tout = torch.zeros(R, M), torch.zeros(R, M)
    emu.emu_intersect(_p(rays), C.c_int64(R), _p(bx["box_center"]), _p(bx["box_half"]), _p(bx["box_rot"]),
                      None, None, C.c_int64(0), B, M, _p(hit), _p(bid), _p(tin), _p(tout))
    assert torch.equal(hit.bool(), ref[0]) and torch.equal(bid, ref[1])
    assert torch.equal(tin, ref[2]) and torch.equal(tout, ref[3])
    assert B < 64 or ref[0].any()


@pytest.mark.parametrize("N,perturb", [(64, 0.0), (64, 1.0), (192, 1.0), (2, 1.0)])
def test_stratified_order(emu, N, perturb):
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=2, row0=10)
    near, far = O.scene_near_far(rays[:, :3], rays[:, 3:], torch.tensor(S.SCENE_AABB), cfg.near, cfg.far)
    bx = S.make_boxes(64, 45, 64)
    _, bid, tin, tout = O.intersect(rays[:, :3], rays[:, 3:], bx["box_center"], bx["box_half"], bx["box_rot"], 4)
    t = torch.linspace(0, 1, N)
    u = torch.rand(rays.shape[0], N, generator=torch.Generator().manual_seed(0))
    z_ref = O.stratified_z(near, far, t, perturb, u)
    sb_ref = O.tag_samples(z_ref, bid, tin, tout)
    z = torch.zeros_like(z_ref)
    sb = torch.zeros_like(sb_ref)
    emu.emu_stratified(_p(near), _p(far), _p(t), _p(u), C.c_int64(rays.shape[0]), N, C.c_float(perturb),
                       _p(bid), _p(tin), _p(tout), 4, _p(z), _p(sb))
    assert torch.equal(z, z_ref) and torch.equal(sb, sb_ref)


@pytest.mark.parametrize("N,perturb,M", [(64, 0.0, 4), (64, 1.0, 4), (192, 0.0, 8), (7, 1.0, 2), (32, 0.0, 1)])
def test_interval_sampling_order(emu, N, perturb, M):
    """a6 interval mode: allocation counts, depths and ids equal the oracle's bit for bit (rays with several
    overlapping hits, rays with none, intervals cut by near/far)."""
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=3, row0=150)
    near, far = O.scene_near_far(rays[:, :3], rays[:, 3:], torch.tensor(S.SCENE_AABB), cfg.near, cfg.far)
    far = torch.minimum(far, torch.full_like(far, 40.0))        # cut some intervals short
    bx = S.make_boxes(12, 45, 64, seed=2)                       # few boxes: some rays hit none
    _, bid, tin, tout = O.intersect(rays[:, :3], rays[:, 3:], bx["box_center"], bx["box_half"], bx["box_rot"], M)
    t = torch.linspace(0, 1, N)
    u = torch.rand(rays.shape[0], N, generator=torch.Generator().manual_seed(0))
    z_ref = O.interval_z(near, far, t, bid, tin, tout, perturb, u)
    sb_ref = O.tag_samples(z_ref, bid, tin, tout)
    z = torch.zeros_like(z_ref)
    sb = torch.zeros_like(sb_ref)
    emu.emu_intervals(_p(near), _p(far), _p(t), _p(u), C.c_int64(rays.shape[0]), N, C.c_float(perturb),
                      _p(bid), _p(tin), _p(tout), M, _p(z), _p(sb))
    assert torch.equal(z, z_ref)
    # rays without a kept interval carry -1 everywhere in both (their samples lie in no interval by construction)
    assert torch.equal(sb, sb_ref)
    hit_rays = (bid >= 0).any(1)
    assert hit_rays.any() and (~hit_rays).any()
    inside = (sb_ref[hit_rays] >= 0).float().mean()
    assert inside > 0.95            # the point of the mode: (almost) every sample of a hit ray lies in a primitive
    assert (z_ref[:, 1:] >= z_ref[:, :-1]).all()


@pytest.mark.parametrize("N,Ni,det", [(64, 128, True), (64, 128, False), (3, 4, True), (192, 64, False)])
def test_sample_pdf_order(emu, N, Ni, det):
    g = torch.Generator().manual_seed(1)
    R = 2000
    z = torch.sort(torch.rand(R, N, generator=g) * 30 + 0.05, -1).values
    w = torch.rand(R, N, generator=g) ** 4 * (torch.rand(R, N, generator=g) > 0.5)
    w[:40] = 0
    u = (torch.linspace(0, 1, Ni)[None].expand(R, Ni) if det else torch.rand(R, Ni, generator=g)).contiguous()
    z_f_ref, idx_ref = O.sample_pdf(0.5 * (z[:, 1:] + z[:, :-1]), w[:, 1:-1], Ni, det=det, u=u)
    z_f = torch.zeros(R, Ni)
    idx = torch.zeros(R, Ni, dtype=torch.int64)
    emu.emu_sample_pdf(_p(z), _p(w), C.c_int64(R), N, Ni, _p(u), _p(z_f), _p(idx))
    assert torch.equal(idx, idx_ref), int((idx != idx_ref).sum())
    assert torch.equal(z_f, z_f_ref)


def test_interval_plan_properties(emu):
    """Property test (hypothesis) of the a6 interval rule through the host build of csrc/ray_math.h: for arbitrary
    interval tables the N depths are sorted, lie inside [near, far], and - when a hit interval survives the clipping -
    every one of them lies inside some kept interval; rays without one get exactly the uniform depths."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=200, deadline=None)
    @given(st.integers(1, 8), st.integers(1, 96), st.floats(0.05, 5.0), st.floats(6.0, 60.0),
           st.lists(st.tuples(st.floats(-5.0, 70.0), st.floats(0.0, 30.0), st.booleans()), min_size=8, max_size=8))
    def run(M, N, near, far, raw):
        tin = torch.tensor([[a for a, _, _ in raw[:M]]], dtype=torch.float32)
        tout = tin + torch.tensor([[b for _, b, _ in raw[:M]]], dtype=torch.float32)
        order = torch.argsort(tin, 1)
        tin, tout = torch.gather(tin, 1, order), torch.gather(tout, 1, order)
        bid = torch.tensor([[i if v else -1 for i, (_, _, v) in enumerate(raw[:M])]], dtype=torch.int32)
        nr, fr = torch.tensor([near], dtype=torch.float32), torch.tensor([far], dtype=torch.float32)
        t = torch.linspace(0, 1, N)
        u = torch.zeros(1, N)
        z = torch.zeros(1, N)
        sb = torch.zeros(1, N, dtype=torch.int32)
        emu.emu_intervals(_p(nr), _p(fr), _p(t), _p(u), C.c_int64(1), N, C.c_float(0.0), _p(bid), _p(tin), _p(tout),
                          M, _p(z), _p(sb))
        assert torch.equal(z, O.interval_z(nr, fr, t, bid, tin, tout))             # and the oracle agrees bit for bit
        assert bool((z[:, 1:] >= z[:, :-1]).all()) and float(z.min()) >= nr.item() - 1e-4 and float(z.max()) <= fr.item() + 1e-4
        a, b = torch.maximum(tin, nr[:, None]), torch.minimum(tout, fr[:, None])
        kept = (bid >= 0) & (b - a > 0)
        if kept.any():
            inside = ((z[0, :, None] >= a[0][None] - 1e-4) & (z[0, :, None] <= b[0][None] + 1e-4) & kept[0][None]).any(1)
            assert bool(inside.all())
        else:
            assert torch.equal(z, O.stratified_z(nr, fr, t))
    run()


def test_fisheye_unprojection_order(emu):
    """The KITTI-360 fisheye (MEI) unprojection the rays kernel calls (ray_math.h::pnr_fisheye_dir), compiled for the
    host, equals the oracle bit for bit on every pixel of a 1400 x 1400 image - also beyond the field of view."""
    k = (1336.3220825849971, 1335.7883350012958, 716.94323510126321, 705.76498308221585, 2.2134047507854890,
         1.6798235660113681e-02, 1.6548773243373522)
    H = W = 1400
    c2w = torch.eye(4)[:3].contiguous()
    out = torch.zeros(H * W, 6)
    assert emu.emu_generate_rays(H, W, 0, H, 2, (C.c_float * 7)(*k), _p(c2w), _p(out)) == 0
    ref = O.generate_rays(H, W, k, c2w, "fisheye")
    assert torch.equal(out[:, 3:], ref[:, 3:]) and torch.isfinite(out[:, 3:]).all()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("camera,code", [("pinhole", 0), ("fisheye", 2)])
def test_generate_rays_order(emu, camera, code):
    """The ray generation the rays kernel runs (ray_math.h: pnr_pinhole_dir / pnr_fisheye_dir, then pnr_cam_to_world),
    compiled for the host: origins and directions equal the oracle's bit for bit, for a rotated and translated camera
    and a window of rows."""
    cfg = make_cfg("cfg2")
    k = (cfg.fx, cfg.fy, cfg.cx, cfg.cy) if camera == "pinhole" else \
        (1336.3220825849971, 1335.7883350012958, 716.94323510126321, 705.76498308221585, 2.2134047507854890,
         1.6798235660113681e-02, 1.6548773243373522)
    H, W = (cfg.H, cfg.W_img) if camera == "pinhole" else (1400, 1400)
    row0, rows = H // 3, 9
    yaw, pitch = 0.3, -0.2
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    rot = torch.tensor([[cy, 0.0, sy], [0.0, 1.0, 0.0], [-sy, 0.0, cy]], dtype=torch.float64) @ \
        torch.tensor([[1.0, 0.0, 0.0], [0.0, cp, -sp], [0.0, sp, cp]], dtype=torch.float64)
    c2w = torch.cat([rot, torch.tensor([[1.5], [-2.25], [0.75]], dtype=torch.float64)], 1).float().contiguous()
    intr = (C.c_float * 7)(*(list(k) + [0.0] * (7 - len(k))))
    out = torch.zeros(rows * W, 6)
    assert emu.emu_generate_rays(H, W, row0, rows, code, intr, _p(c2w), _p(out)) == 0
    ref = O.generate_rays(H, W, k, c2w, camera, row0=row0, rows=rows)
    assert torch.equal(out, ref)
    assert not torch.equal(ref[:, 3:], O.generate_rays(H, W, k, torch.eye(4)[:3], camera, row0=row0, rows=rows)[:, 3:])


def test_pdf_cdf_sums_are_order_independent():
    """The sample_pdf kernel computes the two running sums of pnr_pdf_cdf as a warp scan (32 chunks, tree order)
    instead of sequentially.  That is bit-identical only because every partial sum is exact in double for weights in
    [0, 1]; check the claim on adversarial weights: chunked / tree-ordered double sums == sequential double sums."""
    import numpy as np
    rng = np.random.default_rng(0)
    for N in (3, 5, 64, 192, 256):
        nw = N - 2
        cases = [rng.random(N), np.zeros(N), np.ones(N), rng.random(N) * 1e-7, 1.0 - rng.random(N) * 2.0 ** -23,
                 np.where(rng.random(N) < 0.5, 1.0, 2.0 ** -30 * rng.random(N)), rng.random(N) ** 8]
        for wts in cases:
            v = (wts.astype(np.float32)[1:-1] + np.float32(1e-5)).astype(np.float32)
            seq = np.cumsum(v.astype(np.float64))                      # sequential, one rounding per step (none needed)
            total = np.float32(seq[-1]) if nw else np.float32(0)
            per = (nw + 31) // 32
            chunks = [v[i:i + per].astype(np.float64) for i in range(0, max(nw, 1), per)]
            tree = [c.sum() for c in chunks]
            while len(tree) > 1:                                        # pairwise, like the shuffle ladder
                tree = [tree[i] + (tree[i + 1] if i + 1 < len(tree) else 0.0) for i in range(0, len(tree), 2)]
            assert np.float32(tree[0]) == total and tree[0] == seq[-1]
            pdf = (v / total).astype(np.float32)
            seq2 = np.cumsum(pdf.astype(np.float64))
            offs = np.concatenate([[0.0], np.cumsum([c.sum() for c in (pdf[i:i + per].astype(np.float64) for i in range(0, nw, per))])])
            par = np.concatenate([offs[j] + np.cumsum(pdf[i:i + per].astype(np.float64)) for j, i in enumerate(range(0, nw, per))])
            assert np.array_equal(par.astype(np.float32), seq2.astype(np.float32)) and np.array_equal(par, seq2)
