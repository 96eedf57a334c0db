"""GPU tier of weighted draws: pnr_pixel_cdf against numpy's uint64 cumsum exactly (P = 1 .. 2^26, tile and group
boundaries, 2^31 + 3 sparse pixels), pnr_label_counts against np.bincount, pnr_pixel_weights and pixel_weights against
the host build, weighted batches against the host build bit for bit at the unweighted tests' shapes, ranges, repeats and
a CUDA-graph replay, all-ones weights against the unweighted batch, masks and frame balance over 2^24 draws, and a few
training steps on weighted batches."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_pixel_weights as W
import oracle_ray_batch as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h)
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.datasets.ray_batch import (Camera, FrameSet, PixelWeights, RaySampler, pixel_weights,
                                                      label_counts, sample_ray_batch)
from test_gpu_ray_batch import CASES, _same, device_set

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def hw():
    """the host build of the weighted-draw routines (tests/host_emu_weights.cpp)"""
    return W.host_lib()


def _u16(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.uint16)).to(DEV)


def _cdf(weight: torch.Tensor):
    """pnr_pixel_cdf on the current stream: (cum, totals) as numpy uint64."""
    P = weight.numel()
    cum = torch.empty((P + 31) // 32, dtype=torch.uint64, device=DEV)
    tot = torch.empty(2, dtype=torch.uint64, device=DEV)
    L = _capi.lib()
    ws = torch.empty(L.pnr_pixel_cdf_workspace_bytes(P), dtype=torch.uint8, device=DEV)
    _capi.check(L.pnr_pixel_cdf(weight.data_ptr(), P, cum.data_ptr(), tot.data_ptr(), ws.data_ptr(), ws.numel(),
                                _capi.stream_ptr()), "pnr_pixel_cdf")
    return cum.view(torch.int64).cpu().numpy().view(np.uint64), tot.view(torch.int64).cpu().numpy().view(np.uint64)


# ------------------------------------------------------------------------------------------------ prefix sums
SIZES = [1, 2, 31, 32, 33, 255, 1023, 1024, 1025, 4096 + 17, 32767, 32768, 32769, 65536 + 1024, 3 * 32768 + 31,
         (1 << 20) + 3, (1 << 24) + 32 * 5 + 1, 1 << 26]


@pytest.mark.parametrize("P", SIZES)
def test_cdf_equals_numpy_cumsum(P):
    rng = np.random.default_rng(P % 9973)
    w = rng.integers(0, 65536, P).astype(np.uint16)
    w[rng.random(P) < 0.3] = 0
    if P > 40000:
        w[32768:32768 * 2] = 0                           # a whole tile of zeros
        w[-1] = 65535
    cum, tot = _cdf(_u16(w))
    assert np.array_equal(cum, W.groups(w))
    assert int(tot[0]) == int(w.astype(np.uint64).sum()) and int(tot[1]) == int(np.count_nonzero(w))


def test_cdf_of_two_to_the_31_plus_3_sparse_pixels():
    P = (1 << 31) + 3
    if torch.cuda.mem_get_info(DEV)[0] < 2 * P + P // 4 + (2 << 30):
        pytest.skip("the device lacks the memory for 2^31 + 3 weights")
    rng = np.random.default_rng(17)
    pos = np.unique(np.concatenate([rng.integers(0, P, 5000), [0, 31, 32, (1 << 31) - 1, 1 << 31, P - 1]]))
    val = rng.integers(1, 65536, len(pos)).astype(np.uint16)
    val[-1] = 65535
    w = torch.zeros(P, dtype=torch.uint16, device=DEV)
    w.view(torch.int16)[torch.from_numpy(pos).to(DEV)] = torch.from_numpy(val.view(np.int16)).to(DEV)
    cum, tot = _cdf(w)
    del w
    torch.cuda.empty_cache()
    assert int(tot[0]) == int(val.astype(np.uint64).sum()) and int(tot[1]) == len(pos)
    G = (P + 31) // 32
    assert len(cum) == G
    S = np.concatenate([[0], np.cumsum(val.astype(np.uint64))])
    gs = np.unique(np.concatenate([rng.integers(0, G, 20000), [0, 1, G - 2, G - 1], pos // 32, pos // 32 - 1]))
    gs = gs[(gs >= 0) & (gs < G)]
    want = S[np.searchsorted(pos, np.minimum(P, 32 * (gs + 1)), side="left")]
    assert np.array_equal(cum[gs], want)


def test_cdf_in_a_cuda_graph_replays_into_poisoned_outputs():
    rng = np.random.default_rng(2)
    P = 5 * 32768 + 77
    w = _u16(rng.integers(0, 65536, P))
    L = _capi.lib()
    cum = torch.empty((P + 31) // 32, dtype=torch.uint64, device=DEV)
    tot = torch.empty(2, dtype=torch.uint64, device=DEV)
    ws = torch.empty(L.pnr_pixel_cdf_workspace_bytes(P), dtype=torch.uint8, device=DEV)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        _capi.check(L.pnr_pixel_cdf(w.data_ptr(), P, cum.data_ptr(), tot.data_ptr(), ws.data_ptr(), ws.numel(),
                                    _capi.stream_ptr()), "pnr_pixel_cdf")
    for _ in range(2):
        cum.view(torch.int64).fill_(-1)
        tot.view(torch.int64).fill_(-1)
        ws.fill_(0xAB)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(cum.view(torch.int64).cpu().numpy().view(np.uint64), W.groups(w.cpu().numpy()))
        assert int(tot.view(torch.int64)[0]) == int(w.cpu().numpy().astype(np.uint64).sum())


# ------------------------------------------------------------------------------------------------ label counts
@pytest.mark.parametrize("P,C", [(1, 0), (1000, 1), (77777, 19), ((1 << 24) + 5, 45), (300000, 8191)])
def test_label_counts_equal_bincount(P, C):
    rng = np.random.default_rng(P + C)
    lab = rng.integers(-3, C + 5, P).astype(np.int16)
    if P > 1000:
        lab[: P // 2] = min(C, 7) - 1                      # one dominant class: contended bins
    fs = type("FS", (), {})()
    fs.label, fs.num_pixels = torch.from_numpy(lab).to(DEV), P
    got = label_counts(fs, C).view(torch.int64).cpu().numpy()
    s = W.slots(lab, C)
    assert np.array_equal(got, np.bincount(s, minlength=C + 1))


# ------------------------------------------------------------------------------------------------ weight tables
def _mixed_set(rng, F=40):
    cams = [(0, 37, 61, [40.0, 41.0, 30.3, 18.1]), (2, 45, 45, [20.0, 20.5, 22.3, 22.1, 1.4, 0.02, 0.01]),
            (2, 30, 30, [14.0, 14.0, 15.0, 15.0, 0.9, 0.0, 0.0])]
    return O.random_frame_set(rng, F, cams)


def test_pixel_weights_equal_the_host_build(hw):
    rng = np.random.default_rng(4)
    fs = _mixed_set(rng)
    F = len(fs["frame_cam"])
    ff = (rng.random(F) * 2).astype(np.float32)
    ff[:3] = [np.nan, -1, np.inf]
    ncls = 12
    cf = (rng.random(ncls + 1) * 3).astype(np.float32)
    cf[2] = np.nan
    masks = [(rng.random((H, Wd)) < 0.8).astype(np.uint8) if k != 2 else None for k, (_, H, Wd, _) in enumerate(fs["cams"])]
    scale = 9876.5
    d = device_set(fs)
    a = _capi.PnrPixelWeightsArgs()
    from panopticnerf_b200.lib.datasets.ray_batch import fill_frame_store
    fill_frame_store(a, d, "test")
    t = lambda x, dt=None: torch.from_numpy(np.ascontiguousarray(x, dt)).to(DEV)
    keep = [t(m) if m is not None else None for m in masks] + [t(ff), t(cf)]
    for k, m in enumerate(keep[:3]):
        a.mask[k] = m.data_ptr() if m is not None else None
    a.label, a.C, a.frame_factor, a.class_factor, a.scale = d.label.data_ptr(), ncls, keep[3].data_ptr(), keep[4].data_ptr(), scale
    out = torch.full((d.num_pixels,), 0x5A5A, dtype=torch.int16, device=DEV)
    a.weight = out.data_ptr()
    _capi.check(_capi.lib().pnr_pixel_weights(C.byref(a), _capi.stream_ptr()), "pnr_pixel_weights")
    got = out.cpu().numpy().view(np.uint16)
    assert np.array_equal(got, W.host_weights(hw, fs, scale, ncls, ff, cf, masks))
    assert np.array_equal(got, W.frame_set_weights(fs, scale, ncls, ff, cf, masks))


@pytest.mark.parametrize("balance,alpha,unlab", [(False, 0.0, 1.0), (True, 0.5, 0.25), (True, 1.0, 0.0), (False, 2.0, 3.0)])
def test_pixel_weights_builds_the_documented_factors(balance, alpha, unlab, hw):
    """pixel_weights' factors restated in float64 and rounded once, through the host build of the rule."""
    rng = np.random.default_rng(int(alpha * 10) + balance)
    fs = _mixed_set(rng, 25)
    fs["label"][rng.random(len(fs["label"])) < 0.5] = 3                   # a dominant class
    fs["label"][fs["label"] == 7] = -1                                   # an empty class
    d = device_set(fs)
    masks = [None, (rng.random((45, 45)) < 0.5), None]
    pw = pixel_weights(d, camera_masks=[None, torch.from_numpy(masks[1]), None], balance_frames=balance,
                       class_alpha=alpha, class_max_ratio=6.0, unlabelled=unlab)
    off = fs["pix_offset"]
    F, P = len(fs["frame_cam"]), int(off[-1])
    ff = (P / F) / np.diff(off).astype(np.float64) if balance else None
    ncls = int(fs["label"].max()) + 1
    n = np.bincount(W.slots(fs["label"], ncls), minlength=ncls + 1)[1:].astype(np.float64)
    cls = np.where(n > 0, np.minimum(6.0, (n.max() / np.maximum(n, 1)) ** alpha), 0.0) if alpha > 0 else np.ones(ncls)
    cf = np.concatenate([[unlab], cls])
    scale = float(np.float32(65535.0 / ((ff.max() if balance else 1.0) * cf.max())))
    use_cf = alpha > 0 or unlab != 1.0
    want = W.host_weights(hw, fs, scale, ncls if use_cf else 0, ff, cf if use_cf else None,
                          [None, masks[1].astype(np.uint8), None])
    got = pw.weight.view(torch.int16).cpu().numpy().view(np.uint16)
    assert np.array_equal(got, want)
    assert np.array_equal(pw.cum.view(torch.int64).cpu().numpy().view(np.uint64), W.groups(want))
    assert pw.total == int(want.astype(np.uint64).sum()) and pw.nonzero == int(np.count_nonzero(want))
    assert got.max() >= 65000                                             # the scale puts the largest product at 65535


# ------------------------------------------------------------------------------------------------ weighted batches
def _weights(rng, P, sparse):
    w = rng.integers(0, 65536, P).astype(np.uint16)
    if sparse:
        w[rng.random(P) < 0.8] = 0
    w[-1] = 1
    return w


@pytest.mark.parametrize("F,ncam,label,depth,R", CASES)
def test_weighted_kernel_equals_the_host_build(F, ncam, label, depth, R, hw):
    rng = np.random.default_rng(F + R + 1)
    fs = O.random_frame_set(rng, F, O.random_cameras(rng, ncam, tiny=ncam >= 3), label, depth)
    P = int(fs["pix_offset"][-1])
    w = _weights(rng, P, F % 2 == 1)
    N, Ni = (64, 128) if R == 1 << 20 else (int(rng.integers(1, 40)), int(rng.integers(0, 30)))
    seed, step = int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 40))
    pw = PixelWeights.from_weight(_u16(w).view(torch.uint16))
    assert np.array_equal(pw.cum.view(torch.int64).cpu().numpy().view(np.uint64), W.groups(w))
    got = sample_ray_batch(device_set(fs), seed, step, 0, R, N, Ni, want_pixel=True, weights=pw)
    want = W.host_weighted_batch(hw, fs, w, seed, step, 0, R, N, Ni)
    assert set(got) == {"rays", "rgb", "u", "pixel", "importance"} | ({"u_fine"} if Ni else set()) | \
        ({"depth"} if depth else set()) | ({"pseudo_label"} if label else set())
    for k, v in got.items():
        assert _same(v, want[k]), k
    assert (w[got["pixel"].cpu().numpy()] > 0).all()


def test_weighted_ranges_repeats_and_a_graph_replay():
    rng = np.random.default_rng(8)
    fs = O.random_frame_set(rng, 30, O.random_cameras(rng, 2))
    d = device_set(fs)
    pw = PixelWeights.from_weight(_u16(_weights(rng, d.num_pixels, True)))
    whole = sample_ray_batch(d, 1, 2, 0, 3000, 16, 32, want_pixel=True, weights=pw)
    again = sample_ray_batch(d, 1, 2, 0, 3000, 16, 32, want_pixel=True, weights=pw)
    assert all(torch.equal(whole[k], again[k]) for k in whole)
    for r0, r1 in ((250, 1000), (256 * 3 + 5, 2999), (0, 1), (2999, 3000)):
        part = sample_ray_batch(d, 1, 2, r0, r1, 16, 32, want_pixel=True, weights=pw)
        for k in whole:
            assert torch.equal(part[k], whole[k][r0:r1]), (k, r0, r1)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        cap = sample_ray_batch(d, 1, 2, 0, 3000, 16, 32, want_pixel=True, weights=pw)
    for _ in range(2):
        for v in cap.values():
            v.view(torch.uint8).fill_(0xFF)
        g.replay()
        torch.cuda.synchronize()
        for k in whole:
            assert torch.equal(cap[k].view(torch.uint8), whole[k].view(torch.uint8)), k


def test_all_ones_weights_give_the_unweighted_batch():
    rng = np.random.default_rng(12)
    fs = O.random_frame_set(rng, 50, O.random_cameras(rng, 3, tiny=True))
    d = device_set(fs)
    pw = PixelWeights.from_weight(torch.ones(d.num_pixels, dtype=torch.int16, device=DEV).view(torch.uint16))
    assert pw.total == pw.nonzero == d.num_pixels
    a = sample_ray_batch(d, 2 ** 63 + 9, 2 ** 32 + 1, 0, 70000, 64, 128, want_pixel=True, want_frame=True, weights=pw)
    b = sample_ray_batch(d, 2 ** 63 + 9, 2 ** 32 + 1, 0, 70000, 64, 128, want_pixel=True, want_frame=True)
    assert set(a) == set(b) | {"importance"}
    for k in b:
        assert torch.equal(a[k].view(torch.uint8), b[k].view(torch.uint8)), k
    assert (a["importance"] == 1.0).all()


def test_masks_and_frame_balance_over_2_24_draws(emu):
    """No masked pixel in 2^24 draws (a fisheye FOV mask and a random pinhole mask), and with balance_frames alone each
    camera's share of the rays is its share of the frames within 2e-3 (binomial sd at 2^24 draws: < 1.3e-4; weight
    rounding: < 1e-4)."""
    from panopticnerf_b200.lib.datasets.kitti360 import fisheye_fov_mask
    cams = [Camera("pinhole", 94, 352, (276.0, 276.0, 175.5, 47.0)),
            Camera("fisheye", 350, 350, (333.0, 333.0, 175.0, 175.0, 2.2, 0.016, 1.6))]
    rng = np.random.default_rng(5)
    fc = [0] * 9 + [1] * 3
    rgb = [torch.from_numpy(rng.integers(0, 256, (cams[c].H, cams[c].W, 3)).astype(np.uint8)) for c in fc]
    c2w = np.stack([np.eye(3, 4)] * len(fc)).astype(np.float32)
    d = FrameSet.from_images(cams, fc, c2w, rgb, device=DEV)
    fov = fisheye_fov_mask(cams[1], 80.0, device=DEV)
    # the mask against the host build's rays of the identity pose, in float64
    rays = np.zeros((350 * 350, 6), np.float32)
    k = np.asarray(cams[1].intr, np.float32)
    eye = np.ascontiguousarray(np.eye(3, 4, dtype=np.float32))
    emu.emu_generate_rays(350, 350, 0, 350, 2, k.ctypes.data_as(C.POINTER(C.c_float)),
                          eye.ctypes.data_as(C.POINTER(C.c_float)), rays.ctypes.data_as(C.POINTER(C.c_float)))
    dd = rays[:, 3:].astype(np.float64)
    want = (dd[:, 2] / np.linalg.norm(dd, axis=1) >= np.cos(np.radians(80.0))).reshape(350, 350)
    assert np.array_equal(fov.cpu().numpy(), want) and want.any() and not want.all()
    pin = torch.from_numpy(rng.random((94, 352)) < 0.6)
    pw = pixel_weights(d, camera_masks=[pin, fov])
    keep = np.concatenate([(pin.numpy() if c == 0 else fov.cpu().numpy()).reshape(-1) for c in fc])
    R = 1 << 24
    p = sample_ray_batch(d, 99, 1, 0, R, 1, want_pixel=True, weights=pw)["pixel"].cpu().numpy()
    assert keep[p].all()
    assert len(np.unique(p)) > 0.9 * keep.sum()
    pb = pixel_weights(d, balance_frames=True)
    f = sample_ray_batch(d, 7, 1, 0, R, 1, want_frame=True, weights=pb)["frame"].cpu().numpy()
    share = np.bincount(np.asarray(fc)[f], minlength=2) / R
    assert abs(share[1] - 3 / 12) < 2e-3 and abs(share[0] - 9 / 12) < 2e-3, share
    plain = sample_ray_batch(d, 7, 1, 0, 1 << 20, 1, want_frame=True)["frame"].cpu().numpy()
    assert np.bincount(np.asarray(fc)[plain], minlength=2)[1] / (1 << 20) > 0.5   # unweighted: by resolution


def test_training_steps_on_weighted_batches():
    from test_gpu_data_parallel import _nets, _params, cfg3
    from panopticnerf_b200 import parallel, synthetic as S
    from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper
    cfg = cfg3("frequency")
    rng = np.random.default_rng(31)
    fs = O.random_frame_set(rng, 6, O.random_cameras(rng, 2))
    d = device_set(fs)
    scene = {k: v.to(DEV) for k, v in S.make_boxes(64, 45, 64, seed=3).items()}
    scene["scene_aabb"] = torch.tensor(S.SCENE_AABB, dtype=torch.float32, device=DEV)
    pw = pixel_weights(d, balance_frames=True, class_alpha=0.5)
    sampler = RaySampler(d, seed=8, scene=scene, weights=pw)
    net, fine = _nets(cfg, False, seed=51)
    opt = FusedAdam(_params(net, fine))
    wrapper = NetworkWrapper(cfg, net, fine)
    for step in range(4):
        batch = sampler.batch(step=step, R=256, N=int(cfg.N_samples), Ni=int(cfg.N_importance))
        assert batch["importance"].shape == (256,) and torch.isfinite(batch["importance"]).all()
        shard = parallel.shard_training_batch(batch, 1, 2)
        assert torch.equal(shard["importance"], batch["importance"][128:])
        opt.zero_grad()
        _, loss, _, _ = wrapper(batch)
        loss.backward()
        opt.step()
        assert np.isfinite(float(loss.detach())), step
