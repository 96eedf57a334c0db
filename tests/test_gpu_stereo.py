"""GPU tier of stereo depth targets (pnr_stereo_depth, kitti360/stereo.py): the kernels bit for bit against the numpy
oracle (disparity and depth) from small shapes to KITTI-360's 376 x 1408 at D = 128 and 256, n = 1 .. 17 frames of a
mixed pinhole / fisheye store in one call, untouched rows, the same bytes across launches, split calls and a CUDA-graph
replay, and a sequence written in the KITTI-360 layout trained on through load_frames(stereo=...)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_stereo as O
import panopticnerf_b200 as PN
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.datasets.kitti360 import stereo as ST

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
f32 = np.float32
B16 = float(f32(16 * 552.554 * 0.6))


def _pair(rng, H, W, d0=5):
    left, right = O.random_dots(rng, H, W, min(d0, W - 1))
    if H > 2:
        left[: H // 3] //= 64
        right[: H // 3] //= 64
    return left, right


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


SHAPES = [(1, 1), (1, 33), (7, 9), (33, 65), (48, 64)]
PARAMS = [(10, 120, 10), (0, 0, 0), (2048, 2048, 99)]


@pytest.mark.parametrize("H,W", SHAPES)
@pytest.mark.parametrize("D", list(range(32, 257, 32)))
def test_disparity_equals_the_oracle(H, W, D):
    rng = np.random.default_rng(H * 7 + W + D)
    for k, (P1, P2, U) in enumerate(PARAMS):
        if k and (H, W) != (33, 65):      # all penalties at one shape, the defaults at the others
            break
        pairs = [_pair(rng, H, W, 3 + i) for i in range(2)]
        got = ST.stereo_disparity(_dev(np.stack([p[0] for p in pairs])), _dev(np.stack([p[1] for p in pairs])),
                                  D, P1, P2, U).cpu().numpy()
        for i, (l, r) in enumerate(pairs):
            assert np.array_equal(got[i], O.sgm(l, r, D, P1, P2, U)), (i, P1, P2, U)


@pytest.mark.parametrize("D", [128, 256])
def test_kitti_sized_pair_equals_the_oracle(D):
    fx, b = 552.554, 0.6
    H, W = 376, 1408
    # a far plane and a near box, textured, ray-cast into the pair
    left, right = O.render_pair(H, W, fx, 682.049, 238.77, b, [(30.0, None, 1), (6.0, (500, 800, 100, 300), 2),
                                                               (2.5, (1000, 1200, 150, 330), 3)])
    got = ST.stereo_disparity(_dev(left[None]), _dev(right[None]), D).cpu().numpy()[0]
    want = O.sgm(left, right, D)
    assert np.array_equal(got, want)
    assert (want >= 0).mean() > 0.5


def _mixed_store(rng, H, W, n, extra=3):
    """A store of pinhole H x W frames interleaved with fisheye frames of another size: (rgb8 [P, 3], pix_offset,
    the store indices of the n pinhole frames)."""
    sizes, rows, pin = [], [], []
    k = 0
    while len(pin) < n or extra > 0:
        if k % 3 == 1 or len(pin) == n:
            extra -= len(pin) == n
            h, w = 11, 13
        else:
            h, w = H, W
            pin.append(len(sizes))
        sizes.append(h * w)
        rows.append(rng.integers(0, 256, (h * w, 3), dtype=np.uint8))
        k += 1
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return np.concatenate(rows), off, pin


def _call(rgb8, off, frames, right, D=64, depth=None, disparity=None, P1=10, P2=120, U=10, b16=B16, max_depth=40.0):
    a = _capi.PnrStereoArgs()
    a.rgb8, a.pix_offset, a.P, a.F = rgb8.data_ptr(), off.data_ptr(), rgb8.shape[0], off.shape[0] - 1
    fr = np.ascontiguousarray(frames, np.int32)
    a.frames, a.n, a.H, a.W = fr.ctypes.data, len(fr), right.shape[1], right.shape[2]
    a.right, a.D, a.P1, a.P2, a.U = right.data_ptr(), D, P1, P2, U
    a.B16, a.min_depth, a.max_depth = b16, 0.1, max_depth
    a.depth = depth.data_ptr() if depth is not None else None
    a.disparity = disparity.data_ptr() if disparity is not None else None
    need = _capi.lib().pnr_stereo_workspace_bytes(a.n, a.H, a.W, D)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    a.workspace, a.workspace_bytes = ws.data_ptr(), need
    _capi.check(_capi.lib().pnr_stereo_depth(C.byref(a), torch.cuda.current_stream().cuda_stream), "pnr_stereo_depth")
    return ws, fr


@pytest.mark.parametrize("n", [1, 2, 5, 17])
def test_frames_of_a_mixed_store_in_one_call(n):
    rng = np.random.default_rng(n)
    H, W, D = 24, 40, 64
    rgb8, off, pin = _mixed_store(rng, H, W, n)
    pairs = [_pair(rng, H, W, 2 + i % 7) for i in range(n)]
    for k, (l, _) in enumerate(pairs):
        rgb8[off[pin[k]]:off[pin[k] + 1]] = l.reshape(-1, 3)
    order = rng.permutation(n)                         # the call names the frames out of store order
    right = _dev(np.stack([pairs[k][1] for k in order]))
    sentinel = rng.uniform(-9, -1, int(off[-1])).astype(f32)
    depth = _dev(sentinel)
    disp = torch.empty((n, H, W), dtype=torch.int16, device=DEV)
    keep = _call(_dev(rgb8), _dev(off), [pin[k] for k in order], right, D, depth, disp)
    torch.cuda.synchronize()
    del keep
    depth, disp = depth.cpu().numpy(), disp.cpu().numpy()
    named = set(pin)
    for i, k in enumerate(order):
        want = O.sgm(*pairs[k], D)
        assert np.array_equal(disp[i], want)
        sl = slice(int(off[pin[k]]), int(off[pin[k] + 1]))
        assert depth[sl].tobytes() == O.depth_of(want, B16, 0.1, 40.0).reshape(-1).tobytes()
    for f in range(len(off) - 1):
        if f not in named:
            sl = slice(int(off[f]), int(off[f + 1]))
            assert depth[sl].tobytes() == sentinel[sl].tobytes(), f


def test_repeat_split_and_graph_replay_give_the_same_bytes():
    rng = np.random.default_rng(9)
    H, W, D, n = 40, 96, 96, 6
    rgb8, off, pin = _mixed_store(rng, H, W, n)
    pairs = [_pair(rng, H, W, 4 + i) for i in range(n)]
    for k, (l, _) in enumerate(pairs):
        rgb8[off[pin[k]]:off[pin[k] + 1]] = l.reshape(-1, 3)
    rgb8, off = _dev(rgb8), _dev(off)
    right = _dev(np.stack([p[1] for p in pairs]))
    base = torch.zeros(int(off[-1]), dtype=torch.float32, device=DEV)
    _call(rgb8, off, pin, right, D, base)
    again = torch.full_like(base, 5.0)
    _call(rgb8, off, pin, right, D, again)
    named = torch.zeros_like(base, dtype=torch.bool)
    for f in pin:
        named[int(off[f]):int(off[f + 1])] = True
    assert torch.equal(again[named], base[named])
    split = torch.zeros_like(base)
    for part in (slice(0, 2), slice(2, 3), slice(3, n)):
        _call(rgb8, off, pin[part], right[part].contiguous(), D, split)
    assert torch.equal(split, base)
    poisoned = torch.full_like(base, -3.0)
    disp = torch.empty((n, H, W), dtype=torch.int16, device=DEV)
    ref_disp = torch.empty_like(disp)
    _call(rgb8, off, pin, right, D, disparity=ref_disp)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        keep = _call(rgb8, off, pin, right, D, poisoned, disp)
    for _ in range(2):
        poisoned.fill_(-3.0)
        disp.fill_(7)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(poisoned[named], base[named])
        assert bool((poisoned[~named] == -3.0).all())
        assert torch.equal(disp, ref_disp)
    del keep


# ------------------------------------------------------------------------------------------------ end to end
def _scene_pairs(n, H, W, fx, b):
    out = []
    for i in range(n):
        layers = [(fx * b / 4, None, 10 + i), (fx * b / (12 + i), (20 + 2 * i, 44 + 2 * i, 8, 30), 20 + i)]
        out.append(O.render_pair(H, W, fx, (W - 1) / 2, (H - 1) / 2, b, layers))
    return out


def test_a_sequence_with_a_stereo_pair_trains_with_a_depth_term(tmp_path):
    from panopticnerf_b200.lib.datasets.kitti360 import load_frames, save_depth_png
    from panopticnerf_b200.lib.datasets.ray_batch import RaySampler, sample_ray_batch
    from panopticnerf_b200.lib.train import NetworkWrapper
    frames = [10, 11, 12]
    H, W, fx, b = 48, 80, 40.0, 0.6
    pairs = _scene_pairs(len(frames), H, W, fx, b)
    info = O.write_stereo_sequence(tmp_path, frames, pairs, fx=fx, cx=(W - 1) / 2, cy=(H - 1) / 2, b=b)
    seq = info["seq"]
    opts = {"num_disparities": 32, "max_depth": 20.0, "chunk_frames": 2}
    fs = load_frames(tmp_path, seq, frames, device=DEV, stereo=opts)
    # the same table as one direct call over the set's frames
    b16 = float(f32(16 * fx * b))
    assert b16 == ST.stereo_baseline(tmp_path)[0]
    rights = _dev(np.stack([p[1] for p in pairs]))
    direct = torch.zeros_like(fs.depth)
    _call(fs.rgb8, fs.pix_offset, [0, 1, 2], rights, 32, direct, b16=b16, max_depth=20.0)
    torch.cuda.synchronize()
    assert fs.depth.cpu().numpy().tobytes() == direct.cpu().numpy().tobytes()
    want = np.concatenate([O.depth_of(O.sgm(l, r, 32), b16, 0.1, 20.0).reshape(-1) for l, r in pairs])
    assert fs.depth.cpu().numpy().tobytes() == want.tobytes()
    assert float((fs.depth > 0).float().mean()) > 0.5
    # RaySampler's depth is the set's depth at the sampled pixels
    bt = sample_ray_batch(fs, 3, 0, 0, 4096, 16, want_pixel=True)
    assert bt["depth"].cpu().numpy().tobytes() == fs.depth[bt["pixel"]].cpu().numpy().tobytes()
    cfg = PN.make_cfg("cfg1", num_classes=5, perturb=1.0)
    batch = RaySampler(fs, 9).batch(0, 1024, int(cfg.N_samples))
    assert int((batch["depth"] > 0).sum()) > 0
    net = S.init_network_weights(PN.make_network(cfg), seed=2).to(DEV)
    _, loss, stats, _ = NetworkWrapper(cfg, net)(batch)
    assert float(stats["depth_loss"]) > 0 and bool(torch.isfinite(loss))
    # the PNG cache reads back as rne(t 256) / 256
    (tmp_path / "depth").mkdir()
    for i, f in enumerate(frames):
        save_depth_png(fs.depth[i * H * W:(i + 1) * H * W].view(H, W), tmp_path / "depth" / f"{f:010d}.png")
    back = load_frames(tmp_path, seq, frames, device=DEV, depth_dir=tmp_path / "depth")
    code = np.rint(want * f32(256))
    assert back.depth.cpu().numpy().tobytes() == (np.where(code > 65535, 0, code).astype(f32) / f32(256)).tobytes()
