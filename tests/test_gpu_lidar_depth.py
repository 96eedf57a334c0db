"""GPU tier of LiDAR depth targets (pnr_project_depth, kitti360/lidar.py): the kernels bit for bit against the host
build of the same per-point and per-pixel routines, order independence (permuted points, split calls, a second run, a
CUDA-graph replay), untouched frames, a wall and its occluder, P past 2^31, and a sequence written in the KITTI-360
layout trained on through load_frames(lidar=...) and RaySampler."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_lidar as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h and stereo_math.h)
import panopticnerf_b200 as PN
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.datasets.kitti360 import lidar as L

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
f32 = np.float32
SMALL_PINHOLE = (0, 48, 64, (40.0, 40.0, 31.7, 23.2))
SMALL_FISHEYE = (2, 50, 50, (47.8, 47.7, 25.6, 25.2, 2.2134, 0.01647, 1.6035))


def prepare(cams, fc, po, pts, so, pf, ps, pm, mind, maxd, radius=0, margin=0.1, depth=None):
    """pnr_project_depth_args over device copies of the tables and a workspace (depth: a device tensor rewritten in
    place; default zeros).  Returns (args, depth, what the args point into)."""
    t = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x), dtype=dt).to(DEV)
    keep = [t(fc, torch.int32), t(po, torch.int64), t(np.asarray(pts, f32).reshape(-1, 4), torch.float32)]
    if depth is None:
        depth = torch.zeros(int(po[-1]), dtype=torch.float32, device=DEV)
    a, _, host = O.args_struct(cams, fc, po, np.zeros((0, 4), f32), so, pf, ps, pm, mind, maxd, radius, margin,
                               depth=np.zeros(0, f32))
    a.frame_cam, a.pix_offset, a.points = keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr()
    a.Npts, a.P, a.depth = keep[2].shape[0], int(po[-1]), depth.data_ptr()
    need = int(_capi.lib().pnr_project_depth_workspace_bytes(a.P, radius))
    if need:
        keep.append(torch.empty(need, dtype=torch.uint8, device=DEV))
        a.workspace, a.workspace_bytes = keep[-1].data_ptr(), need
    return a, depth, (keep, host)


def launch(prep, stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    _capi.check(_capi.lib().pnr_project_depth(C.byref(prep[0]), s.cuda_stream), "pnr_project_depth")
    return prep[1]


def device_call(*args, **kw):
    prep = prepare(*args, **kw)
    return launch(prep), prep


def _bytes(t):
    return t.cpu().numpy().tobytes() if isinstance(t, torch.Tensor) else np.asarray(t).tobytes()


# F, S, points per scan (lo, hi), pairs per frame, filter radius
CASES = [(1, 1, (1, 1), 1, 0), (3, 2, (0, 5000), 2, 0), (40, 12, (100, 30000), 4, 0), (300, 30, (10, 3000), 10, 0),
         (60, 8, (1000, 20000), 3, 2), (25, 5, (100, 5000), 2, 8)]


@pytest.mark.parametrize("F,S_,npts,ppf,radius", CASES)
def test_kernel_equals_the_host_build(F, S_, npts, ppf, radius, emu):
    rng = np.random.default_rng(F * 7 + radius)
    cams = [SMALL_PINHOLE, SMALL_FISHEYE, (0, 1, 1, (1.0, 1.0, 0.0, 0.0))]
    scene = O.random_scene(rng, cams, F, S_, npts[0], npts[1], pairs_per_frame=ppf)
    got, _ = device_call(cams, *scene, 0.1, 60.0, radius, 0.07)
    want = O.host_zbuffer(emu, cams, *scene, 0.1, 60.0, radius, 0.07)
    assert _bytes(got) == want.tobytes()
    if F >= 3:
        assert (want > 0).sum() > 10
        models = {cams[scene[0][f]][0] for f in range(F) if (want[scene[1][f]:scene[1][f + 1]] > 0).any()}
        assert models == {0, 2} or F < 40


def test_kernel_at_2_24_plus_3_points_on_one_pixel_and_spread(emu):
    rng = np.random.default_rng(24)
    n = (1 << 24) + 3
    cams = [SMALL_PINHOLE]
    pts = np.empty((n, 4), f32)
    pts[:, 0] = rng.uniform(-20, 20, n)
    pts[:, 1] = rng.uniform(-10, 10, n)
    pts[:, 2] = rng.uniform(0.05, 70, n)
    pts[:, 3] = 0
    pts[: n // 2, :2] = 0                     # half of them on the principal point's pixel
    M = np.eye(3, 4, dtype=f32).reshape(1, 12)
    po = np.array([0, 48 * 64, 2 * 48 * 64], np.int64)
    args = (cams, [0, 0], po, pts, [0, n], [0, 1], [0, 0], np.concatenate([M, M * 1.0]))
    got, _ = device_call(*args, 0.1, 60.0)
    want = O.host_zbuffer(emu, *args, 0.1, 60.0)
    assert _bytes(got) == want.tobytes()
    assert (want > 0).sum() > 1000


def test_order_split_repeat_and_graph_replay_give_the_same_bytes(emu):
    rng = np.random.default_rng(77)
    cams = [SMALL_PINHOLE, SMALL_FISHEYE]
    fc, po, pts, so, pf, ps, pm = O.random_scene(rng, cams, 50, 10, 2000, 40000, pairs_per_frame=5)
    for radius in (0, 2):
        base, _ = device_call(cams, fc, po, pts, so, pf, ps, pm, 0.1, 60.0, radius, 0.05)
        # the points of every scan permuted, the pairs reversed
        perm = np.concatenate([rng.permutation(np.arange(so[s], so[s + 1])) for s in range(len(so) - 1)])
        a, _ = device_call(cams, fc, po, pts[perm], so, pf[::-1], ps[::-1], pm[::-1], 0.1, 60.0, radius, 0.05)
        assert _bytes(a) == _bytes(base)
        # the frames split across three calls into the same table
        d = torch.full_like(base, 7.0)
        for part in np.array_split(np.arange(50), 3):
            sel = np.isin(pf, part)
            device_call(cams, fc, po, pts, so, pf[sel], ps[sel], pm[sel], 0.1, 60.0, radius, 0.05, depth=d)
        assert _bytes(d) == _bytes(base)
        again, _ = device_call(cams, fc, po, pts, so, pf, ps, pm, 0.1, 60.0, radius, 0.05)
        assert _bytes(again) == _bytes(base)
        # captured in a CUDA graph, replayed twice into a poisoned table
        d = torch.full_like(base, -3.0)
        prep = prepare(cams, fc, po, pts, so, pf, ps, pm, 0.1, 60.0, radius, 0.05, depth=d)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            launch(prep, torch.cuda.current_stream())
        for _ in range(2):
            d.fill_(-3.0)
            g.replay()
            torch.cuda.synchronize()
            assert _bytes(d) == _bytes(base)


def test_only_the_named_frames_are_written():
    rng = np.random.default_rng(5)
    cams = [SMALL_PINHOLE, SMALL_FISHEYE]
    fc, po, pts, so, pf, ps, pm = O.random_scene(rng, cams, 20, 4, 1000, 5000, pairs_per_frame=2)
    sel = pf % 3 == 1
    for radius in (0, 3):
        before = torch.from_numpy(rng.uniform(-5, 5, int(po[-1])).astype(f32)).to(DEV)
        d = before.clone()
        device_call(cams, fc, po, pts, so, pf[sel], ps[sel], pm[sel], 0.1, 60.0, radius, 0.2, depth=d)
        for f in range(20):
            sl = slice(int(po[f]), int(po[f + 1]))
            if f % 3 == 1:
                assert bool((d[sl] >= 0).all()) and bool((d[sl] > 0).any())
            else:
                assert _bytes(d[sl]) == _bytes(before[sl]), f


@pytest.mark.parametrize("cam", [O.PINHOLE, O.FISHEYE], ids=["pinhole", "fisheye"])
def test_a_wall_at_10_m_and_a_nearer_occluder(cam):
    """A dense fronto-parallel wall at z = 10 m of the camera frame, seen from a scanner posed far from the world's
    origin (M composed in float64 and rounded once), and a 2 m square at z = 6 m in front of part of it."""
    rng = np.random.default_rng(10)
    c2w = np.eye(4)
    c2w[:3, :3] = O.rotation(rng.uniform(-0.5, 0.5, 3))
    c2w[:3, 3] = O.WORLD0
    velo = np.eye(4)
    velo[:3, :3] = O.rotation(rng.uniform(-0.5, 0.5, 3))
    velo[:3, 3] = O.WORLD0 + [1.5, -0.3, 0.8]
    M = (np.linalg.inv(c2w) @ velo)[:3, :4].astype(f32)
    gx, gy = (np.linspace(-13, 13, 3000), np.linspace(-4.5, 4.5, 1000)) if cam[0] == 0 else \
        (np.linspace(-25, 25, 2500), np.linspace(-25, 25, 2500))
    X, Y = np.meshgrid(gx, gy)
    wall = np.stack([X.ravel(), Y.ravel(), np.full(X.size, 10.0)], 1)
    sq = lambda r, n: np.stack([*(g.ravel() for g in np.meshgrid(np.linspace(-r, r, n), np.linspace(-r, r, n))),
                                np.full(n * n, 6.0)], 1)
    occ = sq(1.0, 500)
    pc = np.concatenate([wall, occ])
    pv = (np.linalg.inv(velo) @ c2w @ np.concatenate([pc, np.ones((len(pc), 1))], 1).T).T   # camera -> world -> scanner
    pts = np.concatenate([pv[:, :3], np.zeros((len(pv), 1))], 1).astype(f32)
    H, W = cam[1], cam[2]
    d, _ = device_call([cam], [0], [0, H * W], pts, [0, len(pts)], [0], [0], M.reshape(1, 12), 0.1, 80.0)
    d = d.cpu().numpy()
    # the pixels of the occluder: surely inside (a 1.8 m square) and possibly (a 2.2 m square)
    pixels = lambda p: O.project_points(cam, np.eye(3, 4), p, 0.1, 80.0)[1]
    inner = np.zeros(H * W, bool)
    inner[pixels(sq(0.9, 400))] = True
    near = np.zeros(H * W, bool)
    near[pixels(sq(1.1, 600))] = True
    covered = d > 0
    assert covered.mean() > (0.5 if cam[0] == 0 else 0.1)
    assert inner.sum() > 100
    wall_px = covered & ~near
    if cam[0] == 0:   # t = z: 10 m and 6 m up to the fp32 rounding of M and of the transform
        assert np.abs(d[wall_px] - 10.0).max() < 1e-4
        assert np.abs(d[inner] - 6.0).max() < 1e-4
    else:             # t = |p| >= z, and |p| <= sqrt(6^2 + 2) on the occluder
        assert d[wall_px].min() > 10.0 - 1e-4
        assert (np.abs(d[inner] - 6.0) < 0.17).all()


def test_two_to_the_31_plus_3_pixels(emu):
    big = (0, 8192, 16384, (8000.0, 8000.0, 8191.5, 4095.5))
    tiny = (0, 1, 3, (1.0, 1.0, 1.0, 0.0))
    P = 16 * (1 << 27) + 3
    if torch.cuda.mem_get_info(DEV)[0] < 4 * P + (2 << 30):
        pytest.skip("the device lacks the memory for 2^31 + 3 pixels")
    cams = [big, tiny]
    fc = np.array([0] * 16 + [1], np.int32)
    po = np.concatenate([[0], np.cumsum([1 << 27] * 16 + [3])]).astype(np.int64)
    rng = np.random.default_rng(31)
    n = 200000
    pts = np.stack([rng.uniform(-5, 5, n), rng.uniform(-5, 5, n), rng.uniform(1, 30, n), np.zeros(n)], 1).astype(f32)
    pts[:3] = [[-2, 0, 2, 0], [0, 0, 3, 0], [4, 0, 4, 0]]   # onto the tiny frame's pixels u = 0, 1, 2
    I = np.eye(3, 4, dtype=f32).reshape(1, 12)
    depth = torch.full((P,), -1.0, dtype=torch.float32, device=DEV)
    device_call(cams, fc, po, pts, [0, n], [15, 16], [0, 0], np.concatenate([I, I]), 0.1, 60.0, depth=depth)
    for f, cam in ((15, big), (16, tiny)):
        want = O.host_zbuffer(emu, [cam], [0], [0, cam[1] * cam[2]], pts, [0, n], [0], [0], I, 0.1, 60.0)
        assert _bytes(depth[int(po[f]):int(po[f + 1])]) == want.tobytes(), f
    assert bool((depth[-3:] > 0).all())
    assert bool((depth[int(po[14]):int(po[15])] == -1).all()) and bool((depth[:1 << 20] == -1).all())
    del depth
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ end to end
def _boxes(seq, frames):
    """One cuboid in front of camera 0 at each frame (world coordinates near the poses)."""
    from panopticnerf_b200.lib.datasets.kitti360 import Box3D
    out = []
    for i, f in enumerate(frames):
        T = np.eye(4)
        T[:3, :3] = seq["c0w"][f][:3, :3] @ np.diag([3.0, 2.0, 1.5])
        T[:3, 3] = (seq["c0w"][f] @ np.array([0.5 * (i - 1.5), 0.3, 7.0 + i, 1.0]))[:3]
        v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
        out.append(Box3D(f"box{i}", T, v, 26 + i % 2, 26000 + i, -1, 0))
    return out


def _surface_points(prims, rng, n):
    """n points on the faces of each cuboid of a primitive table (world coordinates)."""
    out = []
    for c, h, r in zip(prims["box_center"], prims["box_half"], prims["box_rot"]):
        u = rng.uniform(-1, 1, (n, 3))
        ax = rng.integers(0, 3, n)
        u[np.arange(n), ax] = np.where(rng.random(n) < 0.5, -1.0, 1.0)
        out.append((u * h) @ np.asarray(r, np.float64).reshape(3, 3).T + c)
    return np.concatenate(out)


def test_a_sequence_with_scans_trains_with_a_depth_term(tmp_path):
    from panopticnerf_b200.lib.datasets.kitti360 import boxes_to_primitives, load_frames, primitive_batch
    from panopticnerf_b200.lib.datasets.ray_batch import RaySampler, sample_ray_batch
    from panopticnerf_b200.lib.train import NetworkWrapper
    frames = [10, 11, 12, 13]
    rng = np.random.default_rng(4)
    seq = O.write_sequence(tmp_path, frames, cams=("image_00",), scans=[], world0=(1.0, 2.0, 0.5))
    prims = boxes_to_primitives(_boxes(seq, frames))
    world = _surface_points(prims, rng, 20000)
    for s in frames:   # each scan: the cuboids' surfaces in its Velodyne frame
        v2w = L.velo_to_world(seq["imu"][s], seq["c2p"]["image_00"], seq["c2v"])
        pv = (np.linalg.inv(v2w) @ np.concatenate([world, np.ones((len(world), 1))], 1).T).T[:, :3]
        np.concatenate([pv, rng.random((len(pv), 1))], 1).astype(f32).tofile(L.scan_path(tmp_path, seq["seq"], s))
    opts = {"lidar_window": 1, "max_depth": 40.0, "occlusion_radius": 1, "occlusion_margin": 0.2, "chunk_frames": 3}
    fs = load_frames(tmp_path, seq["seq"], frames, device=DEV, lidar=opts)
    fs2 = load_frames(tmp_path, seq["seq"], frames, device=DEV, lidar=opts)
    assert _bytes(fs.depth) == _bytes(fs2.depth)
    assert float((fs.depth > 0).float().mean()) > 0.02
    assert float(fs.depth[fs.depth > 0].min()) > 2.0
    b = sample_ray_batch(fs, 3, 0, 0, 4096, 16, want_pixel=True)
    assert _bytes(b["depth"]) == _bytes(fs.depth[b["pixel"]])
    cfg = PN.make_cfg("cfg1", num_classes=5, perturb=1.0)
    scene = primitive_batch(prims, sem_to_train={26: 1, 27: 2}, inst_to_slot={}, device=DEV)
    scene["scene_aabb"] = torch.tensor([-60.0, -60.0, -60.0, 60.0, 60.0, 60.0], device=DEV)
    batch = RaySampler(fs, 9, scene=scene).batch(0, 1024, int(cfg.N_samples))
    assert int((batch["depth"] > 0).sum()) > 0
    net = S.init_network_weights(PN.make_network(cfg), seed=2).to(DEV)
    _, loss, stats, _ = NetworkWrapper(cfg, net)(batch)
    assert float(stats["depth_loss"]) > 0 and bool(torch.isfinite(loss))
