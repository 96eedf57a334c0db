"""CPU tier of LiDAR depth targets (pnr_project_depth, kitti360/lidar.py): the host build of pnr_project_point and of
the whole call against the numpy oracle bit for bit, the round trip through pnr_generate_rays' rays, the readers, the
transform chain on fixtures written in the KITTI-360 layout, every refusal by name before any device call, the ctypes
layout, and the PNG cache read back through load_frames."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_lidar as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h)
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.datasets.kitti360 import lidar as L
from panopticnerf_b200.lib.datasets.kitti360 import load_frames
from panopticnerf_b200.lib.datasets.ray_batch import Camera, FrameSet

ROOT = Path(__file__).resolve().parent.parent
f32 = np.float32
TINY_FISHEYE = (2, 6, 7, (3.0, 2.5, 3.1, 2.4, 1.2, 0.05, 0.02))


def _same(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _check_points(emu, cam, M, p, mind, maxd):
    want = O.project_points(cam, M, p, mind, maxd)
    got = O.host_point(emu, cam, M, p, mind, maxd)
    for g, w, k in zip(got, want, ("ok", "pix", "t")):
        assert _same(g, w), k
    return got


@pytest.mark.parametrize("cam", [O.PINHOLE, O.FISHEYE, TINY_FISHEYE], ids=["pinhole", "fisheye", "tiny_fisheye"])
def test_point_equals_the_oracle_on_random_points(cam, emu):
    rng = np.random.default_rng(cam[1])
    for trial in range(4):
        M = np.concatenate([O.rotation(rng.uniform(-0.3, 0.3, 3)), rng.uniform(-2, 2, (3, 1))], 1)
        p = np.stack([rng.uniform(-40, 40, 3000), rng.uniform(-10, 10, 3000), rng.uniform(-20, 80, 3000)], 1)
        ok, _, _ = _check_points(emu, cam, M, p, 0.1, 80.0)
        assert 0 < ok.sum() < len(p)


def test_point_at_the_pixel_half_boundaries(emu):
    # fx = 2, cx = 0.5, z = 1: uf = (2 x) / 1 + 0.5 is exact, so x = k / 2 puts the point on uf = k + 0.5
    cam = (0, 4, 9, (2.0, 2.0, 0.5, 0.5))
    M = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    k = np.arange(-1, 9, dtype=f32)
    xs = np.concatenate([k / 2, np.nextafter(k / 2, f32(-np.inf)), np.nextafter(k / 2, f32(np.inf))])
    p = np.stack([xs, np.full_like(xs, 0.5), np.ones_like(xs)], 1)
    ok, pix, _ = _check_points(emu, cam, M, p, 0.5, 2.0)
    n = len(k)
    # exactly on k + 0.5: fp32(k + 0.5 + 0.5) = k + 1 -> pixel u = k + 1 (kept while < W = 9)
    on = (k + 1 >= 0) & (k + 1 < 9)
    assert np.array_equal(ok[:n], on)
    assert np.array_equal(pix[:n][on] % 9, (k + 1)[on].astype(np.int64))
    assert np.array_equal(pix[:n][on] // 9, np.full(on.sum(), 2))   # vf = (2 * 0.5) / 1 + 0.5 = 1.5 -> v = 2
    assert ok[n:].any()


def test_point_at_the_depth_limits_and_behind_the_camera(emu):
    cam = (0, 8, 8, (4.0, 4.0, 3.5, 3.5))
    M = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    mind, maxd = f32(0.25), f32(50.0)
    zs = [mind, np.nextafter(mind, f32(1)), np.nextafter(mind, f32(0)), maxd, np.nextafter(maxd, f32(0)),
          np.nextafter(maxd, f32(100)), f32(0), f32(-1), f32(-0.0), f32(10)]
    p = np.stack([np.zeros(len(zs), f32), np.zeros(len(zs), f32), np.array(zs, f32)], 1)
    ok, _, t = _check_points(emu, cam, M, p, mind, maxd)
    assert ok.tolist() == [False, True, False, True, True, False, False, False, False, True]
    assert t[1] == zs[1] and t[3] == maxd


def test_point_at_the_fisheye_mirror_limit(emu):
    # p = (4, 0, -3): n = 5 exactly, x_s.z = fp32(-3 / 5); xi = -x_s.z gives x_s.z + xi = 0 (refused), one ulp more
    # projects
    zs = f32(-3) / f32(5)
    M = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    p = np.array([[4, 0, -3], [40, 0, -30]], f32)
    for xi, want in ((-zs, False), (np.nextafter(-zs, f32(1)), True), (np.nextafter(-zs, f32(0)), False)):
        cam = (2, 4000, 4000, (1e-6, 1e-6, 2000.0, 2000.0, float(xi), 0.0, 0.0))
        ok, _, t = _check_points(emu, cam, M, p, 0.1, 80.0)
        assert ok.tolist() == [want, want]
        if want:
            assert t[0] == 5.0 and t[1] == 50.0


@pytest.mark.parametrize("cam", [O.PINHOLE, O.FISHEYE], ids=["pinhole", "fisheye"])
def test_point_with_nan_and_inf_coordinates(cam, emu):
    rng = np.random.default_rng(3)
    M = np.concatenate([O.rotation(rng.uniform(-0.2, 0.2, 3)), rng.uniform(-1, 1, (3, 1))], 1)
    bad = [np.nan, np.inf, -np.inf]
    p = np.array([[b if i == j else 1.0 for j in range(3)] for i in range(3) for b in bad] +
                 [[1.0, 1.0, 10.0]], f32)
    ok, _, _ = _check_points(emu, cam, M, p, 0.1, 80.0)
    assert not ok[:-1].any() and ok[-1]


def _rays(emu, cam, c2w):
    model, H, W, intr = cam
    rays = np.empty((H * W, 6), f32)
    c2w = np.ascontiguousarray(c2w, f32).reshape(12)
    intr = np.ascontiguousarray(intr, f32)
    assert emu.emu_generate_rays(H, W, 0, H, model, intr.ctypes.data_as(C.POINTER(C.c_float)),
                                 c2w.ctypes.data_as(C.POINTER(C.c_float)), rays.ctypes.data_as(C.POINTER(C.c_float))) == 0
    return rays


def test_round_trip_pinhole_is_exact(emu):
    cam = (0, 47, 61, (52.5, 51.0, 30.2, 23.7))
    I = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    rays = _rays(emu, cam, I)
    rng = np.random.default_rng(0)
    t = rng.uniform(0.2, 79.0, len(rays)).astype(f32)
    p = rays[:, 3:] * t[:, None]
    ok, pix, tt = _check_points(emu, cam, I, p, 0.1, 80.0)
    assert ok.all()
    assert np.array_equal(pix, np.arange(len(rays)))
    assert np.array_equal(tt, t)


# The fisheye's ray undoes the distortion with 8 Newton steps in fp32, so the pixel the point at t along the ray
# projects back to is off by the Newton residual and the roundings: < 2e-3 px inside the mirror's field of view (the
# same bound as the ray round trip of test_cpu_ray_math), and |p| = t |d| with |d| = 1 within 2^-20 relative
FISHEYE_ROUND_TRIP_PX = 2e-3


def test_round_trip_fisheye_within_the_newton_bound(emu):
    model, H, W, intr = O.FISHEYE
    sub = (2, 140, 140, (intr[0] / 10, intr[1] / 10, intr[2] / 10, intr[3] / 10) + tuple(intr[4:]))
    I = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    rays = _rays(emu, sub, I)
    v, u = np.divmod(np.arange(len(rays)), sub[2])
    inner = np.hypot(u - sub[3][2], v - sub[3][3]) < 55   # inside the mirror's field of view
    rng = np.random.default_rng(1)
    t = rng.uniform(0.5, 70.0, len(rays)).astype(f32)
    p = (rays[:, 3:] * t[:, None])[inner]
    ok, pix, tt, uf, vf = O.project_points(sub, I, p, 0.1, 80.0, want_uv=True)
    _check_points(emu, sub, I, p, 0.1, 80.0)
    assert ok.all()
    err = np.maximum(np.abs(uf - u[inner]), np.abs(vf - v[inner]))
    assert err.max() < FISHEYE_ROUND_TRIP_PX, err.max()
    assert np.array_equal(pix, np.arange(len(rays))[inner])
    assert np.abs(tt / t[inner] - 1).max() < 1e-6


@pytest.mark.parametrize("radius", [0, 1, 8])
def test_zbuffer_equals_the_oracle(radius, emu):
    rng = np.random.default_rng(10 + radius)
    cams = [(0, 9, 13, (6.0, 6.0, 6.3, 4.1)), TINY_FISHEYE, (0, 1, 1, (1.0, 1.0, 0.0, 0.0))]
    fc, po, pts, so, pf, ps, pm = O.random_scene(rng, cams, F=7, S=4, n_lo=20, n_hi=4000, pairs_per_frame=3)
    # duplicate points (scan 1 starts with scan 0's first 20), an empty scan, and repeated pairs (exact ties)
    pts[so[1]:so[1] + 20] = pts[so[0]:so[0] + 20]
    so = np.concatenate([so[:3], so[2:]])
    pf, ps, pm = np.concatenate([pf, pf[:3]]), np.concatenate([ps, ps[:3]]), np.concatenate([pm, pm[:3]])
    depth_in = rng.uniform(1, 2, int(po[-1])).astype(f32)
    named = set(pf.tolist())
    want = O.zbuffer(cams, fc, po, pts, so, pf, ps, pm, 0.1, 60.0, radius, 0.05, depth_in=depth_in)
    got = O.host_zbuffer(emu, cams, fc, po, pts, so, pf, ps, pm, 0.1, 60.0, radius, 0.05, depth_in=depth_in)
    assert _same(got, want)
    plain = O.zbuffer(cams, fc, po, pts, so, pf, ps, pm, 0.1, 60.0, 0, 0.05)
    assert (plain > 0).sum() > 20 and (want > 0).any()
    for f in range(len(fc)):
        sl = slice(int(po[f]), int(po[f + 1]))
        if f not in named:
            assert _same(got[sl], depth_in[sl])
    if radius:
        assert ((plain > 0) & (want == 0)).any()          # the filter removed something
        assert np.all((want == 0) | (want == plain))       # and changed nothing else


def test_zbuffer_with_all_points_on_one_pixel_and_a_wall(emu):
    cams = [(0, 5, 6, (4.0, 4.0, 2.5, 2.0))]
    I = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(f32).reshape(1, 12)
    rng = np.random.default_rng(5)
    z = rng.uniform(1, 50, 1000).astype(f32)
    pts = np.stack([np.zeros_like(z), np.zeros_like(z), z, z], 1)
    got = O.host_zbuffer(emu, cams, [0], [0, 30], pts, [0, 1000], [0], [0], I, 0.1, 80.0)
    want = np.zeros(30, f32)
    want[2 * 6 + 3] = z.min()      # uf = (4 * 0) / z + 2.5 -> u = floor(3.0) = 3; vf = 2 -> v = 2
    assert _same(got, want)
    assert _same(O.zbuffer(cams, [0], [0, 30], pts, [0, 1000], [0], [0], I, 0.1, 80.0), want)


# ---------------------------------------------------------------------------------------------------- readers
def test_load_velodyne_and_its_refusals(tmp_path):
    pts = np.arange(40, dtype=f32).reshape(10, 4)
    pts.tofile(tmp_path / "a.bin")
    assert _same(L.load_velodyne(tmp_path / "a.bin"), pts)
    (tmp_path / "b.bin").write_bytes(pts.tobytes()[:-4])
    with pytest.raises(ValueError, match="b.bin: 156 bytes is not a whole number of points"):
        L.load_velodyne(tmp_path / "b.bin")
    with pytest.raises(FileNotFoundError, match="missing Velodyne scan"):
        L.load_velodyne(tmp_path / "c.bin")
    (tmp_path / "e.bin").write_bytes(b"")
    assert L.load_velodyne(tmp_path / "e.bin").shape == (0, 4)


def test_load_cam_to_velo_and_its_refusal(tmp_path):
    m = np.arange(12, dtype=np.float64).reshape(3, 4) / 7
    (tmp_path / "c.txt").write_text(" ".join(repr(float(x)) for x in m.reshape(-1)) + "\n")
    got = L.load_cam_to_velo(tmp_path / "c.txt")
    assert np.array_equal(got[:3], m) and np.array_equal(got[3], [0, 0, 0, 1])
    (tmp_path / "d.txt").write_text("1 2 3\n")
    with pytest.raises(ValueError, match="d.txt: expected 12 numbers, got 3"):
        L.load_cam_to_velo(tmp_path / "d.txt")


def test_the_transform_chain_puts_a_world_point_on_its_pixel(tmp_path, emu):
    seq = O.write_sequence(tmp_path, [5, 6])
    # a world point 12 m in front of camera 0 at frame 5, on pixel (u, v) = (9, 17) (z = 12: x = (9 - 15.5) 12 / 20)
    u, v, z = 9, 17, 12.0
    pc = np.array([(u - 15.5) * z / 20.0, (v - 11.5) * z / 20.0, z, 1.0])
    pw = seq["c0w"][5] @ pc
    # the same point in the Velodyne frame of scan 6: world -> velo = cam_to_velo @ inv(cam_to_pose) @ inv(poses[6])
    pv = seq["c2v"] @ np.linalg.inv(seq["c2p"]["image_00"]) @ np.linalg.inv(seq["imu"][6]) @ pw
    rows = L.frame_scans([("image_00", 5)], tmp_path, seq["seq"], lidar_window=1)
    assert [s for s, _ in rows[0]] == [5, 6]            # scan 4 has no pose or file: skipped
    M = dict(rows[0])[6]
    cam = (0, 24, 32, (20.0, 20.0, 15.5, 11.5))
    ok, pix, t = O.host_point(emu, cam, M, pv[None, :3], 0.1, 80.0)
    assert ok[0] and pix[0] == v * 32 + u and abs(t[0] - z) < 1e-4
    # a fisheye frame: its pose is poses.txt @ cam_to_pose["image_02"]
    rows = L.frame_scans([("image_02", 6)], tmp_path, seq["seq"])
    want = np.linalg.inv(seq["imu"][6] @ seq["c2p"]["image_02"]) @ seq["imu"][6] @ seq["c2p"]["image_00"] @ \
        np.linalg.inv(seq["c2v"])
    assert _same(rows[0][0][1], want[:3, :4].astype(f32))


def test_frame_scans_and_lidar_depth_refuse_by_name(tmp_path):
    seq = O.write_sequence(tmp_path, [5, 6, 7], scans=[5, 7])["seq"]
    with pytest.raises(FileNotFoundError, match="0000000006.bin: missing Velodyne scan of frame 6"):
        L.frame_scans([("image_00", 6)], tmp_path, seq)
    with pytest.raises(ValueError, match="poses.txt: no pose for frame 9"):
        L.frame_scans([("image_02", 9)], tmp_path, seq)
    with pytest.raises(ValueError, match="cam0_to_world.txt: no pose for frame 9"):
        L.frame_scans([("image_00", 9)], tmp_path, seq)
    with pytest.raises(ValueError, match="not of a KITTI-360 camera"):
        L.frame_scans([("image_05", 5)], tmp_path, seq)
    assert [s for s, _ in L.frame_scans([("image_00", 6 - 1)], tmp_path, seq, 2)[0]] == [5, 7]
    fs = FrameSet.from_images([Camera("pinhole", 24, 32, (20, 20, 15.5, 11.5))], [0],
                              np.eye(4)[:3][None], [torch.zeros(24, 32, 3, dtype=torch.uint8)],
                              names=[("image_00", 6)], device="cpu")
    bad = [dict(lidar_window=-1), dict(lidar_window=1.5), dict(min_depth=0.0), dict(min_depth=float("nan")),
           dict(max_depth=0.05), dict(max_depth=float("inf")), dict(occlusion_radius=9),
           dict(occlusion_radius=-1), dict(occlusion_margin=1.0, occlusion_radius=1),
           dict(occlusion_margin=0.0, occlusion_radius=1), dict(chunk_frames=0)]
    for kw in bad:
        with pytest.raises(ValueError, match=f"lidar_depth: {next(iter(kw))}="):
            L.lidar_depth(fs, tmp_path, seq, **kw)
    with pytest.raises(FileNotFoundError, match="frame 6"):
        L.lidar_depth(fs, tmp_path, seq)
    assert fs.depth is None                                 # refused before anything was allocated
    unnamed = FrameSet(fs.cameras, fs.c2w, fs.frame_cam, fs.pix_offset, fs.rgb8)
    with pytest.raises(ValueError, match="names 0 of its 1 frames"):
        L.lidar_depth(unnamed, tmp_path, seq)


def test_load_frames_refuses_lidar_with_depth_dir(tmp_path):
    seq = O.write_sequence(tmp_path, [5])["seq"]
    with pytest.raises(ValueError, match="lidar and depth_dir both give the depth table"):
        load_frames(tmp_path, seq, [5], depth_dir=tmp_path, lidar=True, device="cpu")
    with pytest.raises(ValueError, match="lidar=.*keys from"):
        load_frames(tmp_path, seq, [5], lidar={"window": 2}, device="cpu")


def test_save_depth_png_round_trips_through_load_frames(tmp_path):
    seq = O.write_sequence(tmp_path, [5, 6])["seq"]
    rng = np.random.default_rng(2)
    d = rng.uniform(0, 300, (2, 24, 32)).astype(f32)
    d[:, 0, :4] = [0.0, 1 / 512, 3 / 512, 255.998]        # ties of the rounding (to even) and the last code
    d[:, 1, :2] = [65535.5 / 256, 65536 / 256]            # both above 65535 after rounding -> 0
    (tmp_path / "depth").mkdir()
    dropped = [L.save_depth_png(d[i], tmp_path / "depth" / f"{f:010d}.png") for i, f in enumerate((5, 6))]
    code = np.rint(d * f32(256))
    assert dropped == [int((code[i] > 65535).sum()) for i in range(2)]
    fs = load_frames(tmp_path, seq, [5, 6], depth_dir=tmp_path / "depth", device="cpu")
    want = np.where(code > 65535, 0, code).astype(f32) / f32(256)
    assert _same(fs.depth.numpy(), want.reshape(-1))
    assert want[0, 0, 1] == 0 and want[0, 0, 2] == f32(4 / 512)   # 0.5 -> 0, 1.5 -> 2 (ties to even)


def test_load_frames_without_lidar_is_unchanged(tmp_path):
    seq = O.write_sequence(tmp_path, [5, 6])["seq"]
    a = load_frames(tmp_path, seq, [5, 6], device="cpu")
    b = load_frames(tmp_path, seq, [5, 6], device="cpu", lidar=False)
    assert a.depth is None and b.depth is None and torch.equal(a.c2w, b.c2w) and torch.equal(a.rgb8, b.rgb8)


# ---------------------------------------------------------------------------------------------------- C ABI
def _valid_args(keep):
    cams = [O.PINHOLE, O.FISHEYE]
    a, _, keep = O.args_struct(cams, [0, 1], [0, 376 * 1408, 376 * 1408 + 1400 * 1400], np.zeros((8, 4), f32),
                               [0, 4, 8], [0, 1], [1, 0], np.tile(np.eye(3, 4, dtype=f32).reshape(12), (2, 1)),
                               0.1, 80.0, keep=keep)
    # the device pointers of a real call: never dereferenced before the checks pass
    a.points, a.frame_cam, a.pix_offset, a.depth = 0x100000, 0x200000, 0x300000, 0x400000
    return a


def _refused(a, what):
    rc = _capi.lib().pnr_project_depth(C.byref(a), None)
    assert rc == -1
    msg = _capi.lib().pnr_last_error().decode()
    assert what in msg, msg


def test_every_argument_is_refused_by_name_before_any_device_call():
    keep = []
    bad_so = np.array([0, 5, 3], np.int64)
    neg_so = np.array([-1, 4, 8], np.int64)
    past_so = np.array([0, 4, 9], np.int64)
    bad_pf = np.array([0, 2], np.int32)
    bad_ps = np.array([0, 2], np.int32)
    keep += [bad_so, neg_so, past_so, bad_pf, bad_ps]
    cases = [
        (lambda a: setattr(a, "F", 0), "F=0"),
        (lambda a: setattr(a, "P", 0), "P=0"),
        (lambda a: setattr(a, "Q", -1), "Q=-1"),
        (lambda a: setattr(a, "S", -1), "S=-1"),
        (lambda a: setattr(a, "Npts", -1), "Npts=-1"),
        (lambda a: setattr(a, "num_cameras", 0), "num_cameras=0"),
        (lambda a: setattr(a, "num_cameras", 5), "num_cameras=5"),
        (lambda a: setattr(a.cams[1], "model", 1), "camera 1 is equirect"),
        (lambda a: setattr(a.cams[0], "model", 3), "camera 0 model 3"),
        (lambda a: setattr(a.cams[0], "W", 0), "camera 0 size"),
        (lambda a: setattr(a.cams[1], "H", 1 << 24), "camera 1 size"),
        (lambda a: setattr(a, "min_depth", 0.0), "min_depth=0"),
        (lambda a: setattr(a, "min_depth", float("inf")), "min_depth=inf"),
        (lambda a: setattr(a, "max_depth", 0.1), "max_depth=0.1"),
        (lambda a: setattr(a, "max_depth", float("nan")), "max_depth=nan"),
        (lambda a: setattr(a, "occlusion_radius", 9), "occlusion_radius=9"),
        (lambda a: setattr(a, "occlusion_radius", -1), "occlusion_radius=-1"),
        (lambda a: (setattr(a, "occlusion_radius", 2), setattr(a, "occlusion_margin", 1.0)), "occlusion_margin=1"),
        (lambda a: (setattr(a, "occlusion_radius", 2), setattr(a, "occlusion_margin", 0.0)), "occlusion_margin=0"),
        (lambda a: setattr(a, "frame_cam", None), "null frame-set pointer"),
        (lambda a: setattr(a, "depth", None), "null frame-set pointer"),
        (lambda a: setattr(a, "scan_offset", None), "null scan_offset"),
        (lambda a: setattr(a, "pair_M", None), "null pair table"),
        (lambda a: setattr(a, "points", None), "null points"),
        (lambda a: setattr(a, "points", 0x100004), "points is not 16-byte aligned"),
        (lambda a: setattr(a, "scan_offset", bad_so.ctypes.data), "scan_offset decreases at 2"),
        (lambda a: setattr(a, "scan_offset", neg_so.ctypes.data), "scan_offset[0]=-1"),
        (lambda a: setattr(a, "scan_offset", past_so.ctypes.data), "scan_offset[2]=9"),
        (lambda a: setattr(a, "pair_frame", bad_pf.ctypes.data), "pair_frame[1]=2"),
        (lambda a: setattr(a, "pair_scan", bad_ps.ctypes.data), "pair_scan[1]=2"),
        (lambda a: setattr(a, "occlusion_radius", 1), "workspace of 0 bytes"),
        (lambda a: (setattr(a, "occlusion_radius", 1), setattr(a, "workspace", 0x500000),
                    setattr(a, "workspace_bytes", 100)), "the filter needs"),
        (lambda a: (setattr(a, "occlusion_radius", 1), setattr(a, "workspace", 0x500008),
                    setattr(a, "workspace_bytes", 1 << 40)), "16-byte aligned"),
    ]
    for mutate, what in cases:
        a = _valid_args(keep)
        mutate(a)
        _refused(a, what)
    assert _capi.lib().pnr_project_depth(None, None) == -1
    P = 376 * 1408 + 1400 * 1400
    assert _capi.lib().pnr_project_depth_workspace_bytes(P, 0) == 0
    assert _capi.lib().pnr_project_depth_workspace_bytes(P, 3) == (4 * P + 15) // 16 * 16
    assert _capi.lib().pnr_project_depth_workspace_bytes(P, 9) == 0
    assert _capi.lib().pnr_project_depth_workspace_bytes(0, 1) == 0


def test_an_empty_pair_table_is_accepted_without_a_device():
    a = _valid_args([])
    a.Q = 0
    assert _capi.lib().pnr_project_depth(C.byref(a), None) == 0


def test_project_depth_args_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _capi.PnrProjectDepthArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(pnr_project_depth_args, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(pnr_project_depth_args));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [getattr(_capi.PnrProjectDepthArgs, f).offset for f in fields] + [C.sizeof(_capi.PnrProjectDepthArgs)]
    assert got == want
