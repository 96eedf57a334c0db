"""numpy float32 oracle of pnr_project_depth (include/pnr.h, DESIGN 3.4): the same operation order as
pnr_project_point / pnr_depth_pixel of ray_math.h, every operation a rounded float32 one (numpy does not contract to
FMA; its sqrt and division are correctly rounded), and helpers to call the host build (tests/host_emu.cpp)."""
import ctypes as C
from pathlib import Path

import numpy as np

from panopticnerf_b200 import _capi

f32 = np.float32


def camera_struct(cam):
    """cam = (model, H, W, intr) -> pnr_ray_camera."""
    model, H, W, intr = cam
    c = _capi.PnrRayCamera()
    c.model, c.H, c.W = int(model), int(H), int(W)
    for i, x in enumerate(intr):
        c.intr[i] = float(x)
    return c


def host_point(lib, cam, M, p, min_depth, max_depth):
    """The host build on each point of p [n, 3]: (ok [n] bool, pix [n] i64 (-1 where not), t [n] f32 (0 where not))."""
    c = camera_struct(cam)
    Mf = np.ascontiguousarray(M, dtype=f32).reshape(12)
    ok = np.zeros(len(p), bool)
    pix = np.full(len(p), -1, np.int64)
    t = np.zeros(len(p), f32)
    q, tt = C.c_int64(), C.c_float()
    for i, (x, y, z) in enumerate(np.asarray(p, f32)):
        if lib.emu_project_point(C.byref(c), Mf.ctypes.data, float(x), float(y), float(z), float(min_depth),
                                 float(max_depth), C.byref(q), C.byref(tt)):
            ok[i], pix[i], t[i] = True, q.value, tt.value
    return ok, pix, t


def project_points(cam, M, p, min_depth, max_depth, want_uv=False):
    """The oracle of pnr_project_point on p [n, 3] -> (ok, pix, t) as host_point (and (uf, vf) with want_uv)."""
    model, H, W, intr = cam
    M = np.asarray(M, dtype=f32).reshape(12)
    intr = [f32(v) for v in intr]
    p = np.asarray(p, f32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    mind, maxd = f32(min_depth), f32(max_depth)
    with np.errstate(all="ignore"):
        xc = ((M[0] * x + M[1] * y) + M[2] * z) + M[3]
        yc = ((M[4] * x + M[5] * y) + M[6] * z) + M[7]
        zc = ((M[8] * x + M[9] * y) + M[10] * z) + M[11]
        if model == 0:
            fx, fy, cx, cy = intr[:4]
            t = zc
            ok = (t > mind) & (t <= maxd)
            uf = (fx * xc) / zc + cx
            vf = (fy * yc) / zc + cy
        else:
            g1, g2, u0, v0, xi, k1, k2 = intr
            n = np.sqrt((xc * xc + yc * yc) + zc * zc)
            xs, ys, zs = xc / n, yc / n, zc / n
            den = zs + xi
            ok = den > 0
            mx, my = xs / den, ys / den
            r2 = mx * mx + my * my
            d = (f32(1) + k1 * r2) + k2 * (r2 * r2)
            uf = (g1 * mx) * d + u0
            vf = (g2 * my) * d + v0
            t = n
            ok &= (t > mind) & (t <= maxd)
        fu, fv = np.floor(uf + f32(0.5)), np.floor(vf + f32(0.5))
        ok &= (fu >= 0) & (fu < f32(W)) & (fv >= 0) & (fv < f32(H))
    pix = np.where(ok, np.where(ok, fv, 0).astype(np.int64) * W + np.where(ok, fu, 0).astype(np.int64), -1)
    t = np.where(ok, t, f32(0)).astype(f32)
    return (ok, pix, t, uf, vf) if want_uv else (ok, pix, t)


def zbuffer(cams, frame_cam, pix_offset, points, scan_offset, pair_frame, pair_scan, pair_M, min_depth, max_depth,
            radius=0, margin=0.1, depth_in=None):
    """The whole call on well-formed tables: depth [P] f32 (depth_in outside the named frames)."""
    P = int(pix_offset[-1])
    depth = np.zeros(P, f32) if depth_in is None else np.array(depth_in, f32)
    z = np.full(P, np.inf, f32)
    for k in range(len(pair_frame)):
        f, s = int(pair_frame[k]), int(pair_scan[k])
        lo = int(pix_offset[f])
        pts = np.asarray(points, f32)[int(scan_offset[s]):int(scan_offset[s + 1]), :3]
        ok, pix, t = project_points(cams[frame_cam[f]], pair_M[k], pts, min_depth, max_depth)
        np.minimum.at(z, lo + pix[ok], t[ok])
    for f in sorted(set(int(x) for x in pair_frame)):
        model, H, W, _ = cams[frame_cam[f]]
        lo = int(pix_offset[f])
        zf = z[lo:lo + H * W].reshape(H, W)
        out = np.where(np.isinf(zf), f32(0), zf)
        if radius > 0:
            pad = np.full((H + 2 * radius, W + 2 * radius), np.inf, f32)
            pad[radius:radius + H, radius:radius + W] = zf
            m = np.full((H, W), np.inf, f32)
            for dv in range(2 * radius + 1):
                for du in range(2 * radius + 1):
                    m = np.minimum(m, pad[dv:dv + H, du:du + W])
            thr = m * (f32(1) + f32(margin))
            out = np.where(np.isfinite(zf) & (zf <= thr), zf, f32(0))
        depth[lo:lo + H * W] = out.reshape(-1)
    return depth


def args_struct(cams, frame_cam, pix_offset, points, scan_offset, pair_frame, pair_scan, pair_M, min_depth, max_depth,
                radius=0, margin=0.1, depth=None, keep=None):
    """pnr_project_depth_args over host arrays (for the host build); `keep` collects the arrays it points into."""
    keep = [] if keep is None else keep
    arr = lambda x, dt: keep.append(np.ascontiguousarray(x, dtype=dt)) or keep[-1]
    a = _capi.PnrProjectDepthArgs()
    pts = arr(points, f32).reshape(-1, 4)
    a.points, a.Npts = pts.ctypes.data, pts.shape[0]
    so = arr(scan_offset, np.int64)
    a.scan_offset, a.S = so.ctypes.data, so.size - 1
    pf, ps, pm = arr(pair_frame, np.int32), arr(pair_scan, np.int32), arr(pair_M, f32)
    a.pair_frame, a.pair_scan, a.pair_M, a.Q = pf.ctypes.data, ps.ctypes.data, pm.ctypes.data, pf.size
    fc, po = arr(frame_cam, np.int32), arr(pix_offset, np.int64)
    a.frame_cam, a.pix_offset, a.F, a.P = fc.ctypes.data, po.ctypes.data, fc.size, int(po[-1])
    for k, c in enumerate(cams):
        a.cams[k] = camera_struct(c)
    a.num_cameras = len(cams)
    a.min_depth, a.max_depth, a.occlusion_radius, a.occlusion_margin = min_depth, max_depth, radius, margin
    if depth is None:
        depth = arr(np.zeros(a.P, f32), f32)
    a.depth = depth.ctypes.data
    return a, depth, keep


def host_zbuffer(lib, *args, **kw):
    """The host build of the whole call (same arguments as zbuffer) -> depth [P] f32."""
    depth_in = kw.pop("depth_in", None)
    P = int(args[2][-1])
    depth = np.zeros(P, f32) if depth_in is None else np.array(depth_in, f32)
    a, depth, keep = args_struct(*args, depth=depth, **kw)
    lib.emu_project_depth(C.byref(a))
    return depth


def random_scene(rng, cams, F, S, n_lo, n_hi, pairs_per_frame=1, spread=20.0):
    """A frame set of F frames over `cams` and S random scans (points in front of the cameras and around them), with
    random pairs and near-identity random rigid M.  Returns (frame_cam, pix_offset, points [N, 4], scan_offset,
    pair_frame, pair_scan, pair_M)."""
    frame_cam = rng.integers(0, len(cams), F).astype(np.int32)
    sizes = [cams[c][1] * cams[c][2] for c in frame_cam]
    pix_offset = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    counts = rng.integers(n_lo, n_hi + 1, S)
    scan_offset = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    N = int(scan_offset[-1])
    pts = np.empty((N, 4), f32)
    pts[:, 0] = rng.uniform(-spread, spread, N)
    pts[:, 1] = rng.uniform(-spread / 4, spread / 4, N)
    pts[:, 2] = rng.uniform(-spread / 4, 3 * spread, N)
    pts[:, 3] = rng.uniform(0, 1, N)
    pf, ps, pm = [], [], []
    for f in range(F):
        for s in rng.choice(S, size=min(S, pairs_per_frame), replace=False):
            a = rng.uniform(-0.1, 0.1, 3)
            R = rotation(a)
            M = np.concatenate([R, rng.uniform(-1, 1, (3, 1))], 1)
            pf.append(f), ps.append(int(s)), pm.append(M.astype(f32).reshape(12))
    return (frame_cam, pix_offset, pts, scan_offset, np.array(pf, np.int32), np.array(ps, np.int32),
            np.array(pm, f32).reshape(-1, 12))


def rotation(a):
    cx, cy, cz = np.cos(a)
    sx, sy, sz = np.sin(a)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


# A small sequence in the KITTI-360 layout: a pinhole image_00, a fisheye image_02, poses far from the origin (as in
# KITTI-360, thousands of metres), and the rigid transforms of the calibration.
WORLD0 = np.array([1834.25, -3710.5, 115.75])   # the poses' offset from the world origin


def _rigid(rng, scale=0.3, t=1.0):
    M = np.eye(4)
    M[:3, :3] = rotation(rng.uniform(-scale, scale, 3))
    M[:3, 3] = rng.uniform(-t, t, 3)
    return M


def write_sequence(root: Path, frames, seq="2013_05_28_drive_0000_sync", cams=("image_00", "image_02"), scans=None,
                   rng=None, images=True, points=None, world0=WORLD0):
    """Calibration, poses, colour images (with `images`) and scans (points(f) -> [n, 4], default random) of `frames`
    (scans of `scans` when given).  Returns dict(imu, c2p, c2v, c0w, seq)."""
    import cv2
    rng = rng or np.random.default_rng(0)
    cal = root / "calibration"
    cal.mkdir(parents=True, exist_ok=True)
    m, H, W, intr = 0, 24, 32, (20.0, 20.0, 15.5, 11.5)
    (cal / "perspective.txt").write_text(f"P_rect_00: {intr[0]} 0 {intr[2]} 0 0 {intr[1]} {intr[3]} 0 0 0 1 0\n"
                                         f"S_rect_00: {W} {H}\n")
    (cal / "image_02.yaml").write_text("%YAML:1.0\n---\nmodel_type: MEI\ncamera_name: image_02\nimage_width: 30\n"
                                       "image_height: 28\nmirror_parameters:\n   xi: 1.5\ndistortion_parameters:\n"
                                       "   k1: 0.02\n   k2: 0.1\n   p1: 0.0\n   p2: 0.0\nprojection_parameters:\n"
                                       "   gamma1: 20.0\n   gamma2: 19.5\n   u0: 14.5\n   v0: 13.5\n")
    c2p = {k: _rigid(rng) for k in ("image_00", "image_01", "image_02", "image_03")}
    c2v = _rigid(rng)
    fmt = lambda M, n: " ".join(repr(float(x)) for x in M[:n].reshape(-1))
    (cal / "calib_cam_to_pose.txt").write_text("".join(f"{k}: {fmt(v, 3)}\n" for k, v in c2p.items()))
    (cal / "calib_cam_to_velo.txt").write_text(fmt(c2v, 3) + "\n")
    pd = root / "data_poses" / seq
    pd.mkdir(parents=True, exist_ok=True)
    imu = {}
    for f in frames:
        P = _rigid(rng, 0.2, 3.0)
        P[:3, 3] += np.asarray(world0) + [2.0 * f, 0.5 * f, 0]
        imu[f] = P
    (pd / "poses.txt").write_text("".join(f"{f} {fmt(imu[f], 3)}\n" for f in frames))
    # rectified camera 0 -> world: the unrectified one (R_rect = I here)
    c0w = {f: imu[f] @ c2p["image_00"] for f in frames}
    (pd / "cam0_to_world.txt").write_text("".join(f"{f} {fmt(c0w[f], 4)}\n" for f in frames))
    if images:
        for cam, (h, w) in (("image_00", (H, W)), ("image_02", (28, 30))):
            if cam not in cams:
                continue
            d = root / "data_2d_raw" / seq / cam / ("data_rect" if cam == "image_00" else "data_rgb")
            d.mkdir(parents=True, exist_ok=True)
            for f in frames:
                cv2.imwrite(str(d / f"{f:010d}.png"), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    vd = root / "data_3d_raw" / seq / "velodyne_points" / "data"
    vd.mkdir(parents=True, exist_ok=True)
    for f in (frames if scans is None else scans):
        p = points(f) if points is not None else rng.uniform(-20, 20, (500, 4)).astype(f32)
        np.asarray(p, f32).tofile(vd / f"{f:010d}.bin")
    return {"imu": imu, "c2p": c2p, "c2v": c2v, "c0w": c0w, "seq": seq}


PINHOLE = (0, 376, 1408, (552.554, 552.554, 682.049, 238.77))      # KITTI-360 image_00 (rectified)
FISHEYE = (2, 1400, 1400, (1336.9, 1335.6, 716.9, 705.8, 2.2134, 0.01647, 1.6035))   # KITTI-360 image_02
