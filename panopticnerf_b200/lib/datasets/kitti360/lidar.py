"""KITTI-360 Velodyne scans -> the depth table of a FrameSet, projected on the device (`pnr_project_depth`, DESIGN 3.4).

Layout under `root` (public KITTI-360 layout):
  data_3d_raw/<seq>/velodyne_points/data/<frame:010d>.bin   float32 x4 per point: x, y, z (Velodyne frame), reflectance
  calibration/calib_cam_to_velo.txt                         one line of 12 numbers: unrectified camera 0 -> Velodyne
  calibration/calib_cam_to_pose.txt, data_poses/<seq>/poses.txt, the frames' own poses: as frames.py
Rules (chosen here; the reference's preprocessing is not public):
  scan s -> world:   poses.txt[s] @ calib_cam_to_pose["image_00"] @ inv(cam_to_velo)
  scan s -> frame f: M = inv(cam_to_world_f) @ (scan s -> world), composed in float64 and rounded to fp32 once, so the
                     device never sees world coordinates (thousands of metres in KITTI-360)
  window:            frame f takes the scans f - w .. f + w (lidar_window = w).  Its own scan and its poses.txt entry
                     must exist (refused by name otherwise); a neighbour without a scan file or a pose is skipped.  w > 0
                     densifies the static scene but smears whatever moves: a car's points from scan f + 1 land where the
                     car is not at frame f.  So the default is w = 0.
  depth:             the nearest point per pixel, in the units of the camera's ray direction (include/pnr.h), 0 = none;
                     optionally the occlusion filter (occlusion_radius > 0).
`save_depth_png` writes a set's depth in the KITTI encoding, so a projected set can be cached and read back through
`load_frames(depth_dir=...)`."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import torch

from .... import _capi
from ..ray_batch import FrameSet, fill_frame_store
from .calib import _floats, load_cam_to_pose, load_poses
from .frames import CAMERAS, camera_poses, check_depth_range, check_names, ensure_depth

DEFAULT_MIN_DEPTH = 0.1          # metres
DEFAULT_MAX_DEPTH = 80.0         # metres: the Velodyne HDL-64E's usable range
DEFAULT_OCCLUSION_MARGIN = 0.1
LIDAR_OPTIONS = ("lidar_window", "min_depth", "max_depth", "occlusion_radius", "occlusion_margin", "chunk_frames")


def scan_path(root, seq: str, frame: int) -> Path:
    return Path(root) / "data_3d_raw" / seq / "velodyne_points" / "data" / f"{int(frame):010d}.bin"


def load_velodyne(path) -> np.ndarray:
    """A Velodyne scan -> [N, 4] float32 (x, y, z, reflectance)."""
    path = Path(path)
    if not path.is_file():
        raise FileNotFoundError(f"{path}: missing Velodyne scan")
    size = path.stat().st_size
    if size % 16:
        raise ValueError(f"{path}: {size} bytes is not a whole number of points (16 bytes each: x, y, z, reflectance "
                         "as float32)")
    return np.fromfile(path, dtype="<f4").reshape(-1, 4)


def load_cam_to_velo(path) -> np.ndarray:
    """calib_cam_to_velo.txt (one line of 12 numbers, unrectified camera 0 -> Velodyne) -> 4x4 float64."""
    m = np.eye(4)
    m[:3, :4] = _floats(Path(path).read_text().split(), 12, str(path)).reshape(3, 4)
    return m


def velo_to_world(pose: np.ndarray, cam_to_pose: np.ndarray, cam_to_velo: np.ndarray) -> np.ndarray:
    """Scan -> world (float64 4x4): poses.txt[s] @ calib_cam_to_pose["image_00"] @ inv(cam_to_velo)."""
    return np.asarray(pose, np.float64) @ np.asarray(cam_to_pose, np.float64) @ np.linalg.inv(cam_to_velo)


def project_depth(frames: FrameSet, points: torch.Tensor, scan_offset, pair_frame, pair_scan, pair_M,
                  min_depth: float = DEFAULT_MIN_DEPTH, max_depth: float = DEFAULT_MAX_DEPTH,
                  occlusion_radius: int = 0, occlusion_margin: float = DEFAULT_OCCLUSION_MARGIN) -> None:
    """One `pnr_project_depth` call into frames.depth (which must exist): points [Npts, 4] f32 on the set's device;
    scan_offset [S+1], pair_frame / pair_scan [Q] and pair_M [Q, 12] (or [Q, 3, 4]) host arrays.  Rewrites every pixel
    of the frames some pair names and nothing else."""
    if frames.depth is None:
        raise ValueError("project_depth: the frame set has no depth table (lidar_depth allocates one)")
    dev = frames.rgb8.device
    so = np.ascontiguousarray(scan_offset, dtype=np.int64)
    pf = np.ascontiguousarray(pair_frame, dtype=np.int32)
    ps = np.ascontiguousarray(pair_scan, dtype=np.int32)
    pm = np.ascontiguousarray(pair_M, dtype=np.float32).reshape(-1, 12)
    if so.ndim != 1 or so.size < 1:
        raise ValueError(f"project_depth: scan_offset has shape {so.shape}; one entry per scan plus one")
    if not (pf.shape == ps.shape == (pm.shape[0],)):
        raise ValueError(f"project_depth: pair_frame {pf.shape}, pair_scan {ps.shape} and pair_M {pm.shape} disagree")
    if points.dim() != 2 or points.shape[1] != 4:
        raise ValueError(f"project_depth: points {tuple(points.shape)}; expected [Npts, 4]")
    a = _capi.PnrProjectDepthArgs()
    a.points, a.Npts = _capi.ptr(points, torch.float32, "points"), int(points.shape[0])
    a.scan_offset, a.S = so.ctypes.data, so.size - 1
    a.pair_frame, a.pair_scan, a.pair_M, a.Q = pf.ctypes.data, ps.ctypes.data, pm.ctypes.data, pf.size
    fill_frame_store(a, frames, "project_depth")
    a.min_depth, a.max_depth = float(min_depth), float(max_depth)
    a.occlusion_radius, a.occlusion_margin = int(occlusion_radius), float(occlusion_margin)
    a.depth = _capi.ptr(frames.depth, torch.float32, "depth")
    need = int(_capi.lib().pnr_project_depth_workspace_bytes(a.P, a.occlusion_radius))
    ws = torch.empty(need, dtype=torch.uint8, device=dev) if need else None   # freed in stream order
    if ws is not None:
        a.workspace, a.workspace_bytes = ws.data_ptr(), need
    with torch.cuda.device(dev):
        _capi.check(_capi.lib().pnr_project_depth(C.byref(a), _capi.stream_ptr()), "pnr_project_depth")


def _check_options(lidar_window, min_depth, max_depth, occlusion_radius, occlusion_margin, chunk_frames):
    if int(lidar_window) != lidar_window or lidar_window < 0:
        raise ValueError(f"lidar_depth: lidar_window={lidar_window}; an integer >= 0")
    check_depth_range("lidar_depth", min_depth, max_depth)
    if int(occlusion_radius) != occlusion_radius or not 0 <= occlusion_radius <= 8:
        raise ValueError(f"lidar_depth: occlusion_radius={occlusion_radius}; an integer in [0, 8]")
    if occlusion_radius > 0 and not 0 < occlusion_margin < 1:
        raise ValueError(f"lidar_depth: occlusion_margin={occlusion_margin}; in (0, 1)")
    if int(chunk_frames) != chunk_frames or chunk_frames < 1:
        raise ValueError(f"lidar_depth: chunk_frames={chunk_frames}; an integer >= 1")


def frame_scans(names, root, seq: str, lidar_window: int = 0):
    """Per frame (camera, frame id) of `names`: the list of (scan id, M) of its window, M the float32 3x4 scan -> camera
    matrix composed in float64 (module docstring).  Host only: reads the calibration and pose files, checks that every
    frame's own scan and poses exist (refused by name otherwise) and skips the neighbours without a scan or a pose."""
    if int(lidar_window) != lidar_window or lidar_window < 0:
        raise ValueError(f"lidar_depth: lidar_window={lidar_window}; an integer >= 0")
    w, root = int(lidar_window), Path(root)
    cal = root / "calibration"
    c2p = load_cam_to_pose(cal / "calib_cam_to_pose.txt")
    if "image_00" not in c2p:
        raise ValueError(f"{cal / 'calib_cam_to_pose.txt'}: no image_00")
    c2v = load_cam_to_velo(cal / "calib_cam_to_velo.txt")
    imu_path = root / "data_poses" / seq / "poses.txt"
    imu = load_poses(imu_path)
    readers, c2w = {}, []
    for camera, fid in names:
        if camera not in CAMERAS:
            raise ValueError(f"lidar_depth: frame ({camera!r}, {fid}) is not of a KITTI-360 camera {CAMERAS}")
        if camera not in readers:
            readers[camera] = camera_poses(root, seq, camera)
        pose_of, src = readers[camera]
        try:
            c2w.append(np.asarray(pose_of(int(fid)), dtype=np.float64))
        except KeyError:
            raise ValueError(f"{src}: no pose for frame {fid}") from None
        if int(fid) not in imu:
            raise ValueError(f"{imu_path}: no pose for frame {fid}, whose scan its depth comes from")
        if not scan_path(root, seq, fid).is_file():
            raise FileNotFoundError(f"{scan_path(root, seq, fid)}: missing Velodyne scan of frame {fid}")
    v2w = {}
    out = []
    for (camera, fid), pose in zip(names, c2w):
        w2c = np.linalg.inv(pose)
        row = []
        for s in range(int(fid) - w, int(fid) + w + 1):
            if s not in imu or not scan_path(root, seq, s).is_file():
                continue
            if s not in v2w:
                v2w[s] = velo_to_world(imu[s], c2p["image_00"], c2v)
            row.append((s, (w2c @ v2w[s])[:3, :4].astype(np.float32)))
        out.append(row)
    return out


def lidar_depth(frames: FrameSet, root, seq: str, lidar_window: int = 0, min_depth: float = DEFAULT_MIN_DEPTH,
                max_depth: float = DEFAULT_MAX_DEPTH, occlusion_radius: int = 0,
                occlusion_margin: float = DEFAULT_OCCLUSION_MARGIN, chunk_frames: int = 64) -> FrameSet:
    """Fill frames.depth (allocated, zero, when the set has none) from the Velodyne scans of `seq` under `root`
    (module docstring: layout and rules).  The frames are identified by frames.names (camera, frame id), as
    `load_frames` and `concat_frame_sets` leave them.  chunk_frames frames go to the device per call, with the scans
    their windows need, so the device holds at most chunk_frames + 2 w scans at a time.  Returns `frames`."""
    _check_options(lidar_window, min_depth, max_depth, occlusion_radius, occlusion_margin, chunk_frames)
    check_names(frames, "lidar_depth")
    pairs = frame_scans(frames.names, root, seq, lidar_window)
    ensure_depth(frames)
    F = frames.num_frames
    for f0 in range(0, F, int(chunk_frames)):
        chunk = range(f0, min(F, f0 + int(chunk_frames)))
        scans = sorted({s for f in chunk for s, _ in pairs[f]})
        index = {s: i for i, s in enumerate(scans)}
        pts = [load_velodyne(scan_path(root, seq, s)) for s in scans]
        offset = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int64)
        pair_frame = [f for f in chunk for _ in pairs[f]]
        pair_scan = [index[s] for f in chunk for s, _ in pairs[f]]
        pair_M = np.stack([M for f in chunk for _, M in pairs[f]])
        points = torch.from_numpy(np.concatenate(pts)).to(frames.rgb8.device)
        project_depth(frames, points, offset, pair_frame, pair_scan, pair_M, min_depth, max_depth, occlusion_radius,
                      occlusion_margin)
    return frames


def save_depth_png(depth_hw, path) -> int:
    """One frame's depth [H, W] (metres, 0 = none) as a 16-bit PNG of rne(t * 256) (the KITTI encoding that
    `load_frames(depth_dir=...)` reads).  A depth whose code is above 65535 (>= 255.998 m) is written as 0 (none);
    returns how many were."""
    import cv2
    d = depth_hw.detach().cpu().numpy() if isinstance(depth_hw, torch.Tensor) else np.asarray(depth_hw)
    if d.ndim != 2:
        raise ValueError(f"save_depth_png: depth has shape {d.shape}; expected [H, W]")
    q = np.rint(d.astype(np.float32) * np.float32(256.0))   # the product is exact; rint rounds half to even
    over = ~(q <= 65535)
    q[over | (q < 0)] = 0
    if not cv2.imwrite(str(path), q.astype(np.uint16)):
        raise ValueError(f"save_depth_png: could not write {path}")
    return int(over.sum())


__all__ = ["load_velodyne", "load_cam_to_velo", "velo_to_world", "frame_scans", "project_depth", "lidar_depth", "save_depth_png",
           "scan_path", "LIDAR_OPTIONS"]
