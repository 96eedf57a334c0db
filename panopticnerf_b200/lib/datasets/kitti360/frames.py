"""KITTI-360 frames of one camera -> a device FrameSet (lib/datasets/ray_batch.py) for training-batch sampling.

Layout under `root` (public KITTI-360 layout):
  data_2d_raw/<seq>/image_00/data_rect/<frame:010d>.png     rectified perspective camera, 8-bit colour
  data_2d_raw/<seq>/image_02|03/data_rgb/<frame:010d>.png   fisheye cameras, 8-bit colour
  calibration/perspective.txt (P_rect_00, S_rect_00), calibration/image_02.yaml / image_03.yaml,
  calibration/calib_cam_to_pose.txt, data_poses/<seq>/cam0_to_world.txt, data_poses/<seq>/poses.txt
Poses: image_00 -> cam0_to_world[frame]; image_02 / image_03 -> poses.txt[frame] @ calib_cam_to_pose[camera].

Targets (rules chosen here, one format per kind; the reference's preprocessing is not in the mount):
  <pseudo_dir>/<frame:010d>.png   8-bit single channel, KITTI-360 semanticIds, mapped to class channels through
                                  sem_to_train as primitive_batch maps box ids (an id without a channel -> -1; no
                                  table: the id itself)
  <depth_dir>/<frame:010d>.png    16-bit single channel, metres x 256, 0 = no depth (the KITTI depth encoding)
A missing file, a wrong bit depth or channel count and an image whose size is not its camera's calibration are refused
by name."""
from __future__ import annotations

from pathlib import Path
from typing import Dict, Iterable, Optional

import numpy as np
import torch

from ..ray_batch import Camera, FrameSet
from .calib import (fisheye_to_world, load_cam0_to_world, load_cam_to_pose, load_fisheye_yaml, load_perspective,
                    load_poses)

CAMERAS = ("image_00", "image_02", "image_03")


def _read(path: Path, what: str, dtype, channels: int) -> np.ndarray:
    import cv2
    if not path.is_file():
        raise FileNotFoundError(f"{path}: missing {what}")
    img = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    if img is None:
        raise ValueError(f"{path}: not a readable image ({what})")
    got = 1 if img.ndim == 2 else img.shape[2]
    if got != channels:
        raise ValueError(f"{path}: {what} must have {channels} channel(s), got {got}")
    if img.dtype != dtype:
        raise ValueError(f"{path}: {what} must be {np.dtype(dtype).itemsize * 8}-bit, got {img.dtype}")
    return img


def _sized(img: np.ndarray, cam: Camera, path: Path, what: str) -> np.ndarray:
    if img.shape[:2] != (cam.H, cam.W):
        raise ValueError(f"{path}: {what} is {img.shape[1]} x {img.shape[0]}, its camera's calibration says "
                         f"{cam.W} x {cam.H}")
    return img


def camera_of(root, camera: str) -> Camera:
    """The calibrated camera of `camera` (image_00: P_rect_00 and S_rect_00; image_02 / 03: the MEI yaml)."""
    cal = Path(root) / "calibration"
    if camera == "image_00":
        p = load_perspective(cal / "perspective.txt", 0)
        if p["size"] is None:
            raise ValueError(f"{cal / 'perspective.txt'}: no S_rect_00 (the image size)")
        K = p["K"]
        return Camera("pinhole", p["size"][1], p["size"][0], (K[0, 0], K[1, 1], K[0, 2], K[1, 2]))
    fe = load_fisheye_yaml(cal / f"{camera}.yaml")
    if "image_width" not in fe or "image_height" not in fe:
        raise ValueError(f"{cal / (camera + '.yaml')}: no image_width / image_height")
    return Camera("fisheye", int(fe["image_height"]), int(fe["image_width"]),
                  tuple(fe[k] for k in ("gamma1", "gamma2", "u0", "v0", "xi", "k1", "k2")))


def camera_poses(root, seq: str, camera: str):
    """(pose_of, src): pose_of(frame) -> the float64 4x4 camera -> world of `camera` at `frame` (KeyError without a
    pose), src the pose file it reads.  image_00: cam0_to_world; image_02 / 03: poses.txt @ calib_cam_to_pose."""
    root = Path(root)
    poses = root / "data_poses" / seq
    if camera == "image_00":
        table = load_cam0_to_world(poses / "cam0_to_world.txt")
        return (lambda f: table[f]), poses / "cam0_to_world.txt"
    imu = load_poses(poses / "poses.txt")
    c2p = load_cam_to_pose(root / "calibration" / "calib_cam_to_pose.txt")
    if camera not in c2p:
        raise ValueError(f"{root / 'calibration' / 'calib_cam_to_pose.txt'}: no {camera}")
    return (lambda f: fisheye_to_world(c2p[camera], imu[f])), poses / "poses.txt"


def load_frames(root, seq: str, frames: Iterable[int], camera: str = "image_00", pseudo_dir=None, depth_dir=None,
                sem_to_train: Optional[Dict[int, int]] = None, device="cuda", lidar=False, stereo=False) -> FrameSet:
    """The frames `frames` of sequence `seq` seen by `camera`, on `device` (module docstring: layout and formats).
    lidar: False, True or a dict of `lidar.lidar_depth` options - the depth table from the sequence's Velodyne scans
    instead of depth_dir's PNGs (the two are refused together).
    stereo: False, True or a dict of `stereo.stereo_depth` options - the depth table from the image_00 / image_01
    pair by semi-global matching (refused together with depth_dir or lidar)."""
    if camera not in CAMERAS:
        raise ValueError(f"load_frames: camera {camera!r}; one of {CAMERAS}")
    from .lidar import LIDAR_OPTIONS, lidar_depth
    from .stereo import STEREO_OPTIONS, stereo_depth
    # the sources of the depth table, at most one per call: (name, value, option keys, fill).  depth_dir's PNGs are read
    # with the images; lidar / stereo are on unless False or None ({} is on, with the defaults).
    source = None
    for name, value, keys, fill in (("depth_dir", depth_dir, None, None), ("lidar", lidar, LIDAR_OPTIONS, lidar_depth),
                                    ("stereo", stereo, STEREO_OPTIONS, stereo_depth)):
        if value is None or (keys is not None and value is False):
            continue
        if source is not None:
            raise ValueError(f"load_frames: {name} and {source[0]} both give the depth table; pass one of them")
        if keys is not None and value is not True and (not isinstance(value, dict) or set(value) - set(keys)):
            raise ValueError(f"load_frames: {name}={value!r}; False, True or a dict with keys from {keys}")
        source = (name, value, fill)
    root = Path(root)
    frames = [int(f) for f in frames]
    if not frames:
        raise ValueError("load_frames: no frames")
    cam = camera_of(root, camera)
    pose_of, src = camera_poses(root, seq, camera)
    images = root / "data_2d_raw" / seq / camera / ("data_rect" if camera == "image_00" else "data_rgb")
    lut = None
    if sem_to_train is not None:
        lut = np.full(256, -1, dtype=np.int16)
        for k, v in sem_to_train.items():
            if 0 <= int(k) < 256:
                lut[int(k)] = int(v)
    c2w, rgb, lab, dep = [], [], [], []
    for f in frames:
        try:
            c2w.append(np.asarray(pose_of(f), dtype=np.float64)[:3, :4])
        except KeyError:
            raise ValueError(f"{src}: no pose for frame {f}") from None
        name = f"{f:010d}.png"
        bgr = _sized(_read(images / name, "a colour image", np.uint8, 3), cam, images / name, "the colour image")
        rgb.append(torch.from_numpy(np.ascontiguousarray(bgr[:, :, ::-1])))
        if pseudo_dir is not None:
            p = Path(pseudo_dir) / name
            ids = _sized(_read(p, "a pseudo-label image", np.uint8, 1), cam, p, "the pseudo-label image")
            lab.append(torch.from_numpy(lut[ids] if lut is not None else ids.astype(np.int16)))
        if depth_dir is not None:
            p = Path(depth_dir) / name
            d = _sized(_read(p, "a depth image", np.uint16, 1), cam, p, "the depth image")
            dep.append(torch.from_numpy(d.astype(np.float32) / np.float32(256.0)))
    fs = FrameSet.from_images([cam], [0] * len(frames), np.stack(c2w).astype(np.float32), rgb,
                              lab if pseudo_dir is not None else None, dep if depth_dir is not None else None,
                              [(camera, f) for f in frames], device)
    if source is not None and source[2] is not None:
        source[2](fs, root, seq, **({} if source[1] is True else source[1]))
    return fs


def check_depth_range(what: str, min_depth, max_depth) -> None:
    """The depth limits of a depth source (`what` names it): min_depth finite and > 0, max_depth finite and above it."""
    if not (np.isfinite(min_depth) and min_depth > 0):
        raise ValueError(f"{what}: min_depth={min_depth}; finite and > 0")
    if not (np.isfinite(max_depth) and max_depth > min_depth):
        raise ValueError(f"{what}: max_depth={max_depth}; finite and > min_depth={min_depth}")


def check_names(frames: FrameSet, what: str) -> None:
    """A depth source finds each frame of the set by its (camera, frame id) in frames.names."""
    if len(frames.names) != frames.num_frames:
        raise ValueError(f"{what}: the set names {len(frames.names)} of its {frames.num_frames} frames; each frame needs "
                         "its (camera, frame id)")


def ensure_depth(frames: FrameSet) -> None:
    """Allocate frames.depth (zero: no depth) when the set has none."""
    if frames.depth is None:
        frames.depth = torch.zeros(frames.num_pixels, dtype=torch.float32, device=frames.rgb8.device)


__all__ = ["CAMERAS", "camera_of", "camera_poses", "load_frames"]
