"""Camera masks for weighted training draws (ray_batch.pixel_weights): pixels a camera never trains on.

fisheye_fov_mask: the pixels whose ray lies within an angle of the optical axis - for KITTI-360's fisheyes, the
border outside the image circle.  load_camera_mask: a mask drawn by the user (the ego vehicle's body, a region known
to be wrong), an 8-bit single-channel PNG of the camera's size, non-zero = keep."""
from __future__ import annotations

import math
from pathlib import Path

import numpy as np
import torch

from ..ray_batch import Camera


def fisheye_fov_mask(camera: Camera, max_angle_deg: float, device="cuda") -> torch.Tensor:
    """[H, W] bool: True where the pixel's ray (pnr_generate_rays with the identity pose) makes an angle of at most
    max_angle_deg with the camera's +z axis, tested in float64 as z / |d| >= cos(max_angle_deg).  Works for both
    camera models; a fisheye ray past the mirror's field of view (clamped by the lift) lies on the far side."""
    if not 0.0 < float(max_angle_deg) <= 180.0:
        raise ValueError(f"fisheye_fov_mask: max_angle_deg={max_angle_deg} outside (0, 180]")
    from ...networks.renderer.panopticnerf_renderer import generate_rays
    eye = torch.tensor([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], dtype=torch.float32)
    d = generate_rays(camera.H, camera.W, camera.intr, eye, camera.model, device=device)[:, 3:].double()
    cos = d[:, 2] / d.norm(dim=1)
    return (cos >= math.cos(math.radians(float(max_angle_deg)))).reshape(camera.H, camera.W)


def load_camera_mask(path, camera: Camera) -> torch.Tensor:
    """[H, W] u8 (non-zero = keep) from an 8-bit single-channel PNG of the camera's size; anything else is refused."""
    import cv2
    path = Path(path)
    img = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(f"load_camera_mask: {path}: missing or not an image")
    if img.dtype != np.uint8:
        raise ValueError(f"load_camera_mask: {path}: a camera mask must be 8-bit, got {img.dtype}")
    if img.ndim != 2:
        raise ValueError(f"load_camera_mask: {path}: a camera mask must have 1 channel, got {img.shape[2]}")
    if img.shape != (camera.H, camera.W):
        raise ValueError(f"load_camera_mask: {path}: the mask is {img.shape[1]} x {img.shape[0]}, its camera is "
                         f"{camera.W} x {camera.H}")
    return torch.from_numpy(np.ascontiguousarray(img))
