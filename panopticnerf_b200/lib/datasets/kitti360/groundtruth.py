"""KITTI-360 2D ground-truth images for evaluation: `instance/*.png` (16-bit, semanticId*1000 + instanceId, the
panoptic encoding pnr_panoptic_fuse writes; instanceId 0 on a thing class = a crowd region) and `semantic/*.png`
(8-bit semanticId).  Both come back as int32 [H, W] panoptic ids on the CPU; move them to the device for the evaluator.
Anything else - another bit depth, several channels, a missing file - is refused."""
from __future__ import annotations

import numpy as np
import torch


def _read(path, dtype, what: str) -> np.ndarray:
    import cv2
    img = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(f"{path}: not a readable image ({what})")
    if img.ndim != 2:
        raise ValueError(f"{path}: {what} must be a single-channel image, got shape {img.shape}")
    if img.dtype != dtype:
        raise ValueError(f"{path}: {what} must be {np.dtype(dtype).itemsize * 8}-bit, got {img.dtype}")
    return img


def load_panoptic_gt(path) -> torch.Tensor:
    """KITTI-360 `instance/*.png` (uint16) -> int32 [H, W] = semanticId*1000 + instanceId."""
    return torch.from_numpy(_read(path, np.uint16, "a KITTI-360 instance image").astype(np.int32))


def load_semantic_gt(path) -> torch.Tensor:
    """KITTI-360 `semantic/*.png` (uint8) -> int32 [H, W] = semanticId*1000 (no instances)."""
    return torch.from_numpy(_read(path, np.uint8, "a KITTI-360 semantic image").astype(np.int32) * 1000)
