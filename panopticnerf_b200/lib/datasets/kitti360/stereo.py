"""KITTI-360's rectified stereo pair -> the depth table of a FrameSet, by semi-global matching on the device
(`pnr_stereo_depth`, include/pnr.h, DESIGN 3.4).

Layout under `root` (public KITTI-360 layout):
  data_2d_raw/<seq>/image_00/data_rect/<frame:010d>.png   left, 8-bit colour (the frame store's image_00 frames)
  data_2d_raw/<seq>/image_01/data_rect/<frame:010d>.png   right, 8-bit colour, the same size
  calibration/perspective.txt                             P_rect_00 / S_rect_00 and P_rect_01 / S_rect_01
Rules (chosen here; the reference's stereo preprocessing is not public): census 9 x 7 over an integer grey, eight-path
SGM with penalties P1 / P2, winner with a uniqueness margin U (per cent) and a left-right check, subpixel in sixteenths,
depth t = 16 fx b / d16 (z in rectified camera 0, the units of the pinhole's rays), kept inside (min_depth, max_depth].
The defaults (D = 128, P1 = 10, P2 = 120, U = 10, 0.1 .. 40 m) are chosen, not tuned: the depth error of one
sixteenth of a pixel grows as z^2 / (16 fx b), about 0.3 m at 40 m for KITTI-360's fx b of
552.55 px x 0.6 m.
`lidar.save_depth_png` caches the result for `load_frames(depth_dir=...)`."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import torch

from .... import _capi
from ..ray_batch import FrameSet
from .calib import load_perspective
from .frames import check_depth_range, check_names, ensure_depth

DEFAULT_DISPARITIES = 128
DEFAULT_P1 = 10
DEFAULT_P2 = 120
DEFAULT_UNIQUENESS = 10
DEFAULT_MIN_DEPTH = 0.1          # metres
DEFAULT_MAX_DEPTH = 40.0         # metres
STEREO_OPTIONS = ("num_disparities", "P1", "P2", "uniqueness", "min_depth", "max_depth", "chunk_frames")


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool)


def _check_sgm(what, num_disparities, P1, P2, uniqueness):
    if not _is_int(num_disparities) or num_disparities % 32 or not 32 <= num_disparities <= 256:
        raise ValueError(f"{what}: num_disparities={num_disparities}; one of 32, 64, .., 256")
    if not (_is_int(P1) and _is_int(P2) and 0 <= P1 <= P2 <= 2048):
        raise ValueError(f"{what}: P1={P1}, P2={P2}; integers with 0 <= P1 <= P2 <= 2048")
    if not _is_int(uniqueness) or not 0 <= uniqueness <= 99:
        raise ValueError(f"{what}: uniqueness={uniqueness}; an integer in [0, 99]")


def stereo_call(rgb8, pix_offset, frames, right, num_disparities, P1, P2, uniqueness, B16=1.0,
                min_depth=DEFAULT_MIN_DEPTH, max_depth=DEFAULT_MAX_DEPTH, depth=None, disparity=None) -> None:
    """One `pnr_stereo_depth` call: rgb8 [P, 3] u8 and pix_offset [F+1] i64 (a frame store, device), frames a host
    list of n store frames, right [n, H, W, 3] u8 (device); writes depth [P] f32 (the frames' rows) and / or
    disparity [n, H, W] i16."""
    if right.dim() != 4 or right.shape[3] != 3:
        raise ValueError(f"stereo: right images {tuple(right.shape)}; expected [n, H, W, 3]")
    fr = np.ascontiguousarray(frames, dtype=np.int32)
    n, H, W = int(right.shape[0]), int(right.shape[1]), int(right.shape[2])
    if fr.shape != (n,):
        raise ValueError(f"stereo: {fr.size} frames for {n} right images")
    a = _capi.PnrStereoArgs()
    a.rgb8 = _capi.ptr(rgb8, torch.uint8, "rgb8")
    a.pix_offset = _capi.ptr(pix_offset, torch.int64, "pix_offset")
    a.P, a.F = int(rgb8.shape[0]), int(pix_offset.shape[0]) - 1
    a.frames, a.n, a.H, a.W = fr.ctypes.data, n, H, W
    a.right = _capi.ptr(right, torch.uint8, "right")
    a.D, a.P1, a.P2, a.U = int(num_disparities), int(P1), int(P2), int(uniqueness)
    a.B16, a.min_depth, a.max_depth = float(B16), float(min_depth), float(max_depth)
    a.depth = _capi.ptr(depth, torch.float32, "depth")
    a.disparity = _capi.ptr(disparity, torch.int16, "disparity")
    need = int(_capi.lib().pnr_stereo_workspace_bytes(n, H, W, a.D))
    ws = torch.empty(max(need, 16), dtype=torch.uint8, device=right.device)   # freed in stream order
    a.workspace, a.workspace_bytes = ws.data_ptr(), need
    with torch.cuda.device(right.device):
        _capi.check(_capi.lib().pnr_stereo_depth(C.byref(a), _capi.stream_ptr()), "pnr_stereo_depth")


def stereo_disparity(left: torch.Tensor, right: torch.Tensor, num_disparities: int = DEFAULT_DISPARITIES,
                     P1: int = DEFAULT_P1, P2: int = DEFAULT_P2, uniqueness: int = DEFAULT_UNIQUENESS) -> torch.Tensor:
    """Rectified pairs left / right [n, H, W, 3] u8 RGB (CUDA) -> disparity [n, H, W] i16 in sixteenths of a pixel,
    -1 where the match is refused (uniqueness or left-right check)."""
    _check_sgm("stereo_disparity", num_disparities, P1, P2, uniqueness)
    if left.shape != right.shape or left.dim() != 4 or left.shape[3] != 3:
        raise ValueError(f"stereo_disparity: left {tuple(left.shape)} and right {tuple(right.shape)}; expected "
                         "two [n, H, W, 3] tensors")
    n, H, W = int(left.shape[0]), int(left.shape[1]), int(left.shape[2])
    left = left.contiguous()
    off = torch.arange(n + 1, dtype=torch.int64, device=left.device) * (H * W)
    out = torch.empty((n, H, W), dtype=torch.int16, device=left.device)
    stereo_call(left.view(-1, 3), off, list(range(n)), right.contiguous(), num_disparities, P1, P2, uniqueness,
                disparity=out)
    return out


def stereo_baseline(root):
    """(B16, K, size) from calibration/perspective.txt: B16 = fp32(16 (P_rect_00[0,3] - P_rect_01[0,3])) = 16 fx b,
    composed in float64 and rounded once; refused by name unless P_rect_01 has P_rect_00's K and B16 is finite and
    > 0."""
    path = Path(root) / "calibration" / "perspective.txt"
    p0, p1 = load_perspective(path, 0), load_perspective(path, 1)
    if not np.array_equal(p0["K"], p1["K"]):
        raise ValueError(f"{path}: P_rect_01's K {p1['K'].tolist()} is not P_rect_00's {p0['K'].tolist()}; the pair "
                         "is not rectified to one camera")
    b16 = 16.0 * (float(p0["P_rect"][0, 3]) - float(p1["P_rect"][0, 3]))
    with np.errstate(over="ignore"):
        b32 = np.float32(b16)
    if not (np.isfinite(b32) and b32 > 0):
        raise ValueError(f"{path}: 16 fx b = 16 (P_rect_00[0,3] - P_rect_01[0,3]) = {b16}; finite and > 0")
    return float(b32), p0["K"], p1["size"]


def stereo_depth(frames: FrameSet, root, seq: str, num_disparities: int = DEFAULT_DISPARITIES, P1: int = DEFAULT_P1,
                 P2: int = DEFAULT_P2, uniqueness: int = DEFAULT_UNIQUENESS, min_depth: float = DEFAULT_MIN_DEPTH,
                 max_depth: float = DEFAULT_MAX_DEPTH, chunk_frames: int = 8) -> FrameSet:
    """Fill frames.depth (allocated, zero, when the set has none) for every image_00 frame of the set from the
    stereo pair (module docstring: layout and rules).  The frames are identified by frames.names (camera, frame id);
    frames of other cameras are left as they are.  chunk_frames right images go to the device per call.  Returns
    `frames`."""
    import cv2
    _check_sgm("stereo_depth", num_disparities, P1, P2, uniqueness)
    check_depth_range("stereo_depth", min_depth, max_depth)
    if not _is_int(chunk_frames) or chunk_frames < 1:
        raise ValueError(f"stereo_depth: chunk_frames={chunk_frames}; an integer >= 1")
    check_names(frames, "stereo_depth")
    left = [(f, int(fid)) for f, (cam, fid) in enumerate(frames.names) if cam == "image_00"]
    if not left:
        raise ValueError("stereo_depth: the set has no image_00 frames; stereo depth comes from the image_00 / "
                         "image_01 pair")
    root = Path(root)
    b16, _, size = stereo_baseline(root)
    fc = frames.frame_cam.cpu().numpy()
    H, W = None, None
    for f, fid in left:
        cam = frames.cameras[int(fc[f])]
        if cam.model != "pinhole" or (H is not None and (cam.H, cam.W) != (H, W)):
            raise ValueError(f"stereo_depth: frame ('image_00', {fid}) has a {cam.model} camera of {cam.W} x {cam.H}; "
                             "the image_00 frames must share one pinhole camera")
        H, W = cam.H, cam.W
    if size is not None and tuple(size) != (W, H):
        raise ValueError(f"{root / 'calibration' / 'perspective.txt'}: S_rect_01 is {size[0]} x {size[1]}, image_00 "
                         f"is {W} x {H}")
    images = root / "data_2d_raw" / seq / "image_01" / "data_rect"
    dev = frames.rgb8.device
    paths = [images / f"{fid:010d}.png" for _, fid in left]
    for (_, fid), p in zip(left, paths):   # all present before anything is written
        if not p.is_file():
            raise FileNotFoundError(f"{p}: missing right image (image_01) of frame {fid}")
    ensure_depth(frames)
    for c0 in range(0, len(left), int(chunk_frames)):
        chunk = range(c0, min(len(left), c0 + int(chunk_frames)))
        rgb = []
        for k in chunk:
            img = cv2.imread(str(paths[k]), cv2.IMREAD_UNCHANGED)
            if img is None or img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8:
                raise ValueError(f"{paths[k]}: the right image must be an 8-bit colour image")
            if img.shape[:2] != (H, W):
                raise ValueError(f"{paths[k]}: the right image is {img.shape[1]} x {img.shape[0]}, image_00 is "
                                 f"{W} x {H}")
            rgb.append(np.ascontiguousarray(img[:, :, ::-1]))
        stereo_call(frames.rgb8, frames.pix_offset, [left[k][0] for k in chunk], torch.from_numpy(np.stack(rgb)).to(dev),
                    num_disparities, P1, P2, uniqueness, b16, min_depth, max_depth, depth=frames.depth)
    return frames


__all__ = ["stereo_disparity", "stereo_depth", "stereo_baseline", "stereo_call", "STEREO_OPTIONS"]
