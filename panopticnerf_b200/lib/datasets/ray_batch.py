"""Training batches drawn on the device from frames kept there (DESIGN 3.4).

FrameSet: the images of a sequence, resident on the GPU as one flat pixel table (rgb8 [P,3] u8, optional label [P] i16
and depth [P] f32) with per-frame poses, cameras and pixel offsets: what `pnr_sample_ray_batch` reads.
`kitti360.load_frames` builds one from a KITTI-360 sequence; `concat_frame_sets` joins sets of different cameras.

RaySampler(frames, seed).batch(step, R, N, Ni): one launch of `pnr_sample_ray_batch` -> the dict NetworkWrapper /
DataParallelWrapper take (rays, rgb, u, u_fine, depth and pseudo_label when the set has them, plus the scene block given
at construction).  Every row is a function of (seed, step, ray index) alone, so every data-parallel rank that calls
batch(step, R, ...) with the same seed holds the same global batch, with no exchange.

pixel_weights(frames, ...) -> PixelWeights: a per-pixel integer weight table (camera masks, frame balance, class
balance), its exact prefix sums and total, built on the device; RaySampler(frames, seed, weights=...) then draws each
pixel with probability weight / total and every batch carries importance [R] = total / (nonzero * weight), whose mean
under the draw is 1."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ... import _capi

CAMERA_MODEL = {"pinhole": 0, "fisheye": 2}   # the equirect camera (1) has device-only rays: not a batch camera
MAX_SAMPLES_PER_RAY = 256                     # N + Ni, as render_train accepts


@dataclass
class Camera:
    """model 'pinhole' (intr fx, fy, cx, cy) or 'fisheye' (gamma1, gamma2, u0, v0, xi, k1, k2); H x W pixels."""
    model: str
    H: int
    W: int
    intr: Tuple[float, ...]

    def __post_init__(self):
        if self.model not in CAMERA_MODEL:
            raise ValueError(f"Camera: model {self.model!r}; a ray batch takes {sorted(CAMERA_MODEL)} cameras "
                             "(equirect rays are device-only)")
        want = 4 if self.model == "pinhole" else 7
        self.intr = tuple(float(x) for x in self.intr)
        if len(self.intr) != want:
            raise ValueError(f"Camera: a {self.model} camera takes {want} intrinsics, got {len(self.intr)}")
        if int(self.H) < 1 or int(self.W) < 1:
            raise ValueError(f"Camera: size {self.H} x {self.W}")
        self.H, self.W = int(self.H), int(self.W)


@dataclass
class FrameSet:
    """Device buffers of F frames.  Frame f: camera cameras[frame_cam[f]], pose c2w[f] (row-major 3x4 camera -> world),
    pixels [pix_offset[f], pix_offset[f+1]) of the flat tables, row-major over (v, u).  label: -1 = ignore; depth:
    metres, <= 0 = none.  names: one (camera name, frame id) per frame."""
    cameras: List[Camera]
    c2w: torch.Tensor          # [F, 12] f32
    frame_cam: torch.Tensor    # [F] i32
    pix_offset: torch.Tensor   # [F + 1] i64
    rgb8: torch.Tensor         # [P, 3] u8
    label: Optional[torch.Tensor] = None   # [P] i16
    depth: Optional[torch.Tensor] = None   # [P] f32
    names: List[Tuple[str, int]] = field(default_factory=list)

    @property
    def num_frames(self) -> int:
        return int(self.c2w.shape[0])

    @property
    def num_pixels(self) -> int:
        return int(self.rgb8.shape[0])

    @staticmethod
    def from_images(cameras: Sequence[Camera], frame_cam: Sequence[int], c2w, rgb8: Sequence[torch.Tensor],
                    label: Optional[Sequence[torch.Tensor]] = None, depth: Optional[Sequence[torch.Tensor]] = None,
                    names: Optional[Sequence[Tuple[str, int]]] = None, device="cuda") -> "FrameSet":
        """A set from per-frame images: rgb8[f] [H, W, 3] u8, label[f] [H, W] i16, depth[f] [H, W] f32 (each list None
        or one per frame), every image of its camera's size; c2w [F, 3, 4] or [F, 12]."""
        cams = list(cameras)
        if not 1 <= len(cams) <= _capi.RAY_BATCH_MAX_CAMERAS:
            raise ValueError(f"FrameSet: {len(cams)} cameras; a set holds 1..{_capi.RAY_BATCH_MAX_CAMERAS}")
        F = len(rgb8)
        fc = [int(c) for c in frame_cam]
        if F < 1 or len(fc) != F:
            raise ValueError(f"FrameSet: {F} images for {len(fc)} frame cameras")
        for k, name in ((label, "label"), (depth, "depth")):
            if k is not None and len(k) != F:
                raise ValueError(f"FrameSet: {len(k)} {name} images for {F} frames")
        off = [0]
        for f in range(F):
            if not 0 <= fc[f] < len(cams):
                raise ValueError(f"FrameSet: frame {f} has camera {fc[f]} outside [0, {len(cams)})")
            cam = cams[fc[f]]
            want = (cam.H, cam.W)
            checks = [("rgb", rgb8[f], want + (3,), torch.uint8)]
            if label is not None:
                checks.append(("label", label[f], want, torch.int16))
            if depth is not None:
                checks.append(("depth", depth[f], want, torch.float32))
            for what, t, shape, dt in checks:
                if tuple(t.shape) != shape or t.dtype != dt:
                    raise ValueError(f"FrameSet: frame {f} {what} is {tuple(t.shape)} {t.dtype}, its camera wants "
                                     f"{shape} {dt}")
            off.append(off[-1] + cam.H * cam.W)
        flat = lambda ts, *tail: torch.cat([t.reshape(-1, *tail) for t in ts]).to(device).contiguous()
        c2w = torch.as_tensor(c2w, dtype=torch.float32).reshape(F, -1)
        if c2w.shape[1] != 12:
            raise ValueError(f"FrameSet: c2w has {c2w.shape[1]} values per frame, expected 12 (3x4)")
        return FrameSet(cams, c2w.to(device).contiguous(), torch.tensor(fc, dtype=torch.int32, device=device),
                        torch.tensor(off, dtype=torch.int64, device=device), flat(rgb8, 3),
                        flat(label) if label is not None else None, flat(depth) if depth is not None else None,
                        list(names) if names is not None else [])


def concat_frame_sets(*sets: FrameSet) -> FrameSet:
    """One set of the frames of several (e.g. the perspective and the fisheye cameras of a sequence), in order.  Equal
    cameras are merged; a label or depth table that only some sets have is filled with -1 / 0 (none) for the others."""
    if not sets:
        raise ValueError("concat_frame_sets: no sets")
    cams: List[Camera] = []
    fcs, offs, base = [], [sets[0].pix_offset[:1]], 0
    for s in sets:
        remap = []
        for c in s.cameras:
            if c not in cams:
                cams.append(c)
            remap.append(cams.index(c))
        fcs.append(torch.tensor(remap, dtype=torch.int32, device=s.frame_cam.device)[s.frame_cam.long()])
        offs.append(s.pix_offset[1:] + base)
        base += s.num_pixels
    if len(cams) > _capi.RAY_BATCH_MAX_CAMERAS:
        raise ValueError(f"concat_frame_sets: {len(cams)} distinct cameras; a set holds at most "
                         f"{_capi.RAY_BATCH_MAX_CAMERAS}")

    def table(key, fill, dtype):
        if all(getattr(s, key) is None for s in sets):
            return None
        return torch.cat([getattr(s, key) if getattr(s, key) is not None else
                          torch.full((s.num_pixels,), fill, dtype=dtype, device=s.rgb8.device) for s in sets])
    return FrameSet(cams, torch.cat([s.c2w for s in sets]), torch.cat(fcs), torch.cat(offs),
                    torch.cat([s.rgb8 for s in sets]), table("label", -1, torch.int16),
                    table("depth", 0.0, torch.float32), [n for s in sets for n in s.names])


def fill_frame_store(a, frames: FrameSet, what: str) -> None:
    """Write the frame store of `frames` (frame_cam, pix_offset, F, P) and its camera table (cams, num_cameras) into
    the C arguments `a` of `what` (pnr_ray_batch_args or pnr_project_depth_args)."""
    a.frame_cam = _capi.ptr(frames.frame_cam, torch.int32, "frame_cam")
    a.pix_offset = _capi.ptr(frames.pix_offset, torch.int64, "pix_offset")
    a.F, a.P = frames.num_frames, frames.num_pixels
    if len(frames.cameras) > _capi.RAY_BATCH_MAX_CAMERAS:
        raise ValueError(f"{what}: {len(frames.cameras)} cameras > {_capi.RAY_BATCH_MAX_CAMERAS}")
    for k, cam in enumerate(frames.cameras):
        a.cams[k].model, a.cams[k].H, a.cams[k].W = CAMERA_MODEL[cam.model], cam.H, cam.W
        for i, x in enumerate(cam.intr):
            a.cams[k].intr[i] = x
    a.num_cameras = len(frames.cameras)


@dataclass
class PixelWeights:
    """The weight table of a frame set (pixel_weights): weight [P] u16 and its group sums cum [ceil(P/32)] u64
    (cum[g] = the sum of the weights of pixels 0 .. 32 (g+1) - 1) on the set's device; total (T) and nonzero (the
    count of non-zero weights) on the host, read once when the table is built."""
    weight: torch.Tensor
    cum: torch.Tensor
    total: int
    nonzero: int

    @staticmethod
    def from_weight(weight: torch.Tensor) -> "PixelWeights":
        """The prefix sums and totals of a given weight table [P] u16 (pnr_pixel_cdf; one host read of the totals)."""
        P = int(weight.numel())
        if weight.dtype != torch.uint16 or weight.dim() != 1 or P < 1:
            raise ValueError(f"PixelWeights: weight is {tuple(weight.shape)} {weight.dtype}, expected [P] torch.uint16")
        dev = weight.device
        weight = weight.contiguous()
        cum = torch.empty((P + 31) // 32, dtype=torch.uint64, device=dev)
        totals = torch.empty(2, dtype=torch.uint64, device=dev)
        L = _capi.lib()
        ws = torch.empty(max(int(L.pnr_pixel_cdf_workspace_bytes(P)), 16), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _capi.check(L.pnr_pixel_cdf(_capi.ptr(weight, torch.uint16, "weight"), P, _capi.ptr(cum), _capi.ptr(totals),
                                        _capi.ptr(ws), ws.numel(), _capi.stream_ptr()), "pnr_pixel_cdf")
        total, nonzero = (int(x) for x in totals.view(torch.int64).cpu().tolist())
        if total == 0:
            raise ValueError("pixel_weights: the weight table's total is 0 - every pixel is masked out or has a zero "
                             "factor")
        return PixelWeights(weight, cum, total, nonzero)


def label_counts(frames: FrameSet, num_classes: int) -> torch.Tensor:
    """pnr_label_counts of the set's label table: counts [num_classes + 1] u64 on its device, slot 0 = labels outside
    [0, num_classes) (-1 included), slot 1 + c = class c."""
    if frames.label is None:
        raise ValueError("label_counts: the frame set has no label table")
    counts = torch.empty(int(num_classes) + 1, dtype=torch.uint64, device=frames.label.device)
    with torch.cuda.device(frames.label.device):
        _capi.check(_capi.lib().pnr_label_counts(_capi.ptr(frames.label, torch.int16, "label"), frames.num_pixels,
                                                 int(num_classes), _capi.ptr(counts), _capi.stream_ptr()),
                    "pnr_label_counts")
    return counts


def pixel_weights(frames: FrameSet, camera_masks: Optional[Sequence[Optional[torch.Tensor]]] = None,
                  balance_frames: bool = False, class_alpha: float = 0.0, class_max_ratio: float = 16.0,
                  unlabelled: float = 1.0) -> PixelWeights:
    """The weight table of a frame set for weighted draws (pnr_pixel_weights, then pnr_pixel_cdf).
    camera_masks: one [H, W] bool / u8 tensor (non-zero = keep) or None per camera of the set.  balance_frames: frame
    factor mean_pixels / pixels_f, so every frame has the same expected share of rays whatever its camera's size.
    class_alpha > 0: class factor min(class_max_ratio, (n_max / n_c) ** class_alpha) from the label table's class
    histogram (a class with no pixels gets 0); `unlabelled` is the factor of the pixels whose label is outside the
    classes (-1).  The scale maps the largest product of factors to 65535.  Host arithmetic is float64, rounded to fp32
    once."""
    dev = frames.rgb8.device
    F, P = frames.num_frames, frames.num_pixels
    masks = list(camera_masks) if camera_masks is not None else [None] * len(frames.cameras)
    if len(masks) != len(frames.cameras):
        raise ValueError(f"pixel_weights: {len(masks)} camera masks for {len(frames.cameras)} cameras")
    for k, (m, cam) in enumerate(zip(masks, frames.cameras)):
        if m is not None and (tuple(m.shape) != (cam.H, cam.W) or m.dtype not in (torch.bool, torch.uint8)):
            raise ValueError(f"pixel_weights: the mask of camera {k} is {tuple(m.shape)} {m.dtype}, its camera wants "
                             f"({cam.H}, {cam.W}) bool or uint8")
    if not (class_alpha >= 0 and class_max_ratio > 0 and unlabelled >= 0):
        raise ValueError(f"pixel_weights: class_alpha={class_alpha}, class_max_ratio={class_max_ratio} and "
                         f"unlabelled={unlabelled} must be >= 0, > 0 and >= 0")
    if class_alpha > 0 and frames.label is None:
        raise ValueError("pixel_weights: class_alpha > 0 needs a label table, and the frame set has none")
    if frames.label is None and unlabelled == 0:
        raise ValueError("pixel_weights: the weight table's total is 0 - the set has no label table and unlabelled=0")

    ff = None
    if balance_frames:
        sizes = np.diff(frames.pix_offset.cpu().numpy()).astype(np.float64)
        ff = (P / F) / np.maximum(sizes, 1.0)
    ncls, cf = 0, np.array([float(unlabelled)], np.float64)
    if class_alpha > 0 or (frames.label is not None and unlabelled != 1.0):
        ncls = max(int(frames.label.max()) + 1, 0)
        cf = np.concatenate([cf, np.ones(ncls)])
        if class_alpha > 0 and ncls > 0:
            n = label_counts(frames, ncls).view(torch.int64).cpu().numpy()[1:].astype(np.float64)
            ratio = n.max() / np.maximum(n, 1.0)
            cf[1:] = np.where(n > 0, np.minimum(class_max_ratio, ratio ** class_alpha), 0.0)
    top = (ff.max() if ff is not None else 1.0) * cf.max()
    if not top > 0:
        raise ValueError("pixel_weights: the weight table's total is 0 - every factor is 0")
    a = _capi.PnrPixelWeightsArgs()
    fill_frame_store(a, frames, "pixel_weights")
    keep = [m.to(device=dev, dtype=torch.uint8).contiguous() if m is not None else None for m in masks]
    for k, m in enumerate(keep):
        a.mask[k] = _capi.ptr(m)
    a.scale = float(np.float32(65535.0 / top))
    f32 = lambda x: torch.from_numpy(x.astype(np.float32)).to(dev)
    ff_t = f32(ff) if ff is not None else None
    cf_t = f32(cf) if ncls > 0 or unlabelled != 1.0 else None
    a.label = _capi.ptr(frames.label, torch.int16, "label") if ncls > 0 else None
    a.C = ncls
    a.frame_factor, a.class_factor = _capi.ptr(ff_t), _capi.ptr(cf_t)
    weight = torch.empty(P, dtype=torch.uint16, device=dev)
    a.weight = _capi.ptr(weight)
    with torch.cuda.device(dev):
        _capi.check(_capi.lib().pnr_pixel_weights(C.byref(a), _capi.stream_ptr()), "pnr_pixel_weights")
    return PixelWeights.from_weight(weight)


def sample_ray_batch(frames: FrameSet, seed: int, step: int, r0: int, r1: int, N: int, Ni: int = 0,
                     want_pixel: bool = False, want_frame: bool = False,
                     weights: Optional[PixelWeights] = None) -> Dict[str, torch.Tensor]:
    """Rays r0 .. r1-1 of the batch (seed, step): one pnr_sample_ray_batch launch on the frames' device.  Returns
    rays [n,6], rgb [n,3], u [n,N], u_fine [n,Ni] (Ni > 0), depth [n] / pseudo_label [n] i32 when the set has a depth /
    label table, pixel [n] i64 (the flat pixel index) and frame [n] i32 (the frame of the pixel) when asked.  With
    `weights` (pixel_weights) each pixel is drawn with probability weight / total, and importance [n] f32 is returned
    too."""
    if not (0 <= int(seed) < 1 << 64 and 0 <= int(step) < 1 << 64):
        raise ValueError(f"sample_ray_batch: seed {seed} and step {step} must be in [0, 2^64)")
    if weights is not None and tuple(weights.weight.shape) != (frames.num_pixels,):
        raise ValueError(f"sample_ray_batch: the weight table has {tuple(weights.weight.shape)} entries, the frame set "
                         f"{frames.num_pixels} pixels")
    dev = frames.rgb8.device
    n = int(r1) - int(r0)
    e = lambda *shape, dtype=torch.float32: torch.empty(*shape, dtype=dtype, device=dev)
    out = {"rays": e(max(n, 0), 6), "rgb": e(max(n, 0), 3), "u": e(max(n, 0), int(N))}
    if int(Ni) > 0:
        out["u_fine"] = e(max(n, 0), int(Ni))
    if frames.depth is not None:
        out["depth"] = e(max(n, 0))
    if frames.label is not None:
        out["pseudo_label"] = e(max(n, 0), dtype=torch.int32)
    if want_pixel:
        out["pixel"] = e(max(n, 0), dtype=torch.int64)
    if want_frame:
        out["frame"] = e(max(n, 0), dtype=torch.int32)
    if weights is not None:
        out["importance"] = e(max(n, 0))
    a = _capi.PnrRayBatchArgs()
    a.c2w = _capi.ptr(frames.c2w, torch.float32, "c2w")
    fill_frame_store(a, frames, "sample_ray_batch")
    a.rgb8 = _capi.ptr(frames.rgb8, torch.uint8, "rgb8")
    a.label = _capi.ptr(frames.label, torch.int16, "label")
    a.depth = _capi.ptr(frames.depth, torch.float32, "depth")
    a.seed, a.step, a.r0, a.r1, a.N, a.Ni = int(seed), int(step), int(r0), int(r1), int(N), int(Ni)
    a.rays, a.rgb, a.u = _capi.ptr(out["rays"]), _capi.ptr(out["rgb"]), _capi.ptr(out["u"])
    a.u_fine = _capi.ptr(out.get("u_fine"))
    a.depth_out, a.pseudo_label = _capi.ptr(out.get("depth")), _capi.ptr(out.get("pseudo_label"))
    a.pixel, a.frame = _capi.ptr(out.get("pixel")), _capi.ptr(out.get("frame"))
    if weights is None:
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().pnr_sample_ray_batch(C.byref(a), _capi.stream_ptr()), "pnr_sample_ray_batch")
        return out
    w = _capi.PnrRayBatchWeights(_capi.ptr(weights.weight, torch.uint16, "weight"),
                                 _capi.ptr(weights.cum, torch.uint64, "cum"), int(weights.total), int(weights.nonzero),
                                 _capi.ptr(out["importance"]))
    with torch.cuda.device(dev):
        _capi.check(_capi.lib().pnr_sample_ray_batch_weighted(C.byref(a), C.byref(w), _capi.stream_ptr()),
                    "pnr_sample_ray_batch_weighted")
    return out


class RaySampler:
    """RaySampler(frames, seed, scene).batch(step, R, N, Ni) -> a training batch of R random pixels of the frame set.
    `scene`: the replicated block every batch carries (the primitive table of `kitti360.primitive_batch`, a mesh
    table, scene_aabb, ...).  With a sequence table (`kitti360.sequence_primitives` with frame_ids = [fid for _, fid in
    frames.names], so that frame_boxes has one row per frame of the set) each batch also carries ray_frame [R] i32,
    the frame of each ray, and every ray meets the static primitives and its own frame's dynamic ones, as a render of
    that frame does.  Without frame_boxes the table serves every frame as it is (e.g. the static annotations,
    boxes_to_primitives(frame=None)).  With `weights` (pixel_weights of this set) pixels are drawn by weight and each
    batch also carries importance [R] f32."""

    def __init__(self, frames: FrameSet, seed: int, scene: Optional[Dict[str, torch.Tensor]] = None,
                 weights: Optional[PixelWeights] = None):
        self.frames, self.seed, self.weights = frames, int(seed), weights
        if weights is not None and tuple(weights.weight.shape) != (frames.num_pixels,):
            raise ValueError(f"RaySampler: the weight table has {tuple(weights.weight.shape)} entries, the frame set "
                             f"{frames.num_pixels} pixels")
        self.scene = dict(scene or {})
        clash = set(self.scene) & {"rays", "rgb", "u", "u_fine", "depth", "pseudo_label", "ray_frame", "importance"}
        if clash:
            raise ValueError(f"RaySampler: the scene block may not carry the per-ray keys {sorted(clash)}")
        fb = self.scene.get("frame_boxes")
        if fb is not None and tuple(fb.shape) != (frames.num_frames, 2):
            raise ValueError(f"RaySampler: frame_boxes {tuple(fb.shape)} needs one (begin, end) row per frame of the "
                             f"set, ({frames.num_frames}, 2)")

    def batch(self, step: int, R: int, N: int, Ni: int = 0) -> Dict[str, torch.Tensor]:
        """The global batch of `step`: rays 0 .. R-1, identical on every rank that uses the same seed."""
        seq = "frame_boxes" in self.scene
        out = sample_ray_batch(self.frames, self.seed, step, 0, R, N, Ni, want_frame=seq, weights=self.weights)
        if seq:
            out["ray_frame"] = out.pop("frame")
        out.update(self.scene)
        return out


__all__ = ["Camera", "FrameSet", "concat_frame_sets", "sample_ray_batch", "RaySampler", "PixelWeights",
           "pixel_weights", "label_counts"]
