"""ctypes binding of the libpnr C ABI (include/pnr.h).  Thin by design: it only checks dtype /
device / contiguity and forwards ``tensor.data_ptr()`` plus the current CUDA stream handle.

There is no CPU or PyTorch fallback: if libpnr.so is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

import torch

# PNR_LIB: load a development variant of the library (a build with extra flags, _build.build(out=...))
_LIB_PATH = Path(os.environ.get("PNR_LIB") or Path(__file__).resolve().parent / "libpnr.so")
_lib: Optional[C.CDLL] = None

PREC = {"bf16x3": 0, "bf16": 1, "fp16x3": 2, "fp16": 3}


class PnrError(RuntimeError):
    pass


class PnrConfig(C.Structure):
    """pnr_config of include/pnr.h.  Fields left out of a positional call stay zero: the frequency network."""
    _fields_ = [("D", C.c_int32), ("W", C.c_int32), ("xyz_res", C.c_int32), ("view_res", C.c_int32),
                ("num_classes", C.c_int32), ("num_instances", C.c_int32), ("precision", C.c_int32),
                ("device", C.c_int32), ("xyz_encoding", C.c_int32), ("hash_levels", C.c_int32),
                ("hash_features", C.c_int32), ("hash_log2_size", C.c_int32), ("hash_base_resolution", C.c_float),
                ("hash_per_level_scale", C.c_float), ("hash_aabb", C.c_float * 6)]


XYZ_ENCODING = {"frequency": 0, "hashgrid": 1}


class PnrCompositeOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in
                ("rgb_map", "depth_map", "acc_map", "disp_map", "weights", "semantic_map",
                 "instance_map", "fixed_semantic_map", "fixed_instance_map")]


class PnrLossArgs(C.Structure):
    _fields_ = [("R", C.c_int64), ("C", C.c_int32), ("sem_is_prob", C.c_int32)] + \
               [(k, C.c_void_p) for k in ("rgb_map", "rgb_map0", "rgb_gt", "depth_map", "depth_gt", "semantic_map",
                                          "fixed_semantic_map", "label", "label_weight")] + \
               [(k, C.c_float) for k in ("w_rgb", "w_depth", "w_sem", "w_fix", "inv_n_rgb", "inv_n_depth", "inv_n_sem", "eps")] + \
               [(k, C.c_void_p) for k in ("per_ray", "d_rgb_map", "d_rgb_map0", "d_depth_map", "d_semantic_map",
                                          "d_fixed_semantic_map")] + \
               [("K", C.c_int32), ("instance_map", C.c_void_p), ("fixed_instance_map", C.c_void_p),
                ("w_inst", C.c_float), ("inst_min_weight", C.c_float)] + \
               [(k, C.c_void_p) for k in ("per_ray_inst", "inst_label", "n_inst", "d_instance_map")]


class PnrCompositeGrads(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in
                ("rgb_map", "depth_map", "acc_map", "weights", "semantic_map",
                 "instance_map", "fixed_semantic_map", "fixed_instance_map")]


class PnrRenderArgs(C.Structure):
    """pnr_render_args of include/pnr.h (same field order)."""
    _fields_ = [("rays", C.c_void_p), ("R", C.c_int64), ("near", C.c_void_p), ("far", C.c_void_p),
                ("aabb_host", C.POINTER(C.c_float)), ("near_min", C.c_float), ("far_default", C.c_float),
                ("box_center", C.c_void_p), ("box_half", C.c_void_p), ("box_rot", C.c_void_p),
                ("box_sem", C.c_void_p), ("box_inst", C.c_void_p), ("B", C.c_int32), ("M", C.c_int32),
                ("N", C.c_int32), ("Ni", C.c_int32), ("t_vals", C.c_void_p), ("u", C.c_void_p),
                ("perturb", C.c_float), ("u_fine", C.c_void_p), ("u_fine_stride", C.c_int64),
                ("sample_mode", C.c_int32), ("white_bkgd", C.c_int32), ("sem_softmax", C.c_int32),
                ("mask_outside", C.c_int32), ("bound_by_primitives", C.c_int32),
                ("out", PnrCompositeOut), ("out0", PnrCompositeOut), ("z_vals", C.c_void_p), ("z_vals0", C.c_void_p),
                ("hit_mask", C.c_void_p), ("box_id", C.c_void_p), ("t_in", C.c_void_p), ("t_out", C.c_void_p),
                ("sample_box", C.c_void_p), ("near_out", C.c_void_p), ("far_out", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
                ("mesh_tri_start", C.c_void_p), ("mesh_tris", C.c_void_p), ("T", C.c_int64)]


class PnrFrameTable(C.Structure):
    """pnr_frame_table of include/pnr.h: the frame fields of a sequence table (all zero: none)."""
    _fields_ = [("ray_frame", C.c_void_p), ("frame_boxes", C.c_void_p), ("F", C.c_int32), ("S", C.c_int32)]


class PnrIntersectFramesArgs(C.Structure):
    """pnr_intersect_frames_args of include/pnr.h (same field order)."""
    _fields_ = [("rays", C.c_void_p), ("R", C.c_int64), ("box_center", C.c_void_p), ("box_half", C.c_void_p),
                ("box_rot", C.c_void_p), ("B", C.c_int32), ("M", C.c_int32), ("mesh_tri_start", C.c_void_p),
                ("mesh_tris", C.c_void_p), ("T", C.c_int64), ("frames", PnrFrameTable), ("hit_mask", C.c_void_p),
                ("box_id", C.c_void_p), ("t_in", C.c_void_p), ("t_out", C.c_void_p)]


class PnrAdamArgs(C.Structure):
    """pnr_adam_args of include/pnr.h."""
    _fields_ = [("P", C.c_int64), ("ld_grad", C.c_int64), ("G", C.c_int32), ("beta1", C.c_double),
                ("beta2", C.c_double), ("eps", C.c_float), ("weight_decay", C.c_float), ("step_size", C.c_float),
                ("bc2_sqrt", C.c_float)]


RAY_BATCH_MAX_CAMERAS = 4


class PnrRayCamera(C.Structure):
    """pnr_ray_camera of include/pnr.h."""
    _fields_ = [("model", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("intr", C.c_float * 7)]


class PnrRayBatchArgs(C.Structure):
    """pnr_ray_batch_args of include/pnr.h (same field order)."""
    _fields_ = [("c2w", C.c_void_p), ("frame_cam", C.c_void_p), ("pix_offset", C.c_void_p), ("F", C.c_int32),
                ("P", C.c_int64), ("rgb8", C.c_void_p), ("label", C.c_void_p), ("depth", C.c_void_p),
                ("cams", PnrRayCamera * RAY_BATCH_MAX_CAMERAS), ("num_cameras", C.c_int32),
                ("seed", C.c_uint64), ("step", C.c_uint64), ("r0", C.c_int64), ("r1", C.c_int64),
                ("N", C.c_int32), ("Ni", C.c_int32)] + \
               [(k, C.c_void_p) for k in ("rays", "rgb", "depth_out", "pseudo_label", "u", "u_fine", "pixel", "frame")]


class PnrRayBatchWeights(C.Structure):
    """pnr_ray_batch_weights of include/pnr.h (same field order)."""
    _fields_ = [("weight", C.c_void_p), ("weight_cum", C.c_void_p), ("weight_total", C.c_uint64),
                ("weight_nonzero", C.c_int64), ("importance", C.c_void_p)]


class PnrPixelWeightsArgs(C.Structure):
    """pnr_pixel_weights_args of include/pnr.h (same field order)."""
    _fields_ = [("frame_cam", C.c_void_p), ("pix_offset", C.c_void_p), ("F", C.c_int32), ("P", C.c_int64),
                ("cams", PnrRayCamera * RAY_BATCH_MAX_CAMERAS), ("num_cameras", C.c_int32), ("label", C.c_void_p),
                ("C", C.c_int32), ("frame_factor", C.c_void_p), ("class_factor", C.c_void_p),
                ("mask", C.c_void_p * RAY_BATCH_MAX_CAMERAS), ("scale", C.c_float), ("weight", C.c_void_p)]


class PnrProjectDepthArgs(C.Structure):
    """pnr_project_depth_args of include/pnr.h (same field order); scan_offset and the pair tables are host pointers."""
    _fields_ = [("points", C.c_void_p), ("Npts", C.c_int64), ("scan_offset", C.c_void_p), ("S", C.c_int32),
                ("pair_frame", C.c_void_p), ("pair_scan", C.c_void_p), ("pair_M", C.c_void_p), ("Q", C.c_int32),
                ("frame_cam", C.c_void_p), ("pix_offset", C.c_void_p), ("F", C.c_int32), ("P", C.c_int64),
                ("cams", PnrRayCamera * RAY_BATCH_MAX_CAMERAS), ("num_cameras", C.c_int32),
                ("min_depth", C.c_float), ("max_depth", C.c_float), ("occlusion_radius", C.c_int32),
                ("occlusion_margin", C.c_float), ("depth", C.c_void_p), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t)]


class PnrStereoArgs(C.Structure):
    """pnr_stereo_args of include/pnr.h (same field order); frames is a host pointer."""
    _fields_ = [("rgb8", C.c_void_p), ("pix_offset", C.c_void_p), ("P", C.c_int64), ("F", C.c_int32),
                ("frames", C.c_void_p), ("n", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("right", C.c_void_p),
                ("D", C.c_int32), ("P1", C.c_int32), ("P2", C.c_int32), ("U", C.c_int32), ("B16", C.c_float),
                ("min_depth", C.c_float), ("max_depth", C.c_float), ("depth", C.c_void_p), ("disparity", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


SAMPLE_MODE = {"uniform": 0, "intervals": 1}
COMM_ID_BYTES = 128

# name -> (restype, argtypes); mirrors include/pnr.h one to one
_vp, _i32, _i64, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
SIGNATURES = {
    "pnr_version": (C.c_int, []),
    "pnr_last_error": (C.c_char_p, []),
    "pnr_create": (C.c_int, [C.POINTER(PnrConfig), C.POINTER(_vp)]),
    "pnr_destroy": (C.c_int, [_vp]),
    "pnr_status": (C.c_int, [_vp, C.POINTER(C.c_uint32), _i32, _vp]),
    "pnr_bind_hashgrid_table": (C.c_int, [_vp, _vp]),
    "pnr_set_mlp_rows": (C.c_int, [_vp, _i32]),
    "pnr_program_tile_rows": (C.c_int, [_vp, C.c_size_t, C.POINTER(_i32)]),
    "pnr_load_weights": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32]),
    "pnr_intersect": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "pnr_intersect_meshes": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "pnr_intersect_frames": (C.c_int, [C.POINTER(PnrIntersectFramesArgs), _vp]),
    "pnr_scene_near_far": (C.c_int, [_vp, _i64, C.POINTER(_f32), _f32, _f32, _vp, _vp, _vp]),
    "pnr_bound_by_primitives": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "pnr_sample_stratified": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _f32, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "pnr_sample_intervals": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _f32, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "pnr_tag_samples": (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _vp]),
    "pnr_generate_rays": (C.c_int, [_i32, _i32, _i32, _i32, _i32, C.POINTER(_f32), C.POINTER(_f32), _vp, _vp]),
    "pnr_sample_ray_batch": (C.c_int, [C.POINTER(PnrRayBatchArgs), _vp]),
    "pnr_sample_ray_batch_weighted": (C.c_int, [C.POINTER(PnrRayBatchArgs), C.POINTER(PnrRayBatchWeights), _vp]),
    "pnr_pixel_weights": (C.c_int, [C.POINTER(PnrPixelWeightsArgs), _vp]),
    "pnr_label_counts": (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    "pnr_pixel_cdf_workspace_bytes": (C.c_size_t, [_i64]),
    "pnr_pixel_cdf": (C.c_int, [_vp, _i64, _vp, _vp, _vp, C.c_size_t, _vp]),
    "pnr_project_depth_workspace_bytes": (C.c_size_t, [_i64, _i32]),
    "pnr_project_depth": (C.c_int, [C.POINTER(PnrProjectDepthArgs), _vp]),
    "pnr_stereo_workspace_bytes": (C.c_size_t, [_i32, _i32, _i32, _i32]),
    "pnr_stereo_depth": (C.c_int, [C.POINTER(PnrStereoArgs), _vp]),
    "pnr_encode": (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    "pnr_mlp_forward": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp]),
    "pnr_mlp_composite": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _i32,
                                    C.POINTER(PnrCompositeOut), _vp]),
    "pnr_mlp_backward_trunk": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, C.c_float, _vp, _i32, _vp, _vp, _vp]),
    "pnr_mlp_trunk_forward": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp]),
    "pnr_composite": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i32,
                                C.POINTER(PnrCompositeOut), _vp]),
    "pnr_losses": (C.c_int, [C.POINTER(PnrLossArgs), _vp]),
    "pnr_panoptic_fuse": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pnr_hashgrid_encode": (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, C.c_float, C.c_float, _vp, _vp]),
    "pnr_hashgrid_backward": (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, C.c_float, C.c_float, _vp, _vp]),
    "pnr_hashgrid_fixed_workspace_bytes": (C.c_size_t, [_i32, _i32, _i32]),
    "pnr_hashgrid_backward_fixed": (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, C.c_float, C.c_float, _vp, _vp,
                                              C.c_size_t, _vp]),
    "pnr_label_tiles": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "pnr_composite_backward": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp,
                                         _i32, C.POINTER(PnrCompositeGrads), _vp, _vp]),
    "pnr_wgrad_workspace_bytes": (C.c_size_t, [_i32, _i32]),
    "pnr_wgrad": (C.c_int, [_vp, _i64, _i32, _vp, _i64, _i32, _i64, _i32, _vp, _vp, _i64, _vp, _i32, _vp, C.c_size_t, _vp]),
    "pnr_linear_workspace_bytes": (C.c_size_t, [_i32, _i32]),
    "pnr_linear": (C.c_int, [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _i32, _i64, _i32, _i32, _vp, _vp, _i64, _vp, C.c_size_t, _vp]),
    "pnr_sample_pdf": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "pnr_update_weights": (C.c_int, [_vp, C.POINTER(_vp), _i32, _vp]),
    "pnr_program_host": (C.c_int, [C.POINTER(PnrConfig), C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, C.c_size_t,
                                   C.POINTER(C.c_size_t), _vp, C.c_size_t, C.POINTER(C.c_size_t), _vp, C.c_size_t,
                                   C.POINTER(C.c_size_t)]),
    "pnr_render_fused": (C.c_int, [_vp, _vp, C.POINTER(PnrRenderArgs), _vp]),
    "pnr_render_fused_frames": (C.c_int, [_vp, _vp, C.POINTER(PnrRenderArgs), C.POINTER(PnrFrameTable), _vp]),
    "pnr_workspace_bytes": (C.c_size_t, [_vp, _i64, _i32, _i32]),
    "pnr_comm_available": (C.c_int, []),
    "pnr_comm_unique_id": (C.c_int, [C.POINTER(C.c_uint8)]),
    "pnr_comm_init": (C.c_int, [C.POINTER(_vp), C.POINTER(C.c_uint8), _i32, _i32, _i32]),
    "pnr_comm_destroy": (C.c_int, [_vp]),
    "pnr_allgather_outputs": (C.c_int, [_vp, _vp, _vp, C.c_size_t, _vp]),
    "pnr_broadcast": (C.c_int, [_vp, _vp, C.c_size_t, _i32, _vp]),
    "pnr_adam_step": (C.c_int, [_vp, _vp, _vp, _vp, C.POINTER(PnrAdamArgs), _vp, _vp]),
    "pnr_launch_count": (_i64, [_i32]),
    "pnr_eval_workspace_bytes": (C.c_size_t, [_i64]),
    "pnr_eval_semantic": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _i32, _vp, _vp]),
    "pnr_eval_panoptic": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _i32, _vp, _vp, C.c_size_t, _vp, _vp, _vp, _vp, _vp]),
    "pnr_eval_image": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, C.c_size_t, _vp]),
}


def lib() -> C.CDLL:
    """Load libpnr.so (once).  Fails loudly: the product has no path that works without it."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise PnrError(f"{_LIB_PATH} is missing - run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a).  panopticnerf_b200 has no CPU or PyTorch fallback.")
        L = C.CDLL(str(_LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)          # AttributeError here = header/library mismatch
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().pnr_last_error()
        raise PnrError(f"{what or 'libpnr'} failed (rc={rc}): {msg.decode() if msg else '?'}")


def set_mlp_rows(ctx: int, rows: int) -> None:
    """Tile of the context's raw-row MLP launches (pnr_set_mlp_rows): 0 = the one its program allows, 64 or 128."""
    check(lib().pnr_set_mlp_rows(ctx, rows), "pnr_set_mlp_rows")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor], dtype: Optional[torch.dtype] = None, name: str = "tensor"):
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise PnrError(f"{name}: expected a CUDA tensor, got {t.device} - panopticnerf_b200 is GPU-only "
                       "(no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise PnrError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise PnrError(f"{name}: expected a contiguous tensor")
    return t.data_ptr()


def ptr_struct(cls, tensors):
    """A struct of device pointers (PnrCompositeOut, PnrCompositeGrads) from tensors by field name; a field missing
    from `tensors` or None there is NULL."""
    return cls(**{k: ptr(tensors.get(k)) for k, _ in cls._fields_})
