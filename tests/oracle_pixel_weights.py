"""numpy restatement of the weighted draws (include/pnr.h, DESIGN 3.4): the per-pixel composition rule in float32, the
uint64 prefix sum and its group entries, the weighted pick as searchsorted(side="right") and the importance in float64;
plus helpers that call the host build (tests/host_emu_weights.cpp).  Shared by the CPU and GPU weight tests."""
import ctypes as C

import numpy as np

import oracle_ray_batch as O
from panopticnerf_b200 import _capi

GROUP = 32


def host_lib():
    """The host build of the weighted-draw routines (tests/host_emu_weights.cpp), built and loaded, its argtypes set."""
    from panopticnerf_b200._build import build_host_emu_weights
    lib = C.CDLL(str(build_host_emu_weights()))
    lib.emu_weighted_pixel.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint64]
    lib.emu_weighted_pixel.restype = C.c_int64
    lib.emu_pixel_weight.argtypes = [C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.emu_pixel_weight.restype = None
    lib.emu_pixel_weights.argtypes = [C.POINTER(_capi.PnrPixelWeightsArgs)]
    lib.emu_pixel_weights.restype = None
    lib.emu_sample_ray_batch_weighted.argtypes = [C.POINTER(_capi.PnrRayBatchArgs), C.POINTER(_capi.PnrRayBatchWeights)]
    lib.emu_sample_ray_batch_weighted.restype = None
    return lib


def rule(keep, scale, ff, cf):
    """weight u16 of x = (scale * ff) * cf in float32 (each product rounded): 0 when not kept, NaN or <= 0; 65535 at
    or past 65535; otherwise round half to even."""
    with np.errstate(invalid="ignore", over="ignore"):
        x = (np.float32(scale) * np.asarray(ff, np.float32)) * np.asarray(cf, np.float32)
        out = np.where(x >= np.float32(65535), np.float32(65535), np.rint(np.where(x > 0, x, 0)))
        out = np.where(np.asarray(keep, bool) & (x > 0), out, 0)
    return out.astype(np.uint16)


def slots(label, C):
    """class-factor slot of each label: 1 + label in [0, C), else 0."""
    label = np.asarray(label).astype(np.int64)
    return np.where((label >= 0) & (label < C), label + 1, 0)


def frame_set_weights(fs, scale, C=0, ff=None, cf=None, masks=None):
    """weight [P] of a (well-formed) frame set of oracle_ray_batch.random_frame_set under the rule."""
    off = fs["pix_offset"]
    P = int(off[-1])
    out = np.zeros(P, np.uint16)
    for f in range(len(fs["frame_cam"])):
        cam = int(fs["frame_cam"][f])
        lo, hi = int(off[f]), int(off[f + 1])
        keep = np.ones(hi - lo, bool) if masks is None or masks[cam] is None else masks[cam].reshape(-1) != 0
        s = slots(fs["label"][lo:hi], C) if (fs["label"] is not None and C > 0) else np.zeros(hi - lo, np.int64)
        cfv = np.asarray(cf, np.float32)[s] if cf is not None else np.ones(hi - lo, np.float32)
        ffv = np.float32(ff[f]) if ff is not None else np.float32(1)
        out[lo:hi] = rule(keep, scale, np.full(hi - lo, ffv, np.float32), cfv)
    return out


def cumsum(weight):
    return np.cumsum(np.asarray(weight, np.uint64), dtype=np.uint64)


def groups(weight):
    """cum [ceil(P/32)]: the inclusive sum through the last pixel of each group of 32."""
    S = cumsum(weight)
    P = len(S)
    return S[np.minimum(P, GROUP * (np.arange((P + GROUP - 1) // GROUP) + 1)) - 1]


def pick(weight, x):
    """the smallest p with S(p) > x."""
    return np.searchsorted(cumsum(weight), np.asarray(x, np.uint64), side="right").astype(np.int64)


def importance(T, nonzero, w):
    return (np.float64(T) / (np.float64(nonzero) * np.asarray(w, np.float64))).astype(np.float32)


def draws(seed, step, r, T):
    """x of each global ray r: the high 64 bits of (w0 << 32 | w1) * T (Python integers: exact)."""
    w = O.draw(seed, step, r, 0)
    x = (w[0].astype(object) << 32) | w[1].astype(object)
    return np.array([(int(v) * int(T)) >> 64 for v in x], dtype=np.uint64)


def weighted_pixels(seed, step, r, weight):
    S = cumsum(weight)
    return pick(weight, draws(seed, step, r, int(S[-1])))


def host_weights(lib, fs, scale, ncls=0, ff=None, cf=None, masks=None, fill=0xABCD):
    """The host build's weight [P] (emu_pixel_weights) of frame set fs, starting from `fill` everywhere."""
    keep = []

    def ptr(x, dtype=None):
        if x is None:
            return None
        x = np.ascontiguousarray(x, dtype)
        keep.append(x)
        return x.ctypes.data
    P = int(fs["pix_offset"][-1])
    a = _capi.PnrPixelWeightsArgs()
    a.frame_cam, a.pix_offset = ptr(fs["frame_cam"]), ptr(fs["pix_offset"])
    a.F, a.P = len(fs["frame_cam"]), P
    for k, (model, H, W, intr) in enumerate(fs["cams"]):
        a.cams[k].model, a.cams[k].H, a.cams[k].W = model, H, W
        for i, v in enumerate(intr):
            a.cams[k].intr[i] = v
        a.mask[k] = ptr(masks[k], np.uint8) if masks is not None and masks[k] is not None else None
    a.num_cameras = len(fs["cams"])
    a.label = ptr(fs["label"]) if ncls > 0 else None
    a.C = ncls
    a.frame_factor = ptr(ff, np.float32)
    a.class_factor = ptr(cf, np.float32)
    a.scale = scale
    out = np.full(P, fill, np.uint16)
    a.weight = out.ctypes.data
    lib.emu_pixel_weights(C.byref(a))
    return out


def host_weighted_batch(lib, fs, weight, seed, step, r0, r1, N, Ni):
    """The host build's weighted rows r0 .. r1-1 (emu_sample_ray_batch_weighted): oracle_ray_batch.host_batch's keys
    plus importance."""
    n = r1 - r0
    weight = np.ascontiguousarray(weight, np.uint16)
    cum = np.ascontiguousarray(groups(weight))
    out = dict(rays=np.zeros((n, 6), np.float32), rgb=np.zeros((n, 3), np.float32), u=np.zeros((n, N), np.float32),
               u_fine=np.zeros((n, Ni), np.float32), depth=np.zeros(n, np.float32),
               pseudo_label=np.zeros(n, np.int32), pixel=np.zeros(n, np.int64), importance=np.zeros(n, np.float32))
    keep = [weight, cum]

    def ptr(x):
        if x is None:
            return None
        x = np.ascontiguousarray(x)
        keep.append(x)
        return x.ctypes.data
    a = O.fill_args(_capi.PnrRayBatchArgs(), fs, seed, step, r0, r1, N, Ni, ptr)
    a.rays, a.rgb, a.u = out["rays"].ctypes.data, out["rgb"].ctypes.data, out["u"].ctypes.data
    a.u_fine = out["u_fine"].ctypes.data if Ni else None
    a.depth_out, a.pseudo_label, a.pixel = out["depth"].ctypes.data, out["pseudo_label"].ctypes.data, out["pixel"].ctypes.data
    wt = _capi.PnrRayBatchWeights(weight.ctypes.data, cum.ctypes.data, int(cum[-1]), int(np.count_nonzero(weight)),
                                  out["importance"].ctypes.data)
    lib.emu_sample_ray_batch_weighted(C.byref(a), C.byref(wt))
    return out
