"""numpy restatement of pnr_sample_ray_batch's draws (include/pnr.h): Philox4x32-10, the 64-bit multiply-high pixel
pick, the frame search and the jitter words; plus helpers that build frame sets and call the host build of
pnr_ray_batch_row (tests/host_emu.cpp, fixture `emu` of tests/host_emu.py).  Shared by the CPU and GPU ray-batch
tests."""
import ctypes as C

import numpy as np

from panopticnerf_b200 import _capi

MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (broadcast); returns four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for i in range(10):
        if i:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & MASK, (k1 + np.uint64(0xBB67AE85)) & MASK
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & MASK]
    return [x.astype(np.uint32) for x in c]


def draw(seed, step, r, block):
    """Block `block` of the global rays r: counter (block, r, step lo, step hi), key (seed lo, seed hi)."""
    r = np.asarray(r, dtype=np.uint64)
    return philox4x32_10(np.full_like(r, block), r, np.full_like(r, step & 0xFFFFFFFF),
                         np.full_like(r, step >> 32), seed & 0xFFFFFFFF, seed >> 32)


def u01(w):
    return (np.asarray(w) >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def pixels(seed, step, r, P):
    """Flat pixel of each global ray r: the high 64 bits of (w0 << 32 | w1) * P (Python integers: exact)."""
    w = draw(seed, step, r, 0)
    x = (w[0].astype(object) << 32) | w[1].astype(object)
    return np.array([(int(v) * int(P)) >> 64 for v in x], dtype=np.int64)


def frame_of(off, p):
    """The last f with off[f] <= p (an upper-bound search)."""
    return np.searchsorted(np.asarray(off), np.asarray(p), side="right").astype(np.int64) - 1


def jitter(seed, step, r, N, Ni):
    """u [n, N], u_fine [n, Ni]: jitter word k is word k % 4 of block 1 + k // 4."""
    words = []
    for b in range((N + Ni + 3) // 4):
        words += draw(seed, step, r, 1 + b)
    w = np.stack(words, 1)[:, :N + Ni]
    return u01(w[:, :N]), u01(w[:, N:])


# ------------------------------------------------------------------------------------------------ frame sets
def random_cameras(rng, n, fisheye=True, tiny=False):
    """n cameras of mixed models: (model, H, W, intr); tiny adds a 1 x 1 camera (one-pixel frames)."""
    cams = []
    for k in range(n):
        H, W = (1, 1) if (tiny and k == 0) else (int(rng.integers(2, 40)), int(rng.integers(2, 60)))
        if fisheye and k % 2 == 1:
            cams.append((2, H, W, [0.6 * W, 0.6 * W, W / 2 + 0.3, H / 2 - 0.2, 1.2, 0.02, 0.01]))
        else:
            cams.append((0, H, W, [0.9 * W, 0.8 * W, W / 2 - 0.5, H / 2 + 0.25]))
    return cams


def random_frame_set(rng, F, cams, with_label=True, with_depth=True):
    """Host arrays of F frames: c2w [F,12] f32 (rotation + translation), frame_cam, pix_offset, rgb8, label, depth."""
    fc = rng.integers(0, len(cams), F).astype(np.int32)
    sizes = [cams[c][1] * cams[c][2] for c in fc]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    P = int(off[-1])
    c2w = np.empty((F, 12), np.float32)
    for f in range(F):
        q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
        c2w[f] = np.concatenate([q, rng.standard_normal((3, 1)) * 5], 1).astype(np.float32).reshape(-1)
    rgb8 = rng.integers(0, 256, (P, 3)).astype(np.uint8)
    label = rng.integers(-1, 20, P).astype(np.int16) if with_label else None
    depth = np.where(rng.random(P) < 0.6, rng.random(P) * 50, 0).astype(np.float32) if with_depth else None
    return dict(c2w=c2w, frame_cam=fc, pix_offset=off, rgb8=rgb8, label=label, depth=depth, cams=cams)


def fill_args(a, fs, seed, step, r0, r1, N, Ni, ptr):
    """pnr_ray_batch_args `a` of frame set fs (arrays turned into pointers by ptr(array or None))."""
    a.c2w, a.frame_cam, a.pix_offset = ptr(fs["c2w"]), ptr(fs["frame_cam"]), ptr(fs["pix_offset"])
    a.F, a.P = len(fs["frame_cam"]), int(fs["pix_offset"][-1])
    a.rgb8, a.label, a.depth = ptr(fs["rgb8"]), ptr(fs["label"]), ptr(fs["depth"])
    for k, (model, H, W, intr) in enumerate(fs["cams"]):
        a.cams[k].model, a.cams[k].H, a.cams[k].W = model, H, W
        for i, x in enumerate(intr):
            a.cams[k].intr[i] = x
    a.num_cameras = len(fs["cams"])
    a.seed, a.step, a.r0, a.r1, a.N, a.Ni = seed, step, r0, r1, N, Ni
    return a


def host_batch(emu, fs, seed, step, r0, r1, N, Ni):
    """The host build's rows r0 .. r1-1 (numpy outputs; depth / pseudo_label / pixel always written)."""
    n = r1 - r0
    out = dict(rays=np.zeros((n, 6), np.float32), rgb=np.zeros((n, 3), np.float32), u=np.zeros((n, N), np.float32),
               u_fine=np.zeros((n, Ni), np.float32), depth=np.zeros(n, np.float32),
               pseudo_label=np.zeros(n, np.int32), pixel=np.zeros(n, np.int64))
    keep = []

    def ptr(x):
        if x is None:
            return None
        x = np.ascontiguousarray(x)
        keep.append(x)
        return x.ctypes.data
    a = fill_args(_capi.PnrRayBatchArgs(), fs, seed, step, r0, r1, N, Ni, ptr)
    a.rays, a.rgb, a.u = out["rays"].ctypes.data, out["rgb"].ctypes.data, out["u"].ctypes.data
    a.u_fine = out["u_fine"].ctypes.data if Ni else None
    a.depth_out, a.pseudo_label, a.pixel = out["depth"].ctypes.data, out["pseudo_label"].ctypes.data, out["pixel"].ctypes.data
    emu.emu_sample_ray_batch(C.byref(a))
    return out


def host_frame_rays(emu, fs, f):
    """All rays of frame f through the host build of pnr_generate_rays (emu_generate_rays)."""
    model, H, W, intr = fs["cams"][int(fs["frame_cam"][f])]
    rays = np.zeros((H * W, 6), np.float32)
    k = np.asarray(intr, np.float32)
    m = np.ascontiguousarray(fs["c2w"][f])
    assert emu.emu_generate_rays(H, W, 0, H, model, k.ctypes.data_as(C.POINTER(C.c_float)),
                                 m.ctypes.data_as(C.POINTER(C.c_float)), rays.ctypes.data_as(C.POINTER(C.c_float))) == 0
    return rays
