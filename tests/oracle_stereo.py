"""numpy oracle of pnr_stereo_depth (include/pnr.h, DESIGN 3.4): a restatement of the semi-global matching rule in
integers - grey, census, cost, the eight path recursions (vectorised over the axis across the path and over d), the
winner, uniqueness, left-right check and subpixel with C's division written out - and the one float32 division of the
depth.  Also helpers to call the host build of stereo_math.h (tests/host_emu.cpp), scenes with a known disparity, and a
sequence in the KITTI-360 layout with the stereo pair."""
from pathlib import Path

import numpy as np

f32 = np.float32
BIG = 1 << 20                      # an absent d +- 1 term
DIRECTIONS = ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, -1), (1, -1), (-1, 1))


def grey(img):
    """[..., 3] u8 RGB -> [...] grey, (4899 R + 9617 G + 1868 B + 8192) >> 14."""
    c = np.asarray(img).astype(np.int64)
    return ((4899 * c[..., 0] + 9617 * c[..., 1] + 1868 * c[..., 2] + 8192) >> 14).astype(np.int64)


def census(g):
    """[H, W] grey -> [H, W] u64: the 9 x 7 window in raster order, centre skipped, bit k = g(q_k) < g(p), edges
    clamped."""
    H, W = g.shape
    pad = np.pad(g, ((3, 3), (4, 4)), mode="edge")
    bits = np.zeros((H, W), np.uint64)
    k = 0
    for dy in range(7):
        for dx in range(9):
            if dy == 3 and dx == 4:
                continue
            bits |= (pad[dy:dy + H, dx:dx + W] < g).astype(np.uint64) << np.uint64(k)
            k += 1
    return bits


def costs(cl, cr, D):
    """[H, W, D] int32: popcount(census_L(x) ^ census_R(x - d)) for x - d >= 0, else 63."""
    H, W = cl.shape
    out = np.full((H, W, D), 63, np.int32)
    for d in range(min(D, W)):
        out[:, d:, d] = np.bitwise_count(cl[:, d:] ^ cr[:, :W - d])
    return out


def step(prev, c, P1, P2):
    """One path step vectorised over paths: prev [n, D] = L_r(p - r), c [n, D] = C(p) -> L_r(p)."""
    m = prev.min(axis=1, keepdims=True)
    big = np.full((prev.shape[0], 1), BIG, prev.dtype)
    below = np.concatenate([big, prev[:, :-1]], 1)
    above = np.concatenate([prev[:, 1:], big], 1)
    return c + np.minimum(np.minimum(prev, below + P1), np.minimum(above + P1, m + P2)) - m


def aggregate(C_, dx, dy, P1, P2, out=None):
    """L_r of direction (dx, dy) over the cost volume [H, W, D] (added into `out` when given, which is returned).
    With dx != 0 the columns are walked in the direction's order, every row at once (row y continues the path of row
    y - dy of the previous column; rows whose y - dy is outside start afresh); with dx = 0 the rows likewise."""
    H, W, D = C_.shape
    L = np.zeros((H, W, D), np.int32)
    if dx != 0:
        order = range(W) if dx > 0 else range(W - 1, -1, -1)
        for k, x in enumerate(order):
            if k == 0:
                L[:, x] = C_[:, x]
                continue
            prev = L[:, x - dx]
            cur = np.empty((H, D), np.int32)
            if dy == 0:
                cur = step(prev, C_[:, x], P1, P2)
            elif dy > 0:
                cur[0] = C_[0, x]
                cur[1:] = step(prev[:-1], C_[1:, x], P1, P2)
            else:
                cur[-1] = C_[-1, x]
                cur[:-1] = step(prev[1:], C_[:-1, x], P1, P2)
            L[:, x] = cur
    else:
        order = range(H) if dy > 0 else range(H - 1, -1, -1)
        for k, y in enumerate(order):
            L[y] = C_[y] if k == 0 else step(L[y - dy], C_[y], P1, P2)
    if out is None:
        return L
    out += L
    return out


def _cdiv(a, b):
    """C's integer division (toward zero), b > 0."""
    q = np.abs(a) // b
    return np.where(a < 0, -q, q)


def select(S, U):
    """S [H, W, D] -> d16 [H, W] int16 (-1 = invalid)."""
    S = S.astype(np.int32)         # S 100 <= 1688800
    H, W, D = S.shape
    ds = np.argmin(S, axis=2)                            # the first minimum: lowest d on ties
    sb = np.take_along_axis(S, ds[..., None], 2)[..., 0]
    d = np.arange(D)
    far = np.abs(d[None, None, :] - ds[..., None]) > 1
    bad = (far & (S * (100 - U) < (sb * 100)[..., None])).any(axis=2)
    # d_R(x') = argmin_d S(x' + d, d) over x' + d < W
    T = np.full((H, W, D), np.iinfo(np.int32).max, np.int32)
    for k in range(min(D, W)):
        T[:, :W - k, k] = S[:, k:, k]
    dr = np.argmin(T, axis=2)
    xs = np.arange(W)[None, :] - ds
    ok = xs >= 0
    drx = np.take_along_axis(dr, np.clip(xs, 0, W - 1), 1)
    ok &= np.abs(ds - drx) <= 1
    inner = (ds > 0) & (ds < D - 1)
    lo = np.take_along_axis(S, np.clip(ds - 1, 0, D - 1)[..., None], 2)[..., 0]
    hi = np.take_along_axis(S, np.clip(ds + 1, 0, D - 1)[..., None], 2)[..., 0]
    den = np.maximum(lo + hi - 2 * sb, 1)
    sub = _cdiv((lo - hi) * 16 + den, 2 * den)
    d16 = np.where(inner, 16 * ds + sub, 16 * ds)
    return np.where(ok & ~bad, d16, -1).astype(np.int16)


def depth_of(d16, b16, min_depth, max_depth):
    """t = fp32(B16) / fp32(d16) where d16 > 0, kept inside (min_depth, max_depth], else 0."""
    d16 = np.asarray(d16)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = f32(b16) / d16.astype(f32)
    keep = (d16 > 0) & (t > f32(min_depth)) & (t <= f32(max_depth))
    return np.where(keep, t, f32(0)).astype(f32)


def sgm(left, right, D=128, P1=10, P2=120, U=10, want_S=False):
    """One pair [H, W, 3] u8 -> d16 [H, W] (and S [H, W, D])."""
    cl, cr = census(grey(left)), census(grey(right))
    C_ = costs(cl, cr, D)
    S = np.zeros(C_.shape, np.int32)
    for dx, dy in DIRECTIONS:
        aggregate(C_, dx, dy, P1, P2, out=S)
    d16 = select(S, U)
    return (d16, S) if want_S else d16


# ---------------------------------------------------------------------------------------------------- host build
def host_select(lib, S, U):
    """The host build's selection over S [H, W, D] -> d16 [H, W] i16."""
    S = np.ascontiguousarray(S, np.uint16)
    H, W, D = S.shape
    out = np.empty((H, W), np.int16)
    lib.emu_select(S.ctypes.data, H, W, D, U, out.ctypes.data)
    return out


def host_sgm(lib, left, right, D=128, P1=10, P2=120, U=10, b16=1.0, min_depth=0.1, max_depth=40.0, want_S=False):
    """The host build on one pair -> (d16 [H, W] i16, depth [H, W] f32[, S [H, W, D] u16])."""
    left = np.ascontiguousarray(left, np.uint8)
    right = np.ascontiguousarray(right, np.uint8)
    H, W = left.shape[:2]
    d16 = np.empty((H, W), np.int16)
    depth = np.empty((H, W), f32)
    S = np.empty((H, W, D), np.uint16) if want_S else None
    lib.emu_stereo(left.ctypes.data, right.ctypes.data, H, W, D, P1, P2, U, b16, min_depth, max_depth,
                   d16.ctypes.data, depth.ctypes.data, S.ctypes.data if want_S else None)
    return (d16, depth, S) if want_S else (d16, depth)


# ---------------------------------------------------------------------------------------------------- scenes
def random_dots(rng, H, W, d0):
    """A random-dot pair with the constant disparity d0: right(x) = left(x + d0) (fresh dots where x + d0 >= W)."""
    left = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    right = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    right[:, :W - d0] = left[:, d0:]
    return left, right


def _texture(X, Y, cell, seed):
    """A random RGB texture on the plane, constant over squares of side `cell` (metres)."""
    i = np.floor(X / cell).astype(np.int64)
    j = np.floor(Y / cell).astype(np.int64)
    h = (i * 73856093) ^ (j * 19349663) ^ (seed * 83492791)
    h = (h ^ (h >> 13)) * 0x5bd1e995
    h ^= h >> 15
    return np.stack([(h >> s) & 255 for s in (0, 8, 16)], -1).astype(np.uint8)


def render_pair(H, W, fx, cx, cy, b, layers):
    """Ray-cast fronto-parallel textured layers into the rectified pair: the left camera at the origin, the right at
    (b, 0, 0), both looking down +z with focal fx, centre (cx, cy).  layers: (Z, (u0, u1, v0, v1) in left pixels or
    None for the whole plane, seed), nearest first wins.  Returns (left, right) [H, W, 3] u8."""
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    out = []
    for shift in (0.0, b):
        img = np.zeros((H, W, 3), np.uint8)
        done = np.zeros((H, W), bool)
        for Z, box, seed in sorted(layers, key=lambda l: l[0]):
            X = (u - cx) * Z / fx + shift          # the point of the layer on this pixel's ray, in left coordinates
            Y = (v - cy) * Z / fx
            hit = ~done
            if box is not None:
                ul = X * fx / Z + cx                # its left pixel
                hit &= (ul >= box[0]) & (ul < box[1]) & (v >= box[2]) & (v < box[3])
            img[hit] = _texture(X, Y, Z / fx, seed)[hit]
            done |= hit
        out.append(img)
    return out[0], out[1]


# ---------------------------------------------------------------------------------------------------- sequence
def write_stereo_sequence(root: Path, frames, pairs, fx=40.0, cx=31.5, cy=23.5, b=0.6, K01=None, seq=None,
                          right_size=None):
    """A sequence in the KITTI-360 layout (oracle_lidar.write_sequence: poses and calibration) with the stereo pair:
    image_00 / image_01 data_rect PNGs of pairs[i] = (left, right) RGB, and perspective.txt with P_rect_00 / S_rect_00
    and P_rect_01 (K01: its K, default the same; P_rect_01[0, 3] = -fx b) / S_rect_01.  Returns write_sequence's dict."""
    import cv2
    import oracle_lidar as OL
    H, W = pairs[0][0].shape[:2]
    kw = {} if seq is None else {"seq": seq}
    info = OL.write_sequence(root, frames, cams=("image_00",), scans=[], images=False, **kw)
    k = (fx, fx, cx, cy) if K01 is None else K01
    rs = (W, H) if right_size is None else right_size
    (root / "calibration" / "perspective.txt").write_text(
        f"P_rect_00: {fx!r} 0 {cx!r} 0 0 {fx!r} {cy!r} 0 0 0 1 0\nS_rect_00: {W} {H}\n"
        f"P_rect_01: {k[0]!r} 0 {k[2]!r} {-fx * b!r} 0 {k[1]!r} {k[3]!r} 0 0 0 1 0\nS_rect_01: {rs[0]} {rs[1]}\n")
    for cam, idx in (("image_00", 0), ("image_01", 1)):
        d = root / "data_2d_raw" / info["seq"] / cam / "data_rect"
        d.mkdir(parents=True, exist_ok=True)
        for f, p in zip(frames, pairs):
            cv2.imwrite(str(d / f"{f:010d}.png"), np.ascontiguousarray(p[idx][:, :, ::-1]))
    return info
