"""CPU tier of stereo depth targets (pnr_stereo_depth, kitti360/stereo.py): the numpy oracle on hand-worked and known
answers, scenes with a known disparity, the host build of stereo_math.h against the oracle bit for bit, every refusal
of the C entry point by name before any device call, the workspace layout, the ctypes layout, and the readers'
refusals on sequences written in the KITTI-360 layout."""
import ctypes as C
import itertools
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_stereo as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h and stereo_math.h)
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.datasets.kitti360 import load_frames
from panopticnerf_b200.lib.datasets.kitti360 import stereo as ST
from panopticnerf_b200.lib.datasets.ray_batch import Camera, FrameSet

ROOT = Path(__file__).resolve().parent.parent
f32 = np.float32


# ---------------------------------------------------------------------------------------------------- the oracle
def test_hand_worked_aggregation_along_one_row():
    # W = 3, D = 3, P1 = 1, P2 = 3, walked left to right (r = (1, 0)):
    #   x0: L = C = [5, 0, 9], m = 0
    #   x1: C = [2, 7, 1]: d0 2 + min(5, 0 + 1, 3) = 3; d1 7 + min(0, 6, 10, 3) = 7; d2 1 + min(9, 1, 3) = 2; m = 2
    #   x2: C = [0, 4, 4]: d0 0 + min(3, 8, 5) - 2 = 1; d1 4 + min(7, 4, 3, 5) - 2 = 5; d2 4 + min(2, 8, 5) - 2 = 4
    C_ = np.array([[[5, 0, 9], [2, 7, 1], [0, 4, 4]]], np.int32)
    L = O.aggregate(C_, 1, 0, 1, 3)
    assert L[0].tolist() == [[5, 0, 9], [3, 7, 2], [1, 5, 4]]
    # right to left the path starts at x2
    assert O.aggregate(C_, -1, 0, 1, 3)[0, 2].tolist() == [0, 4, 4]


@pytest.mark.parametrize("P1,P2", [(0, 0), (10, 120), (2048, 2048), (7, 9)])
def test_path_costs_stay_within_63_plus_P2(P1, P2):
    rng = np.random.default_rng(P1 + P2)
    C_ = rng.integers(0, 64, (9, 23, 64)).astype(np.int32)
    for dx, dy in O.DIRECTIONS:
        L = O.aggregate(C_, dx, dy, P1, P2)
        assert L.min() >= 0 and L.max() <= 63 + P2
    S = sum(O.aggregate(C_, dx, dy, P1, P2) for dx, dy in O.DIRECTIONS)
    assert S.max() < 1 << 16


def test_a_flat_image_matches_everything_at_zero(emu):
    img = np.full((12, 20, 3), 77, np.uint8)
    cen = O.census(O.grey(img))
    C_ = O.costs(cen, cen, 32)
    x, d = np.meshgrid(np.arange(20), np.arange(32), indexing="ij")
    assert not C_[:, x >= d].any() and (C_[:, x < d] == 63).all()   # every real cost 0; x - d < 0 costs 63
    d16, S = O.sgm(img, img, 32, want_S=True)
    assert not S[..., 0].any()
    assert not d16.any()
    assert not O.depth_of(d16, 1000.0, 0.1, 40.0).any()
    hd, hdep = O.host_sgm(emu, img, img, 32, b16=1000.0)
    assert not hd.any() and not hdep.any()


def _row_volume(vec, W):
    return np.tile(np.asarray(vec, np.int64), (1, W, 1))


def test_ties_pick_the_lowest_disparity(emu):
    # S(d) = 5 min(|d - 3|, |d - 4|): a tie between d = 3 and 4 everywhere; d* = 3 and d_R = 3 (also the lowest),
    # subpixel: lo = 5, hi = 0, den = 5, (5 16 + 5) / 10 = 8 -> d16 = 56 where x >= 3
    d = np.arange(32)
    S = _row_volume(5 * np.minimum(np.abs(d - 3), np.abs(d - 4)), 10)
    got = O.select(S, 0)
    assert got[0].tolist() == [-1, -1, -1] + [56] * 7
    assert np.array_equal(O.host_select(emu, S, 0), got)


def test_uniqueness_at_equality_and_one_unit_past(emu):
    # d* = 2 with S = 90; with U = 10 a far d with S(d) 90 < 90 100 refuses: S(d) = 100 is the equality (kept),
    # S(d) = 99 one unit past (refused)
    for far, want in ((100, 32), (99, -1)):
        vec = np.full(32, 500)
        vec[2] = 90
        vec[1] = vec[3] = 200             # the subpixel neighbours: symmetric, so d16 = 16 d*
        vec[10] = far
        S = _row_volume(vec, 6)
        got = O.select(S, 10)
        assert got[0, 2:].tolist() == [want] * 4, (far, got)
        assert np.array_equal(O.host_select(emu, S, 10), got)
    # d* +- 1 never counts against uniqueness
    vec = np.full(32, 500)
    vec[2], vec[3], vec[1] = 90, 90, 95
    assert O.select(_row_volume(vec, 6), 10)[0, 5] >= 0


def test_subpixel_truncates_negative_numerators_toward_zero(emu):
    # S(d*-1) = 10, S(d*) = 4, S(d*+1) = 30: den = 32, numerator (10 - 30) 16 + 32 = -288, -288 / 64 = -4.5 -> -4
    # (floor division would give -5); d* = 5 -> d16 = 76
    vec = np.full(32, 900)
    vec[4:7] = [10, 4, 30]
    S = _row_volume(vec, 8)
    got = O.select(S, 10)
    assert got[0, 5:].tolist() == [76, 76, 76]
    assert np.array_equal(O.host_select(emu, S, 10), got)
    # positive numerator: S(d*-1) = 30, S(d*+1) = 10: (20 16 + 32) / 64 = 5 (5.5 truncated)
    vec[4:7] = [30, 4, 10]
    assert O.select(_row_volume(vec, 8), 10)[0, 5] == 85


# ---------------------------------------------------------------------------------------------------- scenes
def test_random_dots_at_a_constant_disparity(emu):
    rng = np.random.default_rng(1)
    d0 = 9
    left, right = O.random_dots(rng, 40, 120, d0)
    d16 = O.sgm(left, right, 64)
    assert np.array_equal(O.host_sgm(emu, left, right, 64)[0], d16)
    inner = d16[3:-3, d0 + 4:-4]                    # away from the clamped census border and the unmatched band
    assert (np.rint(inner / 16) == d0).mean() >= 0.99


def test_a_fronto_parallel_plane_reads_its_depth(emu):
    # fx b / Z = 6 exactly: the plane's texture cells are one pixel wide at Z, so each right pixel sees the left
    # pixel six to its right.  Strong smoothness (P1 = 200, P2 = 2048) keeps the parabola's two sides even, so the
    # subpixel rule lands within one sixteenth of 96.
    H, W, fx, b, d0 = 40, 120, 40.0, 0.6, 6
    Z = fx * b / d0
    left, right = O.render_pair(H, W, fx, 59.5, 19.5, b, [(Z, None, 3)])
    b16 = float(f32(16 * fx * b))
    d16, depth = O.host_sgm(emu, left, right, 64, 200, 2048, 10, b16, 0.1, 40.0)
    assert np.array_equal(d16, O.sgm(left, right, 64, 200, 2048, 10))
    inner = (slice(3, -3), slice(d0 + 4, -4))
    assert (d16[inner] >= 0).all()
    assert np.abs(d16[inner].astype(int) - 16 * d0).max() <= 1
    assert np.abs(depth[inner] - Z).max() <= Z / 90       # one sixteenth of 6 px
    assert np.array_equal(depth, O.depth_of(d16, b16, 0.1, 40.0))


def test_the_band_a_near_square_occludes_fails_the_left_right_check(emu):
    # far plane at disparity 4, a square at disparity 12 over left columns [50, 80): the far plane's pixels of left
    # columns [42, 50) are hidden from the right camera by the square.  U = 0 turns uniqueness off, so what refuses
    # them is the left-right check.
    H, W, fx, b = 48, 128, 40.0, 0.6
    left, right = O.render_pair(H, W, fx, 63.5, 23.5, b, [(fx * b / 4, None, 1), (fx * b / 12, (50, 80, 10, 38), 2)])
    d16 = O.sgm(left, right, 32, 10, 120, 0)
    assert np.array_equal(O.host_sgm(emu, left, right, 32, 10, 120, 0)[0], d16)
    band = d16[14:34, 43:49]
    assert (band < 0).mean() >= 0.9
    assert (np.abs(d16[14:34, 54:76].astype(int) - 192) <= 8).mean() >= 0.95
    assert (np.abs(d16[14:34, 20:38].astype(int) - 64) <= 8).mean() >= 0.95


# ---------------------------------------------------------------------------------------------------- host vs oracle
SHAPES = [(1, 1), (1, 33), (7, 9), (33, 65), (48, 64)]
PENALTIES = [(0, 0), (10, 120), (2048, 2048)]
UNIQUENESS = [0, 10, 99]
CASES = [(H, W, D, *PENALTIES[k % 3], UNIQUENESS[(k // 3) % 3])
         for k, ((H, W), D) in enumerate(itertools.product(SHAPES, range(32, 257, 32)))]


@pytest.mark.parametrize("H,W,D,P1,P2,U", CASES)
def test_host_build_equals_the_oracle(H, W, D, P1, P2, U, emu):
    rng = np.random.default_rng(H * 1000 + W * 10 + D)
    left, right = O.random_dots(rng, H, W, min(5, W - 1))
    if H > 1:   # smooth parts too, where ties and flat costs occur
        left[: H // 3] //= 64
        right[: H // 3] //= 64
    b16 = float(f32(16 * 552.554 * 0.6))
    d16, depth, S = O.host_sgm(emu, left, right, D, P1, P2, U, b16, 1.0, 40.0, want_S=True)
    want, wS = O.sgm(left, right, D, P1, P2, U, want_S=True)
    assert np.array_equal(S.astype(np.int32), wS)
    assert np.array_equal(d16, want)
    assert depth.tobytes() == O.depth_of(want, b16, 1.0, 40.0).tobytes()


# ---------------------------------------------------------------------------------------------------- C ABI
def _valid_args():
    a = _capi.PnrStereoArgs()
    frames = np.array([0, 2], np.int32)
    a.rgb8, a.pix_offset, a.P, a.F = 0x100000, 0x200000, 3 * 376 * 1408, 3
    a.frames, a.n, a.H, a.W = frames.ctypes.data, 2, 376, 1408
    a.right, a.D, a.P1, a.P2, a.U = 0x300000, 128, 10, 120, 10
    a.B16, a.min_depth, a.max_depth = 5304.0, 0.1, 40.0
    a.depth, a.disparity = 0x400000, 0x500000
    a.workspace = 0x600000
    a.workspace_bytes = _capi.lib().pnr_stereo_workspace_bytes(2, 376, 1408, 128)
    return a, frames


def test_every_argument_is_refused_by_name_before_any_device_call():
    need = _capi.lib().pnr_stereo_workspace_bytes(2, 376, 1408, 128)
    bad_frames = np.array([0, 3], np.int32)
    cases = [
        (lambda a: setattr(a, "n", 0), "n=0"),
        (lambda a: setattr(a, "n", -3), "n=-3"),
        (lambda a: setattr(a, "H", 0), "H=0"),
        (lambda a: setattr(a, "W", 0), "W=0"),
        (lambda a: setattr(a, "W", 65536), "W=65536"),
        (lambda a: setattr(a, "D", 16), "D=16"),
        (lambda a: setattr(a, "D", 100), "D=100"),
        (lambda a: setattr(a, "D", 288), "D=288"),
        (lambda a: setattr(a, "P1", -1), "P1=-1"),
        (lambda a: setattr(a, "P1", 121), "P1=121 P2=120"),
        (lambda a: (setattr(a, "P1", 2049), setattr(a, "P2", 2049)), "P2=2049"),
        (lambda a: setattr(a, "U", -1), "U=-1"),
        (lambda a: setattr(a, "U", 100), "U=100"),
        (lambda a: setattr(a, "F", 0), "F=0"),
        (lambda a: setattr(a, "P", 0), "P=0"),
        (lambda a: setattr(a, "rgb8", None), "null input pointer"),
        (lambda a: setattr(a, "pix_offset", None), "null input pointer"),
        (lambda a: setattr(a, "right", None), "null input pointer"),
        (lambda a: setattr(a, "frames", None), "null input pointer"),
        (lambda a: (setattr(a, "depth", None), setattr(a, "disparity", None)), "null outputs"),
        (lambda a: setattr(a, "frames", bad_frames.ctypes.data), "frames[1]=3 outside [0, F=3)"),
        (lambda a: setattr(a, "B16", 0.0), "B16=0"),
        (lambda a: setattr(a, "B16", float("inf")), "B16=inf"),
        (lambda a: setattr(a, "min_depth", 0.0), "min_depth=0"),
        (lambda a: setattr(a, "min_depth", float("nan")), "min_depth=nan"),
        (lambda a: setattr(a, "max_depth", 0.05), "max_depth=0.05"),
        (lambda a: setattr(a, "max_depth", float("inf")), "max_depth=inf"),
        (lambda a: setattr(a, "workspace", None), "workspace of"),
        (lambda a: setattr(a, "workspace_bytes", need - 1), f"needs {need} bytes"),
        (lambda a: setattr(a, "workspace", 0x600008), "16-byte aligned"),
    ]
    for mutate, what in cases:
        a, keep = _valid_args()
        mutate(a)
        assert _capi.lib().pnr_stereo_depth(C.byref(a), None) == -1, what
        msg = _capi.lib().pnr_last_error().decode()
        assert what in msg, (what, msg)
    assert _capi.lib().pnr_stereo_depth(None, None) == -1


def _align(b):
    return (b + 15) // 16 * 16


@pytest.mark.parametrize("n,H,W,D", [(1, 1, 1, 32), (2, 376, 1408, 128), (17, 7, 9, 256), (3, 5, 3, 96)])
def test_workspace_bytes_is_the_documented_layout(n, H, W, D):
    N = n * H * W
    assert _capi.lib().pnr_stereo_workspace_bytes(n, H, W, D) == 2 * _align(8 * N) + _align(2 * N * D) + _align(2 * N)


def test_workspace_bytes_is_zero_outside_the_ranges():
    for args in ((0, 4, 4, 32), (1, 0, 4, 32), (1, 4, 65536, 32), (1, 4, 4, 48), (1, 4, 4, 0), (1, 4, 4, 288)):
        assert _capi.lib().pnr_stereo_workspace_bytes(*args) == 0, args


def test_stereo_args_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _capi.PnrStereoArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(pnr_stereo_args, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(pnr_stereo_args));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = [getattr(_capi.PnrStereoArgs, f).offset for f in fields] + [C.sizeof(_capi.PnrStereoArgs)]
    assert got == want


# ---------------------------------------------------------------------------------------------------- readers
def _pairs(n, H=24, W=32, seed=0):
    rng = np.random.default_rng(seed)
    return [O.random_dots(rng, H, W, 3) for _ in range(n)]


def _cpu_set(names, H=24, W=32):
    cams = [Camera("pinhole", H, W, (20.0, 20.0, 15.5, 11.5))]
    return FrameSet.from_images(cams, [0] * len(names), np.tile(np.eye(4)[:3], (len(names), 1, 1)),
                                [torch.zeros(H, W, 3, dtype=torch.uint8)] * len(names), names=names, device="cpu")


def test_stereo_depth_refuses_by_name(tmp_path):
    info = O.write_stereo_sequence(tmp_path, [5, 6], _pairs(2), fx=20.0, cx=15.5, cy=11.5)
    seq = info["seq"]
    fs = _cpu_set([("image_00", 5), ("image_00", 6)])
    bad = [dict(num_disparities=48), dict(num_disparities=288), dict(num_disparities=64.0), dict(P1=-1),
           dict(P1=130), dict(P2=2049), dict(uniqueness=100), dict(uniqueness=-1), dict(min_depth=0.0),
           dict(min_depth=float("nan")), dict(max_depth=0.05), dict(max_depth=float("inf")), dict(chunk_frames=0)]
    for kw in bad:
        with pytest.raises(ValueError, match=f"stereo_depth: .*{next(iter(kw))}="):
            ST.stereo_depth(fs, tmp_path, seq, **kw)
    with pytest.raises(ValueError, match="no image_00 frames"):
        ST.stereo_depth(_cpu_set([("image_02", 5)]), tmp_path, seq)
    unnamed = FrameSet(fs.cameras, fs.c2w, fs.frame_cam, fs.pix_offset, fs.rgb8)
    with pytest.raises(ValueError, match="names 0 of its 2 frames"):
        ST.stereo_depth(unnamed, tmp_path, seq)
    missing = _cpu_set([("image_00", 5), ("image_00", 7)])
    with pytest.raises(FileNotFoundError, match="0000000007.png: missing right image"):
        ST.stereo_depth(missing, tmp_path, seq)
    assert fs.depth is None and missing.depth is None      # refused before anything was allocated


@pytest.mark.parametrize("what", ["K", "baseline0", "baseline_neg", "baseline_inf", "S_rect_01", "image"])
def test_calibration_and_image_refusals(tmp_path, what):
    import cv2
    kw = dict(fx=20.0, cx=15.5, cy=11.5)
    if what == "K":
        kw["K01"] = (20.0, 20.0, 15.5, 12.0)
    if what == "baseline0":
        kw["b"] = 0.0
    if what == "baseline_neg":
        kw["b"] = -0.5
    if what == "baseline_inf":
        kw["b"] = 1e300
    if what == "S_rect_01":
        kw["right_size"] = (30, 24)
    info = O.write_stereo_sequence(tmp_path, [5], _pairs(1), **kw)
    if what == "image":
        p = tmp_path / "data_2d_raw" / info["seq"] / "image_01" / "data_rect" / "0000000005.png"
        cv2.imwrite(str(p), np.zeros((24, 30, 3), np.uint8))
    msg = {"K": "P_rect_01's K", "baseline0": "16 fx b", "baseline_neg": "16 fx b", "baseline_inf": "16 fx b",
           "S_rect_01": "S_rect_01 is 30 x 24", "image": "the right image is 30 x 24"}[what]
    with pytest.raises(ValueError, match=msg):
        ST.stereo_depth(_cpu_set([("image_00", 5)]), tmp_path, info["seq"])


def test_load_frames_refuses_stereo_with_another_depth_source(tmp_path):
    info = O.write_stereo_sequence(tmp_path, [5], _pairs(1), fx=20.0, cx=15.5, cy=11.5)
    seq = info["seq"]
    with pytest.raises(ValueError, match="stereo and depth_dir both give the depth table"):
        load_frames(tmp_path, seq, [5], depth_dir=tmp_path, stereo=True, device="cpu")
    with pytest.raises(ValueError, match="stereo and lidar both give the depth table"):
        load_frames(tmp_path, seq, [5], lidar=True, stereo=True, device="cpu")
    with pytest.raises(ValueError, match="stereo=.*keys from"):
        load_frames(tmp_path, seq, [5], stereo={"disparities": 64}, device="cpu")
    with pytest.raises(ValueError, match="stereo=.*keys from"):
        load_frames(tmp_path, seq, [5], stereo="yes", device="cpu")
    a = load_frames(tmp_path, seq, [5], device="cpu", stereo=False)
    assert a.depth is None


def test_stereo_disparity_refuses_its_options():
    x = torch.zeros(1, 4, 4, 3, dtype=torch.uint8)
    for kw, what in ((dict(num_disparities=16), "num_disparities=16"), (dict(P1=5, P2=4), "P1=5, P2=4"),
                     (dict(uniqueness=100), "uniqueness=100")):
        with pytest.raises(ValueError, match=what):
            ST.stereo_disparity(x, x, **kw)
    with pytest.raises(ValueError, match="expected two"):
        ST.stereo_disparity(x, torch.zeros(1, 4, 5, 3, dtype=torch.uint8))
