"""CPU tier of weighted draws: the host build of the composition rule (pnr_pixel_weight / pnr_weight_of_pixel of
csrc/ray_math.h, tests/host_emu_weights.cpp) against the numpy float32 oracle bit for bit, the weighted pick against a uint64
cumsum + searchsorted, whole weighted batches against the oracle, all-ones weights against the unweighted batch, a
chi-square of the draw, the argument structs' layout against a C compile of include/pnr.h, every refusal before any
device call, and the sharder slicing importance with the rays."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_pixel_weights as W
import oracle_ray_batch as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h)
from panopticnerf_b200 import _capi, parallel

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def hw():
    """the host build of the weighted-draw routines (tests/host_emu_weights.cpp)"""
    return W.host_lib()


def _rule(hw, keep, scale, ff, cf):
    keep = np.ascontiguousarray(keep, np.uint8)
    ff, cf = np.ascontiguousarray(ff, np.float32), np.ascontiguousarray(cf, np.float32)
    out = np.zeros(len(ff), np.uint16)
    hw.emu_pixel_weight(keep.ctypes.data, scale, ff.ctypes.data, cf.ctypes.data, len(ff), out.ctypes.data)
    return out


# ------------------------------------------------------------------------------------------------ the rule
def test_rule_specials_and_ties(hw):
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    cf = np.array([0.5, 1.5, 2.5, 65534.5, 65533.5, 65535, 65535.5, 65536, 1e30, inf, -inf, nan, -1, -0.0, 0, 1e-30,
                   0.49999997, 0.50000006, 3.0, 7.5], np.float32)
    want = [0, 2, 2, 65534, 65534, 65535, 65535, 65535, 65535, 65535, 0, 0, 0, 0, 0, 0, 0, 1, 3, 8]
    ones = np.ones(len(cf), np.float32)
    got = _rule(hw, np.ones(len(cf)), 1.0, ones, cf)
    assert got.tolist() == want
    assert np.array_equal(got, W.rule(np.ones(len(cf)), 1.0, ones, cf))
    assert not _rule(hw, np.zeros(len(cf)), 1.0, ones, cf).any()                 # a mask of 0 wins over every x
    nanf = np.full(len(cf), nan, np.float32)
    assert not _rule(hw, np.ones(len(cf)), 1.0, nanf, cf).any()


def test_rule_equals_the_oracle_on_random_factors(hw):
    rng = np.random.default_rng(1)
    n = 200000
    ff = (rng.random(n) * 3).astype(np.float32)
    cf = np.exp(rng.normal(0, 4, n)).astype(np.float32)
    cf[rng.random(n) < 0.01] = np.nan
    cf[rng.random(n) < 0.01] = -cf[:1000].mean()
    ff[rng.random(n) < 0.005] = np.inf
    keep = rng.random(n) < 0.9
    for scale in (1.0, 0.37, 917.5, 65535.0):
        got = _rule(hw, keep, scale, ff, cf)
        assert np.array_equal(got, W.rule(keep, scale, ff, cf)), scale
    ties = (np.arange(0, 65536) + 0.5).astype(np.float32)                      # every tie in range, exactly representable
    ones = np.ones(len(ties), np.float32)
    assert np.array_equal(_rule(hw, ones, 1.0, ones, ties), W.rule(ones, 1.0, ones, ties))


@pytest.mark.parametrize("ncam,ncls,with_ff,with_cf,with_masks", [
    (1, 0, False, False, False), (2, 12, True, True, True), (4, 5, True, False, True), (3, 25, False, True, True)])
def test_frame_set_weights_equal_the_oracle(ncam, ncls, with_ff, with_cf, with_masks, hw):
    """pinhole and fisheye cameras with masks, labels in [-1, 20) against C classes (so some fall outside), factors
    with NaN, +-Inf, negatives and 0."""
    rng = np.random.default_rng(ncam * 10 + ncls)
    fs = O.random_frame_set(rng, 30, O.random_cameras(rng, ncam))
    F = len(fs["frame_cam"])
    ff = (rng.random(F) * 2).astype(np.float32) if with_ff else None
    if ff is not None:
        ff[:4] = [np.nan, np.inf, -1.0, 0.0]
    cf = (rng.random(ncls + 1) * 3).astype(np.float32) if with_cf else None
    if cf is not None:
        cf[1:4] = [np.nan, -np.inf, 0.0]
        cf[-1] = np.inf
    masks = [(rng.random((H, Wd)) < 0.7).astype(np.uint8) * rng.integers(1, 256) if k != 1 else None
             for k, (_, H, Wd, _) in enumerate(fs["cams"])] if with_masks else None
    scale = float(np.float32(rng.random() * 40000 + 1))
    got = W.host_weights(hw, fs, scale, ncls, ff, cf, masks)
    want = W.frame_set_weights(fs, scale, ncls, ff, cf, masks)
    assert np.array_equal(got, want)
    assert (got > 0).any() and ((got == 0).any() or not (with_ff or with_cf or with_masks))


def test_a_malformed_frame_table_is_clamped(hw):
    """A frame whose range is longer than its camera's H W gets weight 0 past them; ranges past P are cut; pixels no
    frame names are left as they were."""
    a = _capi.PnrPixelWeightsArgs()
    fc, off = np.array([0, 0, 5], np.int32), np.array([2, 6, 14, 99], np.int64)
    out = np.full(16, 7, np.uint16)
    a.frame_cam, a.pix_offset, a.F, a.P = fc.ctypes.data, off.ctypes.data, 3, 16
    a.cams[0].model, a.cams[0].H, a.cams[0].W, a.num_cameras = 0, 2, 3, 1
    a.scale, a.weight = 3.0, out.ctypes.data
    hw.emu_pixel_weights(C.byref(a))
    assert out.tolist() == [7, 7] + [3] * 4 + [3] * 6 + [0] * 2 + [3, 3]


# ------------------------------------------------------------------------------------------------ the weighted pick
def _tables():
    rng = np.random.default_rng(7)
    out = []
    for P in (1, 31, 32, 33, 64, 95, 1000, 4097):
        out.append((f"random-{P}", rng.integers(0, 65536, P)))
    z = rng.integers(0, 9, 32 * 7 + 5)
    z[32:96] = 0                                                              # whole groups of zeros
    z[-5:] = [0, 3, 0, 0, 2]                                                  # a partial last group
    out.append(("zero-groups", z))
    for P, at in ((1, 0), (33, 32), (64, 0), (1000, 517)):
        one = np.zeros(P, np.int64)
        one[at] = 9
        out.append((f"single-{P}-{at}", one))
    out.append(("max-77", np.full(77, 65535)))
    out.append(("ones-100", np.ones(100)))
    for P in rng.integers(2, 3000, 4):
        w = rng.integers(0, 65536, int(P)) * (rng.random(int(P)) < 0.3)
        w[int(rng.integers(0, P))] = 1
        out.append((f"sparse-{P}", w))
    return out


@pytest.mark.parametrize("name,w", _tables(), ids=[n for n, _ in _tables()])
def test_weighted_pick_equals_searchsorted(name, w, hw):
    w = np.ascontiguousarray(w, np.uint16)
    cum = np.ascontiguousarray(W.groups(w))
    S = W.cumsum(w)
    T = int(S[-1])
    xs = {0, T - 1} | {int(v) for v in S[S > 0] - 1} | {int(v) for v in S[S < T]}
    xs |= {int(v) for v in np.random.default_rng(len(w)).integers(0, T, 500)}
    xs = np.array(sorted(xs), np.uint64)
    got = np.array([hw.emu_weighted_pixel(w.ctypes.data, cum.ctypes.data, len(w), int(x)) for x in xs])
    want = W.pick(w, xs)
    assert np.array_equal(got, want)
    assert (w[got] > 0).all()
    if np.count_nonzero(w) == 1:
        assert (got == np.flatnonzero(w)[0]).all()


@pytest.mark.parametrize("F,ncam,N,Ni,sparse", [(1, 1, 1, 0, False), (9, 2, 16, 8, True), (40, 4, 3, 61, False),
                                                (120, 3, 64, 128, True)])
def test_weighted_batch_equals_the_oracle(F, ncam, N, Ni, sparse, hw, emu):
    rng = np.random.default_rng(F + ncam)
    fs = O.random_frame_set(rng, F, O.random_cameras(rng, ncam, tiny=ncam == 4))
    P = int(fs["pix_offset"][-1])
    w = rng.integers(0, 65536, P).astype(np.uint16)
    if sparse:
        w[rng.random(P) < 0.9] = 0
        w[0] = 0
        w[-1] = 5
    seed, step = int(rng.integers(0, 1 << 63)), (1 << 35) + F
    for r0, r1 in ((0, 500), ((1 << 32) - 300, 1 << 32)):
        got = W.host_weighted_batch(hw, fs, w, seed, step, r0, r1, N, Ni)
        r = np.arange(r0, r1, dtype=np.int64)
        p = W.weighted_pixels(seed, step, r, w)
        assert np.array_equal(got["pixel"], p)
        assert (w[p] > 0).all()
        T, nz = int(W.cumsum(w)[-1]), int(np.count_nonzero(w))
        assert np.array_equal(got["importance"].view(np.uint32), W.importance(T, nz, w[p]).view(np.uint32))
        f = O.frame_of(fs["pix_offset"], p)
        assert np.array_equal(got["rgb"].view(np.uint32),
                              (fs["rgb8"][p].astype(np.float32) / np.float32(255.0)).view(np.uint32))
        assert np.array_equal(got["depth"].view(np.uint32), fs["depth"][p].view(np.uint32))
        assert np.array_equal(got["pseudo_label"], fs["label"][p].astype(np.int32))
        u, uf = O.jitter(seed, step, r, N, Ni)
        assert np.array_equal(got["u"].view(np.uint32), u.view(np.uint32))
        assert np.array_equal(got["u_fine"].view(np.uint32), uf.view(np.uint32))
        for fi in np.unique(f):
            rays = O.host_frame_rays(emu, fs, fi)
            sel = f == fi
            assert np.array_equal(got["rays"][sel].view(np.uint32), rays[p[sel] - fs["pix_offset"][fi]].view(np.uint32))


def test_all_ones_weights_give_the_unweighted_batch(hw, emu):
    rng = np.random.default_rng(3)
    fs = O.random_frame_set(rng, 50, O.random_cameras(rng, 4, tiny=True))
    P = int(fs["pix_offset"][-1])
    for seed, step, r0, r1 in ((5, 9, 0, 3000), (2 ** 63 + 1, 2 ** 40, 1 << 31, (1 << 31) + 700)):
        got = W.host_weighted_batch(hw, fs, np.ones(P, np.uint16), seed, step, r0, r1, 20, 12)
        want = O.host_batch(emu, fs, seed, step, r0, r1, 20, 12)
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), k
        assert (got["importance"] == 1.0).all()


def test_chi_square_of_weighted_draws(hw):
    """2^20 draws over 1000 pixels (a tenth of them 0) at a fixed seed: counts against weight / T."""
    from scipy.stats import chisquare
    rng = np.random.default_rng(11)
    cams = [(0, 10, 100, [50.0, 50.0, 50.0, 5.0])]
    fs = dict(c2w=np.eye(3, 4, dtype=np.float32).reshape(1, 12), frame_cam=np.zeros(1, np.int32),
              pix_offset=np.array([0, 1000], np.int64), rgb8=rng.integers(0, 256, (1000, 3)).astype(np.uint8),
              label=None, depth=None, cams=cams)
    w = rng.integers(1, 200, 1000).astype(np.uint16)
    w[rng.random(1000) < 0.1] = 0
    w[:3] = [65535, 1, 0]
    R = 1 << 20
    got = W.host_weighted_batch(hw, fs, w, 20240601, 3, 0, R, 1, 0)
    counts = np.bincount(got["pixel"], minlength=1000)
    assert (counts[w == 0] == 0).all()
    live = w > 0
    expected = w[live].astype(np.float64) / float(w.sum()) * R
    assert chisquare(counts[live], expected).pvalue > 1e-3
    # the importance-weighted count of every pixel estimates the uniform share over the unmasked pixels
    imp = got["importance"].astype(np.float64)
    assert abs(imp.mean() - 1.0) < 0.01


# ------------------------------------------------------------------------------------------------ ABI
def _layout(tmp_path, struct, cls, extra=""):
    fields = [f for f, _ in cls._fields_]
    src = tmp_path / f"{struct}.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof({struct}, {f}));\n' for f in fields)
                   + f'  printf("%zu\\n", sizeof({struct}));\n  return 0;\n}}\n')
    exe = tmp_path / struct
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    return got, [getattr(cls, f).offset for f in fields] + [C.sizeof(cls)]


@pytest.mark.parametrize("struct,cls", [("pnr_ray_batch_weights", _capi.PnrRayBatchWeights),
                                        ("pnr_pixel_weights_args", _capi.PnrPixelWeightsArgs)])
def test_args_layout_matches_the_header(struct, cls, tmp_path):
    got, want = _layout(tmp_path, struct, cls)
    assert got == want


# ------------------------------------------------------------------------------------------------ refusals
def _lib():
    import __graft_entry__ as g
    g.build()
    return _capi.lib()


def _batch_args():
    a = _capi.PnrRayBatchArgs()
    a.c2w = a.frame_cam = a.pix_offset = a.rgb8 = 4096
    a.F, a.P = 2, 10
    a.cams[0].model, a.cams[0].H, a.cams[0].W = 0, 1, 5
    a.num_cameras = 1
    a.r0, a.r1, a.N, a.Ni = 0, 8, 16, 8
    a.rays = a.rgb = a.u = a.u_fine = 8192
    return a, _capi.PnrRayBatchWeights(12288, 16384, 40, 7, None)


BATCH_REFUSALS = [
    ("weight", lambda a, w: setattr(w, "weight", None), "null weight table"),
    ("weight_cum", lambda a, w: setattr(w, "weight_cum", None), "null weight table"),
    ("total", lambda a, w: setattr(w, "weight_total", 0), "weight_total=0"),
    ("nonzero", lambda a, w: setattr(w, "weight_nonzero", 0), "weight_nonzero=0 outside [1, P=10]"),
    ("nonzero", lambda a, w: setattr(w, "weight_nonzero", 11), "weight_nonzero=11 outside [1, P=10]"),
    ("total", lambda a, w: setattr(w, "weight_total", 6), "weight_total=6 outside"),
    ("total", lambda a, w: setattr(w, "weight_total", 65535 * 7 + 1), "weight_total=458746 outside"),
    ("F", lambda a, w: setattr(a, "F", 0), "F=0"),                         # the unweighted call's checks apply too
    ("equirect", lambda a, w: setattr(a.cams[0], "model", 1), "equirect"),
    ("u_fine", lambda a, w: setattr(a, "u_fine", None), "u_fine with Ni=8"),
]


@pytest.mark.parametrize("what,breaks,msg", BATCH_REFUSALS, ids=[f"{w}-{i}" for i, (w, _, _) in enumerate(BATCH_REFUSALS)])
def test_weighted_batch_refuses_before_any_device_call(what, breaks, msg):
    L = _lib()
    a, w = _batch_args()
    breaks(a, w)
    assert L.pnr_sample_ray_batch_weighted(C.byref(a), C.byref(w), None) == -1, what
    text = L.pnr_last_error().decode()
    assert "pnr_sample_ray_batch_weighted:" in text and msg in text, text
    a, w = _batch_args()
    assert L.pnr_sample_ray_batch_weighted(C.byref(a), None, None) == -1
    assert "null weights" in L.pnr_last_error().decode()
    assert L.pnr_sample_ray_batch_weighted(None, C.byref(w), None) == -1


def _weights_args():
    a = _capi.PnrPixelWeightsArgs()
    a.frame_cam, a.pix_offset, a.F, a.P = 4096, 8192, 2, 10
    a.cams[0].model, a.cams[0].H, a.cams[0].W = 2, 1, 5
    a.num_cameras = 1
    a.scale, a.weight = 1.0, 12288
    return a


WEIGHT_REFUSALS = [
    ("F", lambda a: setattr(a, "F", 0), "F=0"),
    ("P", lambda a: setattr(a, "P", 0), "P=0"),
    ("C", lambda a: setattr(a, "C", -1), "C=-1"),
    ("C", lambda a: setattr(a, "C", 32768), "C=32768"),
    ("num_cameras", lambda a: setattr(a, "num_cameras", 5), "num_cameras=5"),
    ("equirect", lambda a: setattr(a.cams[0], "model", 1), "equirect"),
    ("frame_cam", lambda a: setattr(a, "frame_cam", None), "null pointer"),
    ("pix_offset", lambda a: setattr(a, "pix_offset", None), "null pointer"),
    ("weight", lambda a: setattr(a, "weight", None), "null pointer"),
    ("scale", lambda a: setattr(a, "scale", 0.0), "scale=0"),
    ("scale", lambda a: setattr(a, "scale", float("inf")), "scale=inf"),
    ("scale", lambda a: setattr(a, "scale", float("nan")), "scale=nan"),
]


@pytest.mark.parametrize("what,breaks,msg", WEIGHT_REFUSALS, ids=[f"{w}-{i}" for i, (w, _, _) in enumerate(WEIGHT_REFUSALS)])
def test_pixel_weights_refuses_before_any_device_call(what, breaks, msg):
    L = _lib()
    a = _weights_args()
    breaks(a)
    assert L.pnr_pixel_weights(C.byref(a), None) == -1, what
    text = L.pnr_last_error().decode()
    assert "pnr_pixel_weights" in text and msg in text, text
    assert L.pnr_pixel_weights(None, None) == -1


def test_cdf_and_counts_refuse_before_any_device_call():
    L = _lib()
    need = L.pnr_pixel_cdf_workspace_bytes(100000)
    assert need == 4 * 16 and L.pnr_pixel_cdf_workspace_bytes(0) == 0 and L.pnr_pixel_cdf_workspace_bytes(1 << 47) == 0
    cases = [((4096, 0, 8192, 8192, 8192, need), "P=0"), ((4096, 1 << 47, 8192, 8192, 8192, need), "outside [1, 2^47)"),
             ((None, 100000, 8192, 8192, 8192, need), "null pointer"), ((4096, 100000, None, 8192, 8192, need), "null"),
             ((4096, 100000, 8192, None, 8192, need), "null"), ((4098, 100000, 8192, 8192, 8192, need), "16-byte"),
             ((4096, 100000, 8192, 8192, None, need), "workspace"), ((4096, 100000, 8192, 8192, 8192, need - 1), "workspace"),
             ((4096, 100000, 8192, 8192, 8200, need), "workspace")]
    for args, msg in cases:
        assert L.pnr_pixel_cdf(*args, None) == -1, msg
        text = L.pnr_last_error().decode()
        assert "pnr_pixel_cdf" in text and msg in text, text
    for args, msg in (((4096, 0, 3, 8192), "P=0"), ((4096, 10, -1, 8192), "C=-1"), ((4096, 10, 8192, 8192), "C=8192"),
                      ((None, 10, 3, 8192), "null pointer"), ((4096, 10, 3, None), "null pointer")):
        assert L.pnr_label_counts(*args, None) == -1, msg
        text = L.pnr_last_error().decode()
        assert "pnr_label_counts" in text and msg in text, text


def test_python_refusals_by_name(tmp_path):
    """pixel_weights, RaySampler and the KITTI-360 mask reader refuse by name before any device work (a CPU set)."""
    import cv2
    from panopticnerf_b200.lib.datasets.kitti360 import load_camera_mask
    from panopticnerf_b200.lib.datasets.ray_batch import (Camera, FrameSet, PixelWeights, RaySampler,
                                                          pixel_weights, sample_ray_batch)
    cams = [Camera("pinhole", 2, 3, (1, 1, 1, 1)), Camera("fisheye", 4, 5, (1, 1, 2, 2, 1.2, 0.0, 0.0))]
    fs = FrameSet.from_images(cams, [0, 1], np.stack([np.eye(3, 4)] * 2),
                              [torch.zeros(2, 3, 3, dtype=torch.uint8), torch.zeros(4, 5, 3, dtype=torch.uint8)],
                              device="cpu")
    with pytest.raises(ValueError, match="needs a label table"):
        pixel_weights(fs, class_alpha=0.5)
    with pytest.raises(ValueError, match="the mask of camera 1 is \\(5, 4\\)"):
        pixel_weights(fs, camera_masks=[None, torch.ones(5, 4, dtype=torch.bool)])
    with pytest.raises(ValueError, match="the mask of camera 0 is .* torch.float32"):
        pixel_weights(fs, camera_masks=[torch.ones(2, 3), None])
    with pytest.raises(ValueError, match="1 camera masks for 2 cameras"):
        pixel_weights(fs, camera_masks=[None])
    with pytest.raises(ValueError, match="total is 0"):
        pixel_weights(fs, unlabelled=0.0)
    with pytest.raises(ValueError, match="class_alpha=-1"):
        pixel_weights(fs, class_alpha=-1)
    with pytest.raises(ValueError, match="expected \\[P\\] torch.uint16"):
        PixelWeights.from_weight(torch.zeros(4, dtype=torch.int16))
    bad = PixelWeights(torch.zeros(7, dtype=torch.uint16), torch.zeros(1, dtype=torch.uint64), 1, 1)
    with pytest.raises(ValueError, match="the weight table has \\(7,\\) entries, the frame set 26 pixels"):
        RaySampler(fs, 0, weights=bad)
    with pytest.raises(ValueError, match="the weight table has \\(7,\\) entries"):
        sample_ray_batch(fs, 0, 0, 0, 4, 8, weights=bad)
    with pytest.raises(ValueError, match="per-ray keys"):
        RaySampler(fs, 0, scene={"importance": torch.zeros(1)})
    cam = cams[1]
    p = tmp_path / "m.png"
    with pytest.raises(FileNotFoundError, match="m.png: missing"):
        load_camera_mask(p, cam)
    cv2.imwrite(str(p), np.zeros((4, 5), np.uint16))
    with pytest.raises(ValueError, match="must be 8-bit"):
        load_camera_mask(p, cam)
    cv2.imwrite(str(p), np.zeros((4, 5, 3), np.uint8))
    with pytest.raises(ValueError, match="must have 1 channel"):
        load_camera_mask(p, cam)
    cv2.imwrite(str(p), np.zeros((5, 4), np.uint8))
    with pytest.raises(ValueError, match="the mask is 4 x 5, its camera is 5 x 4"):
        load_camera_mask(p, cam)
    m = (np.arange(20).reshape(4, 5) % 3 == 0).astype(np.uint8) * 255
    cv2.imwrite(str(p), m)
    got = load_camera_mask(p, cam)
    assert got.dtype == torch.uint8 and np.array_equal(got.numpy(), m)


# ------------------------------------------------------------------------------------------------ sharding
@pytest.mark.parametrize("R,world", [(10, 3), (11, 4), (0, 2)])
def test_sharder_slices_importance_with_the_rays(R, world):
    b = {"rays": torch.arange(R * 6, dtype=torch.float32).reshape(R, 6), "importance": torch.arange(R) * 0.5,
         "scene_aabb": torch.zeros(6)}
    parts = [parallel.shard_training_batch(b, r, world) for r in range(world)]
    for r, s in enumerate(parts):
        lo, hi = parallel.shard_range(R, r, world)
        assert torch.equal(s["importance"], b["importance"][lo:hi]) and s["scene_aabb"] is b["scene_aabb"]
    assert torch.equal(torch.cat([s["importance"] for s in parts]), b["importance"])
    b["importance"] = b["importance"][:max(R - 1, 0)] if R else torch.zeros(1)
    with pytest.raises(ValueError, match="importance"):
        parallel.shard_training_batch(b, 0, world)
