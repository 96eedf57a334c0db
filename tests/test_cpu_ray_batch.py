"""CPU tier of training ray batches: the numpy Philox4x32-10 against Random123's known answers; the host build of
pnr_ray_batch_row (tests/host_emu.cpp) against the numpy oracle bit for bit (pixels, frames, colours,
targets, u, u_fine, and rays against the host build of pnr_generate_rays); the 64-bit multiply-high; the KITTI-360
frame reader on fixtures written here in the documented layouts, and each refusal by name; the argument refusals of
pnr_sample_ray_batch before any device call; and pnr_ray_batch_args' layout against a C compile of include/pnr.h."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_ray_batch as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h)
from panopticnerf_b200 import _capi

ROOT = Path(__file__).resolve().parent.parent


# ------------------------------------------------------------------------------------------------ Philox
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want, emu):
    got = [int(x) for x in O.philox4x32_10(*ctr, *key)]
    assert got == list(want)
    c, k, out = (C.c_uint32 * 4)(*ctr), (C.c_uint32 * 2)(*key), (C.c_uint32 * 4)()
    emu.emu_philox4x32_10(c, k, out)
    assert list(out) == list(want)


@pytest.mark.parametrize("P", [1, 2, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, 1 << 40, (1 << 31) + 3, (1 << 62) + 7])
def test_mulhi64(P, emu):
    rng = np.random.default_rng(P % 1000)
    xs = [0, 1, (1 << 32) - 1, 1 << 32, (1 << 63), (1 << 64) - 1] + [int(v) for v in rng.integers(0, 1 << 63, 64)]
    for x in xs:
        want = (x * P) >> 64
        assert emu.emu_mulhi64(x, P) == want
        assert 0 <= want < P
    assert emu.emu_mulhi64((1 << 64) - 1, P) == P - 1


# ------------------------------------------------------------------------------------------------ host build vs oracle
def _check_rows(emu, fs, seed, step, r0, r1, N, Ni):
    got = O.host_batch(emu, fs, seed, step, r0, r1, N, Ni)
    r = np.arange(r0, r1, dtype=np.int64)
    off, P = fs["pix_offset"], int(fs["pix_offset"][-1])
    p = O.pixels(seed, step, r, P)
    assert np.array_equal(got["pixel"], p)
    f = O.frame_of(off, p)
    assert ((f >= 0) & (f < len(fs["frame_cam"]))).all()
    assert ((off[f] <= p) & (p < off[f + 1])).all()
    assert np.array_equal(got["rgb"].view(np.uint32),
                          (fs["rgb8"][p].astype(np.float32) / np.float32(255.0)).view(np.uint32))
    want_d = fs["depth"][p] if fs["depth"] is not None else np.zeros(len(p), np.float32)
    want_l = fs["label"][p].astype(np.int32) if fs["label"] is not None else np.full(len(p), -1, np.int32)
    assert np.array_equal(got["depth"].view(np.uint32), want_d.view(np.uint32))
    assert np.array_equal(got["pseudo_label"], want_l)
    u, uf = O.jitter(seed, step, r, N, Ni)
    assert np.array_equal(got["u"].view(np.uint32), u.view(np.uint32))
    assert np.array_equal(got["u_fine"].view(np.uint32), uf.view(np.uint32))
    for fi in np.unique(f):
        rays = O.host_frame_rays(emu, fs, fi)
        sel = f == fi
        assert np.array_equal(got["rays"][sel].view(np.uint32), rays[p[sel] - off[fi]].view(np.uint32))
    return got, f


@pytest.mark.parametrize("F,ncam,N,Ni,label,depth", [
    (1, 1, 1, 0, False, False), (3, 2, 64, 128, True, True), (17, 4, 7, 5, True, False), (60, 3, 32, 0, False, True),
    (200, 4, 3, 253, True, True)])
def test_host_build_equals_the_oracle(F, ncam, N, Ni, label, depth, emu):
    rng = np.random.default_rng(F * 7 + ncam)
    fs = O.random_frame_set(rng, F, O.random_cameras(rng, ncam, tiny=ncam == 4), label, depth)
    seed, step = int(rng.integers(0, 1 << 63)) * 2 + 1, (1 << 33) + F
    _check_rows(emu, fs, seed, step, 0, 700, N, Ni)
    _check_rows(emu, fs, seed, step, 1 << 31, (1 << 31) + 100, N, Ni)   # ray indices past int32: 32-bit words


def test_frame_boundaries_and_one_pixel_frames(emu):
    """A set of one-pixel frames between larger ones: every frame, its first and its last pixel are drawn, and each
    sits in the frame that owns it."""
    rng = np.random.default_rng(5)
    cams = [(0, 1, 1, [1.0, 1.0, 0.0, 0.0]), (2, 3, 4, [2.0, 2.0, 1.5, 1.0, 0.9, 0.01, 0.0]),
            (0, 2, 5, [3.0, 3.0, 2.0, 1.0])]
    fs = O.random_frame_set(rng, 24, cams)
    fs["frame_cam"][::3] = 0                                               # one-pixel frames, some adjacent
    fs["frame_cam"][1:3] = 0
    sizes = [cams[c][1] * cams[c][2] for c in fs["frame_cam"]]
    fs["pix_offset"] = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    P = int(fs["pix_offset"][-1])
    fs["rgb8"], fs["label"], fs["depth"] = fs["rgb8"][:P], fs["label"][:P], fs["depth"][:P]
    got, f = _check_rows(emu, fs, 11, 3, 0, 4000, 4, 4)
    assert set(f.tolist()) == set(range(24))
    assert {int(x) for x in fs["pix_offset"][:-1]} <= set(got["pixel"].tolist())
    assert {int(x) - 1 for x in fs["pix_offset"][1:]} <= set(got["pixel"].tolist())


def test_a_range_is_the_rows_of_the_whole_batch(emu):
    rng = np.random.default_rng(9)
    fs = O.random_frame_set(rng, 12, O.random_cameras(rng, 2))
    whole = O.host_batch(emu, fs, 3, 4, 0, 600, 10, 6)
    part = O.host_batch(emu, fs, 3, 4, 255, 513, 10, 6)
    for k in whole:
        assert np.array_equal(part[k], whole[k][255:513]), k
    other = O.host_batch(emu, fs, 3, 5, 0, 600, 10, 6)                  # another step draws other pixels
    assert not np.array_equal(other["pixel"], whole["pixel"])


# ------------------------------------------------------------------------------------------------ argument refusals
def _valid_args():
    """Arguments that pass every check (never launched: each test breaks one of them first).  Pointers are dummies."""
    a = _capi.PnrRayBatchArgs()
    a.c2w = a.frame_cam = a.pix_offset = a.rgb8 = 4096
    a.F, a.P = 2, 10
    a.cams[0].model, a.cams[0].H, a.cams[0].W = 0, 1, 5
    a.num_cameras = 1
    a.r0, a.r1, a.N, a.Ni = 0, 8, 16, 8
    a.rays = a.rgb = a.u = a.u_fine = 8192
    return a


REFUSALS = [
    ("F", lambda a: setattr(a, "F", 0), "F=0"),
    ("F", lambda a: setattr(a, "F", 2 ** 31 - 1), "F=2147483647"),
    ("P", lambda a: setattr(a, "P", 0), "P=0"),
    ("range", lambda a: setattr(a, "r0", -1), "range"),
    ("range", lambda a: (setattr(a, "r0", 9)), "range"),
    ("range", lambda a: setattr(a, "r1", (1 << 32) + 1), "range"),
    ("N", lambda a: setattr(a, "N", 0), "N=0"),
    ("N", lambda a: setattr(a, "N", 257), "N=257"),
    ("Ni", lambda a: setattr(a, "Ni", -1), "Ni=-1"),
    ("Ni", lambda a: setattr(a, "Ni", 241), "Ni=241"),
    ("num_cameras", lambda a: setattr(a, "num_cameras", 0), "num_cameras=0"),
    ("num_cameras", lambda a: setattr(a, "num_cameras", 5), "num_cameras=5"),
    ("equirect", lambda a: setattr(a.cams[0], "model", 1), "equirect"),
    ("model", lambda a: setattr(a.cams[0], "model", 3), "model 3"),
    ("size", lambda a: setattr(a.cams[0], "H", 0), "size"),
    ("size", lambda a: (setattr(a, "num_cameras", 2), setattr(a.cams[1], "W", -4)), "camera 1 size"),
    ("c2w", lambda a: setattr(a, "c2w", None), "frame-set pointer"),
    ("frame_cam", lambda a: setattr(a, "frame_cam", None), "frame-set pointer"),
    ("pix_offset", lambda a: setattr(a, "pix_offset", None), "frame-set pointer"),
    ("rgb8", lambda a: setattr(a, "rgb8", None), "frame-set pointer"),
    ("rays", lambda a: setattr(a, "rays", None), "output pointer"),
    ("rgb", lambda a: setattr(a, "rgb", None), "output pointer"),
    ("u", lambda a: setattr(a, "u", None), "output pointer"),
    ("u_fine", lambda a: setattr(a, "u_fine", None), "u_fine with Ni=8"),
]


@pytest.mark.parametrize("what,breaks,msg", REFUSALS, ids=[f"{w}-{i}" for i, (w, _, _) in enumerate(REFUSALS)])
def test_sample_ray_batch_refuses_before_any_device_call(what, breaks, msg):
    import __graft_entry__ as g
    g.build()
    a = _valid_args()
    breaks(a)
    rc = _capi.lib().pnr_sample_ray_batch(C.byref(a), None)
    assert rc == -1, what
    text = _capi.lib().pnr_last_error().decode()
    assert "pnr_sample_ray_batch" in text and msg in text, text
    assert _capi.lib().pnr_sample_ray_batch(None, None) == -1


def test_args_layout_matches_the_header(tmp_path):
    """offsetof / sizeof of pnr_ray_batch_args and pnr_ray_camera from a C compile of include/pnr.h equal ctypes'."""
    fields = [f for f, _ in _capi.PnrRayBatchArgs._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(pnr_ray_batch_args, {f}));\n' for f in fields)
                   + '  printf("%zu\\n%zu\\n", sizeof(pnr_ray_batch_args), sizeof(pnr_ray_camera));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    want = [getattr(_capi.PnrRayBatchArgs, f).offset for f in fields] + [C.sizeof(_capi.PnrRayBatchArgs),
                                                                         C.sizeof(_capi.PnrRayCamera)]
    assert got == want


# ------------------------------------------------------------------------------------------------ KITTI-360 frames
def _write_sequence(root, seq="2013_05_28_drive_0000_sync", frames=(3, 4), H=6, W=8, seed=0):
    """A tiny sequence in the KITTI-360 layout: perspective + fisheye calibration, poses, colour images, 8-bit pseudo
    labels, 16-bit depth.  Returns what was written (BGR images, ids, raw depth)."""
    import cv2
    rng = np.random.default_rng(seed)
    cal = root / "calibration"
    cal.mkdir(parents=True)
    (cal / "perspective.txt").write_text(f"P_rect_00: 5.0 0 3.5 0 0 6.0 2.5 0 0 0 1 0\nS_rect_00: {W} {H}\n")
    (cal / "image_02.yaml").write_text(
        "%%YAML:1.0\n---\nmodel_type: MEI\ncamera_name: image_02\nimage_width: %d\nimage_height: %d\n"
        "mirror_parameters:\n   xi: 1.5\ndistortion_parameters:\n   k1: 0.02\n   k2: 0.01\n   p1: 0.0\n   p2: 0.0\n"
        "projection_parameters:\n   gamma1: 4.0\n   gamma2: 4.5\n   u0: 3.0\n   v0: 2.0\n" % (W, H))
    (cal / "calib_cam_to_pose.txt").write_text("image_02: 0 0 1 0.5 -1 0 0 0.1 0 -1 0 0.2\n")
    poses = root / "data_poses" / seq
    poses.mkdir(parents=True)
    c0 = [np.concatenate([np.eye(3) * (1 + 0.1 * f), [[f], [2 * f], [0.5]]], 1) for f in frames]
    (poses / "cam0_to_world.txt").write_text("".join(
        f"{f} " + " ".join(str(x) for x in np.vstack([m, [0, 0, 0, 1]]).reshape(-1)) + "\n" for f, m in zip(frames, c0)))
    (poses / "poses.txt").write_text("".join(
        f"{f} " + " ".join(str(x) for x in m.reshape(-1)) + "\n" for f, m in zip(frames, c0)))
    written = {"bgr": [], "ids": [], "depth": []}
    for cam, sub in (("image_00", "data_rect"), ("image_02", "data_rgb")):
        d = root / "data_2d_raw" / seq / cam / sub
        d.mkdir(parents=True)
        for f in frames:
            bgr = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
            cv2.imwrite(str(d / f"{f:010d}.png"), bgr)
            if cam == "image_00":
                written["bgr"].append(bgr)
    for sub in ("pseudo", "depth"):
        (root / sub).mkdir()
    for f in frames:
        ids = rng.integers(0, 50, (H, W)).astype(np.uint8)
        dep = np.where(rng.random((H, W)) < 0.5, rng.integers(1, 65535, (H, W)), 0).astype(np.uint16)
        cv2.imwrite(str(root / "pseudo" / f"{f:010d}.png"), ids)
        cv2.imwrite(str(root / "depth" / f"{f:010d}.png"), dep)
        written["ids"].append(ids)
        written["depth"].append(dep)
    return seq, list(frames), written, c0


def test_load_frames_reads_the_documented_formats(tmp_path):
    from panopticnerf_b200.lib.datasets.kitti360 import load_frames
    from panopticnerf_b200.lib.datasets.ray_batch import concat_frame_sets
    seq, frames, w, c0 = _write_sequence(tmp_path)
    sem = {7: 0, 8: 1, 11: 2, 26: 3}
    fs = load_frames(tmp_path, seq, frames, pseudo_dir=tmp_path / "pseudo", depth_dir=tmp_path / "depth",
                     sem_to_train=sem, device="cpu")
    assert fs.num_frames == 2 and fs.num_pixels == 2 * 48 and fs.pix_offset.tolist() == [0, 48, 96]
    cam = fs.cameras[0]
    assert (cam.model, cam.H, cam.W, cam.intr) == ("pinhole", 6, 8, (5.0, 6.0, 3.5, 2.5))
    rgb = np.concatenate([b[:, :, ::-1].reshape(-1, 3) for b in w["bgr"]])           # BGR on disk -> RGB
    assert np.array_equal(fs.rgb8.numpy(), rgb)
    ids = np.concatenate([i.reshape(-1) for i in w["ids"]])
    want = np.array([sem.get(int(i), -1) for i in ids], np.int16)
    assert np.array_equal(fs.label.numpy(), want) and (want == -1).any() and (want >= 0).any()
    dep = np.concatenate([d.reshape(-1) for d in w["depth"]])
    assert np.array_equal(fs.depth.numpy(), dep.astype(np.float32) / 256) and (fs.depth == 0).any()
    assert torch.equal(fs.c2w, torch.tensor(np.stack(c0), dtype=torch.float32).reshape(2, 12))
    plain = load_frames(tmp_path, seq, frames[:1], pseudo_dir=tmp_path / "pseudo", device="cpu")   # no table: the ids
    assert np.array_equal(plain.label.numpy(), w["ids"][0].reshape(-1).astype(np.int16)) and plain.depth is None
    fe = load_frames(tmp_path, seq, frames, camera="image_02", device="cpu")
    assert fe.cameras[0].model == "fisheye" and fe.cameras[0].intr == (4.0, 4.5, 3.0, 2.0, 1.5, 0.02, 0.01)
    c2p = np.array([[0, 0, 1, 0.5], [-1, 0, 0, 0.1], [0, -1, 0, 0.2], [0, 0, 0, 1]])
    want_fe = np.stack([(np.vstack([m, [0, 0, 0, 1]]) @ c2p)[:3] for m in c0])
    assert torch.equal(fe.c2w, torch.tensor(want_fe, dtype=torch.float32).reshape(2, 12))
    both = concat_frame_sets(fs, fe, fs)
    assert both.num_frames == 6 and len(both.cameras) == 2 and both.frame_cam.tolist() == [0, 0, 1, 1, 0, 0]
    assert both.pix_offset.tolist() == [0, 48, 96, 144, 192, 240, 288]
    assert (both.label[96:192] == -1).all() and (both.depth[96:192] == 0).all()


def test_load_frames_refuses_by_name(tmp_path):
    import cv2
    from panopticnerf_b200.lib.datasets.kitti360 import load_frames
    seq, frames, _, _ = _write_sequence(tmp_path)
    kw = dict(pseudo_dir=tmp_path / "pseudo", depth_dir=tmp_path / "depth", device="cpu")
    for sub in ("data_2d_raw/" + seq + "/image_00/data_rect", "pseudo", "depth"):
        path = tmp_path / sub / "0000000004.png"
        path.rename(path.with_suffix(".bak"))
        with pytest.raises(FileNotFoundError, match="0000000004.png: missing a"):
            load_frames(tmp_path, seq, frames, **kw)
        path.with_suffix(".bak").rename(path)
    with pytest.raises(ValueError, match="image_01"):
        load_frames(tmp_path, seq, frames, camera="image_01", **kw)
    img = tmp_path / "data_2d_raw" / seq / "image_00" / "data_rect" / "0000000005.png"
    cv2.imwrite(str(img), np.zeros((6, 8, 3), np.uint8))
    with pytest.raises(ValueError, match="no pose for frame 5"):
        load_frames(tmp_path, seq, [5], **kw)
    lab, dep = tmp_path / "pseudo" / "0000000003.png", tmp_path / "depth" / "0000000004.png"
    cv2.imwrite(str(lab), np.zeros((6, 8), np.uint16))
    with pytest.raises(ValueError, match="pseudo-label image must be 8-bit"):
        load_frames(tmp_path, seq, frames, **kw)
    cv2.imwrite(str(lab), np.zeros((6, 8, 3), np.uint8))
    with pytest.raises(ValueError, match="pseudo-label image must have 1 channel"):
        load_frames(tmp_path, seq, frames, **kw)
    cv2.imwrite(str(lab), np.zeros((6, 8), np.uint8))
    cv2.imwrite(str(dep), np.zeros((6, 8), np.uint8))
    with pytest.raises(ValueError, match="depth image must be 16-bit"):
        load_frames(tmp_path, seq, frames, **kw)
    cv2.imwrite(str(dep), np.zeros((6, 8), np.uint16))
    src = tmp_path / "data_2d_raw" / seq / "image_00" / "data_rect" / "0000000004.png"
    cv2.imwrite(str(src), np.zeros((6, 8), np.uint8))
    with pytest.raises(ValueError, match="colour image must have 3 channel"):
        load_frames(tmp_path, seq, frames, **kw)
    cv2.imwrite(str(src), np.zeros((7, 8, 3), np.uint8))
    with pytest.raises(ValueError, match="the colour image is 8 x 7, its camera's calibration says 8 x 6"):
        load_frames(tmp_path, seq, frames, **kw)
    cv2.imwrite(str(src), np.zeros((6, 8, 3), np.uint8))
    cv2.imwrite(str(dep), np.zeros((6, 9), np.uint16))
    with pytest.raises(ValueError, match="the depth image is 9 x 6"):
        load_frames(tmp_path, seq, frames, **kw)
    cv2.imwrite(str(dep), np.zeros((6, 8), np.uint16))
    assert load_frames(tmp_path, seq, frames, **kw).num_frames == 2


def test_ray_sampler_refuses_bad_inputs():
    from panopticnerf_b200.lib.datasets.ray_batch import Camera, RaySampler, sample_ray_batch
    with pytest.raises(ValueError, match="equirect"):
        Camera("equirect", 4, 8, (1, 1, 1, 1))
    with pytest.raises(ValueError, match="7 intrinsics"):
        Camera("fisheye", 4, 8, (1, 1, 1, 1))
    fs = type("FS", (), {})()
    with pytest.raises(ValueError, match="seed"):
        sample_ray_batch(fs, -1, 0, 0, 4, 8)
    with pytest.raises(ValueError, match="per-ray keys"):
        RaySampler(None, 0, scene={"rays": torch.zeros(1, 6)})
