"""GPU tier of training ray batches (pnr_sample_ray_batch, RaySampler, load_frames): the kernel bit for bit against the
host build of the same per-ray routine, every ray against pnr_generate_rays' row for its pixel, ranges, repeat launches
and processes, a frame set of 2^31 + 3 pixels, uniformity, data-parallel sharding, and training a student from a
sequence written in the KITTI-360 layout."""
import hashlib
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_ray_batch as O
from host_emu import emu  # noqa: F401  (session fixture: the host build of ray_math.h)
import panopticnerf_b200 as PN
from panopticnerf_b200 import parallel, synthetic as S
from panopticnerf_b200.lib.datasets.ray_batch import Camera, FrameSet, RaySampler, sample_ray_batch
from panopticnerf_b200.lib.networks.renderer.panopticnerf_renderer import generate_rays

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = Path(__file__).resolve().parent.parent
MODEL = {0: "pinhole", 2: "fisheye"}


def device_set(fs) -> FrameSet:
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV) if x is not None else None
    cams = [Camera(MODEL[m], H, W, intr) for m, H, W, intr in fs["cams"]]
    return FrameSet(cams, t(fs["c2w"]), t(fs["frame_cam"]), t(fs["pix_offset"]), t(fs["rgb8"]), t(fs["label"]),
                    t(fs["depth"]))


def _same(got: torch.Tensor, want: np.ndarray) -> bool:
    g = got.cpu().numpy()
    return g.shape == want.shape and g.tobytes() == np.ascontiguousarray(want).tobytes()


CASES = [(1, 1, False, False, 1), (1, 2, True, True, 255), (7, 3, True, False, 256), (40, 4, False, True, 257),
         (200, 4, True, True, 1 << 20), (1500, 2, True, True, 4099)]   # F = 1500: offsets searched in global memory


@pytest.mark.parametrize("F,ncam,label,depth,R", CASES)
def test_kernel_equals_the_host_build(F, ncam, label, depth, R, emu):
    rng = np.random.default_rng(F + R)
    fs = O.random_frame_set(rng, F, O.random_cameras(rng, ncam, tiny=ncam >= 3), label, depth)
    N, Ni = (64, 128) if R == 1 << 20 else (int(rng.integers(1, 40)), int(rng.integers(0, 30)))
    seed, step = int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 40))
    got = sample_ray_batch(device_set(fs), seed, step, 0, R, N, Ni, want_pixel=True)
    want = O.host_batch(emu, fs, seed, step, 0, R, N, Ni)
    assert set(got) == {"rays", "rgb", "u", "pixel"} | ({"u_fine"} if Ni else set()) | \
        ({"depth"} if depth else set()) | ({"pseudo_label"} if label else set())
    for k, v in got.items():
        assert _same(v, want[k]), k
    if ncam >= 2:
        models = {fs["cams"][c][0] for c in fs["frame_cam"][O.frame_of(fs["pix_offset"], want["pixel"])]}
        assert models == {0, 2} or R < 300


def test_each_ray_is_the_row_of_generate_rays():
    rng = np.random.default_rng(3)
    fs = O.random_frame_set(rng, 9, O.random_cameras(rng, 4, tiny=True))
    got = sample_ray_batch(device_set(fs), 77, 5, 0, 5000, 8, 0, want_pixel=True)
    p = got["pixel"].cpu().numpy()
    f = O.frame_of(fs["pix_offset"], p)
    for fi in range(9):
        model, H, W, intr = fs["cams"][int(fs["frame_cam"][fi])]
        rows = generate_rays(H, W, intr, torch.from_numpy(fs["c2w"][fi]), MODEL[model], device=DEV).cpu().numpy()
        sel = f == fi
        assert sel.any()
        assert _same(got["rays"][torch.from_numpy(sel).to(DEV)], rows[p[sel] - fs["pix_offset"][fi]])


def test_a_range_equals_the_rows_of_the_whole_batch():
    rng = np.random.default_rng(4)
    d = device_set(O.random_frame_set(rng, 30, O.random_cameras(rng, 2)))
    whole = sample_ray_batch(d, 1, 2, 0, 3000, 16, 32, want_pixel=True)
    for r0, r1 in ((250, 1000), (256 * 3 + 5, 2999), (0, 1), (2999, 3000)):
        part = sample_ray_batch(d, 1, 2, r0, r1, 16, 32, want_pixel=True)
        for k in whole:
            assert torch.equal(part[k], whole[k][r0:r1]), (k, r0, r1)


_DIGEST = """
import hashlib, sys
import numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
import oracle_ray_batch as O
from test_gpu_ray_batch import device_set
from panopticnerf_b200.lib.datasets.ray_batch import sample_ray_batch
rng = np.random.default_rng(12)
fs = O.random_frame_set(rng, 50, O.random_cameras(rng, 3, tiny=True))
out = sample_ray_batch(device_set(fs), 2 ** 63 + 9, 2 ** 32 + 1, 0, 70000, 64, 128, want_pixel=True)
h = hashlib.sha256()
for k in sorted(out):
    h.update(out[k].cpu().numpy().tobytes())
print(h.hexdigest())
"""


def test_two_launches_and_two_processes_give_the_same_bytes():
    code = _DIGEST.format(root=str(ROOT), tests=str(ROOT / "tests"))
    rng = np.random.default_rng(12)
    fs = O.random_frame_set(rng, 50, O.random_cameras(rng, 3, tiny=True))
    d = device_set(fs)
    outs = [sample_ray_batch(d, 2 ** 63 + 9, 2 ** 32 + 1, 0, 70000, 64, 128, want_pixel=True) for _ in range(2)]
    h = hashlib.sha256()
    for k in sorted(outs[0]):
        assert torch.equal(outs[0][k], outs[1][k]), k
        h.update(outs[0][k].cpu().numpy().tobytes())
    other = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=str(ROOT), timeout=600)
    assert other.returncode == 0, other.stderr[-2000:]
    assert other.stdout.split()[-1] == h.hexdigest()


def test_two_to_the_31_plus_3_pixels():
    """A 3-pixel frame, then one of 32768 x 65536 pixels (rgb only, 6.4 GB): the pick over more than 2^31 pixels, the
    offsets past 2^31 and the colour byte offsets past 2^32 go through the 64-bit paths."""
    P = (1 << 31) + 3
    if torch.cuda.mem_get_info(DEV)[0] < 3 * P + (2 << 30):
        pytest.skip("the device lacks the memory for 2^31 + 3 pixels")
    cams = [Camera("pinhole", 1, 3, (2.0, 2.0, 1.0, 0.0)), Camera("pinhole", 32768, 65536, (3e4, 3e4, 32768.5, 16384.25))]
    c2w = np.stack([np.eye(3, 4), np.concatenate([np.eye(3)[[1, 2, 0]], [[1.0], [2.0], [3.0]]], 1)]).astype(np.float32)
    rgb8 = torch.randint(0, 256, (P, 3), dtype=torch.uint8, device=DEV)
    fs = FrameSet(cams, torch.from_numpy(c2w.reshape(2, 12)).to(DEV), torch.tensor([0, 1], dtype=torch.int32, device=DEV),
                  torch.tensor([0, 3, P], dtype=torch.int64, device=DEV), rgb8)
    R = 4096
    got = sample_ray_batch(fs, 99, 7, 0, R, 4, 4, want_pixel=True)
    want = O.pixels(99, 7, np.arange(R), P)
    assert np.array_equal(got["pixel"].cpu().numpy(), want) and (3 * want >= 1 << 32).any()
    # true division, as torch on the CPU (its CUDA kernel multiplies by the reciprocal instead)
    assert torch.equal(got["rgb"].cpu(), rgb8[got["pixel"]].cpu().float() / 255)
    u, uf = O.jitter(99, 7, np.arange(R), 4, 4)
    assert _same(got["u"], u) and _same(got["u_fine"], uf)
    for i in range(0, R, 16):                             # rays: the row of generate_rays that holds the pixel
        q = int(want[i]) - 3
        v, u_ = divmod(q, 65536)
        row = generate_rays(32768, 65536, cams[1].intr, torch.from_numpy(c2w[1]), "pinhole", row0=v, rows=1, device=DEV)
        assert torch.equal(got["rays"][i], row[u_]), i
    del rgb8, fs
    torch.cuda.empty_cache()


def test_draws_are_uniform_over_frames_and_rows():
    """Chi-square at R = 2^22 with a fixed seed: counts per frame, per pixel row and per pixel against the sizes."""
    from scipy.stats import chisquare
    rng = np.random.default_rng(21)
    fs = O.random_frame_set(rng, 37, O.random_cameras(rng, 4, tiny=True), False, False)
    R = 1 << 22
    p = sample_ray_batch(device_set(fs), 2024, 1, 0, R, 1, 0, want_pixel=True)["pixel"].cpu().numpy()
    off = fs["pix_offset"]
    P = int(off[-1])
    f = O.frame_of(off, p)
    sizes = np.diff(off)
    assert chisquare(np.bincount(f, minlength=37), sizes / P * R).pvalue > 1e-3
    W = np.array([fs["cams"][c][2] for c in fs["frame_cam"]])
    row_start = np.concatenate([np.arange(off[i], off[i + 1], W[i]) for i in range(37)])
    rows = np.searchsorted(row_start, p, side="right") - 1
    row_w = np.diff(np.concatenate([row_start, [P]]))
    assert chisquare(np.bincount(rows, minlength=len(row_start)), row_w / P * R).pvalue > 1e-3
    assert chisquare(np.bincount(p, minlength=P), np.full(P, R / P)).pvalue > 1e-3


# ------------------------------------------------------------------------------------------------ data-parallel use
def test_a_sampled_batch_shards_like_a_hand_built_one():
    from test_gpu_data_parallel import _nets, _params, cfg3, simulate_shards
    from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper
    cfg = cfg3("frequency")
    rng = np.random.default_rng(31)
    fs = O.random_frame_set(rng, 6, O.random_cameras(rng, 2))
    scene = {k: v.to(DEV) for k, v in S.make_boxes(64, 45, 64, seed=3).items()}
    scene["scene_aabb"] = torch.tensor(S.SCENE_AABB, dtype=torch.float32, device=DEV)
    sampler = RaySampler(device_set(fs), seed=8, scene=scene)
    batch = sampler.batch(step=3, R=160, N=int(cfg.N_samples), Ni=int(cfg.N_importance))
    again = sampler.batch(step=3, R=160, N=int(cfg.N_samples), Ni=int(cfg.N_importance))
    hand = {k: v.clone() for k, v in batch.items()}
    assert all(torch.equal(batch[k], again[k]) for k in batch)
    assert set(batch) >= {"rays", "rgb", "u", "u_fine", "depth", "pseudo_label", "box_center", "scene_aabb"}
    G = 3
    for g in range(G):
        a, b = parallel.shard_training_batch(batch, g, G), parallel.shard_training_batch(hand, g, G)
        lo, hi = parallel.shard_range(160, g, G)
        for k in batch:
            assert torch.equal(a[k], b[k]), k
            want = batch[k][lo:hi] if k in parallel.TRAIN_RAY_KEYS else batch[k]
            assert torch.equal(a[k], want), k
    net, fine = _nets(cfg, False, seed=51)
    opt = FusedAdam(_params(net, fine))
    res_s, st_s = simulate_shards(cfg, net, fine, batch, G, opt)
    res_h, st_h = simulate_shards(cfg, net, fine, hand, G, opt)
    for (_, la, sa), (_, lb, sb) in zip(res_s, res_h):
        assert torch.equal(la, lb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    assert all(torch.equal(x, y) for x, y in zip(st_s, st_h))
    opt.zero_grad()
    _, loss_w, _, _ = NetworkWrapper(cfg, net, fine)(batch)
    loss_w.backward()
    g_whole, g_sum = opt.flat_grads()[0], st_s[0].sum(0)
    assert float(res_s[-1][1]) == pytest.approx(float(loss_w.detach()), rel=1e-5)
    scale = g_whole.abs().max()
    assert float((g_whole - g_sum).abs().max() / scale) < 1e-4


# ------------------------------------------------------------------------------------------------ end to end
def _write_teacher_sequence(root: Path, cfg, frames, seq="synthetic_drive"):
    """A teacher network's renders of a few poses, written as a KITTI-360 sequence: rectified colour PNGs, 8-bit
    semanticIds (its semantic argmax), 16-bit depth x 256, perspective calibration and cam0_to_world."""
    import cv2
    teacher = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
    ren = PN.make_renderer(cfg, teacher)
    (root / "calibration").mkdir(parents=True)
    (root / "calibration" / "perspective.txt").write_text(
        f"P_rect_00: {cfg.fx} 0 {cfg.cx} 0 0 {cfg.fy} {cfg.cy} 0 0 0 1 0\nS_rect_00: {cfg.W_img} {cfg.H}\n")
    img = root / "data_2d_raw" / seq / "image_00" / "data_rect"
    for d in (img, root / "data_poses" / seq, root / "pseudo", root / "depth"):
        d.mkdir(parents=True)
    lines = []
    H, W = int(cfg.H), int(cfg.W_img)
    for f in frames:
        a = 0.15 * (f - frames[0])
        m = np.array([[np.cos(a), 0, np.sin(a), 0.3 * f], [0, 1, 0, 0.5], [-np.sin(a), 0, np.cos(a), 1.0 + 0.5 * f],
                      [0, 0, 0, 1]])
        lines.append(f"{f} " + " ".join(repr(float(x)) for x in m.reshape(-1)))
        out = ren.render({"c2w": torch.tensor(m[:3], dtype=torch.float32),
                          "scene_aabb": torch.tensor(S.SCENE_AABB, dtype=torch.float32, device=DEV)})
        rgb = (out["rgb_map"].clamp(0, 1) * 255).round().to(torch.uint8).reshape(H, W, 3).cpu().numpy()
        cv2.imwrite(str(img / f"{f:010d}.png"), rgb[:, :, ::-1])
        sem = out["semantic_map"].argmax(-1).to(torch.uint8).reshape(H, W).cpu().numpy() + 20
        cv2.imwrite(str(root / "pseudo" / f"{f:010d}.png"), sem)
        dep = (out["depth_map"] * 256).round().clamp(0, 65535).to(torch.int32).reshape(H, W).cpu().numpy()
        cv2.imwrite(str(root / "depth" / f"{f:010d}.png"), dep.astype(np.uint16))
    (root / "data_poses" / seq / "cam0_to_world.txt").write_text("\n".join(lines) + "\n")
    return seq


def _train(root, seq, frames, cfg, steps=50, R=1024, seed=5):
    from panopticnerf_b200.lib.datasets.kitti360 import load_frames
    from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper
    fs = load_frames(root, seq, frames, pseudo_dir=root / "pseudo", depth_dir=root / "depth",
                     sem_to_train={20 + c: c for c in range(int(cfg.num_classes))}, device=DEV)
    sampler = RaySampler(fs, seed, scene={"scene_aabb": torch.tensor(S.SCENE_AABB, dtype=torch.float32, device=DEV)})
    student = S.init_network_weights(PN.make_network(cfg), seed=2).to(DEV)
    wrapper = NetworkWrapper(cfg, student)
    opt = FusedAdam(student.parameters(), lr=5e-3)
    losses = []
    for step in range(steps):
        opt.zero_grad()
        _, loss, _, _ = wrapper(sampler.batch(step, R, int(cfg.N_samples)))
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return losses, [p.detach().clone() for p in student.parameters()]


def test_a_student_trained_from_a_written_sequence_learns_and_repeats(tmp_path):
    cfg = PN.make_cfg("cfg1", num_classes=5, perturb=1.0)
    frames = [10, 11, 12, 13]
    seq = _write_teacher_sequence(tmp_path, cfg, frames)
    la, pa = _train(tmp_path, seq, frames, cfg)
    lb, pb = _train(tmp_path, seq, frames, cfg)
    assert np.mean(la[-10:]) < 0.8 * np.mean(la[:5]), la
    assert la == lb
    assert all(torch.equal(x, y) for x, y in zip(pa, pb))
