"""GPU: the evaluation kernels (pnr_eval_*) through lib/evaluators against oracle/reference_eval.py - confusion matrix
and panoptic tallies exact (the matched IoUs are summed exactly, so iou_sum is bit-equal to the reference's fsum),
image / depth sums against float64 numpy, determinism, argument errors, and render -> fuse -> evaluate end to end."""
import numpy as np
import pytest
import torch

from oracle import reference_eval as RE
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.evaluators import Evaluator, make_evaluator, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def synth_frame(H, W, C, is_thing, seed, table=None, block=(8, 12)):
    """Blocky panoptic ids with boundary noise: gt blocks of dataset ids (void, unmapped and crowd blocks among them),
    the prediction = the gt shifted by an eighth / a sixth of a block, 15 % of its blocks relabelled, 3 % of its pixels
    random."""
    g = np.random.default_rng(seed)
    bh, bw = block
    shift = (bh // 8, bw // 6)
    nby, nbx = -(-H // bh), -(-W // bw)
    D = C if table is None else len(table)
    d = g.integers(0, D, (nby, nbx))
    ch = RE.channels(d * 1000, C, table)
    thing = np.asarray(is_thing, bool)[np.clip(ch, 0, C - 1)] & (ch >= 0)
    n = np.where(thing, g.integers(1, 1000, d.shape), 0)
    n = np.where(thing & (g.random(d.shape) < 0.1), 0, n)                  # crowd regions
    ids = d * 1000 + n
    ids = np.where(g.random(d.shape) < 0.05, -1, ids)                      # void
    ids = np.where(g.random(d.shape) < 0.02, (D + 3) * 1000, ids)          # an id no channel takes
    gt = np.repeat(np.repeat(ids, bh, 0), bw, 1)[:H, :W]
    relabel = np.where(g.random(d.shape) < 0.15, g.integers(0, D, d.shape) * 1000 + g.integers(0, 1000, d.shape), ids)
    pred = np.roll(np.repeat(np.repeat(relabel, bh, 0), bw, 1)[:H, :W], shift, (0, 1))
    noise = g.random((H, W)) < 0.03
    pred = np.where(noise, g.integers(-1, D + 2, (H, W)) * 1000 + g.integers(0, 1000, (H, W)), pred)
    return pred.astype(np.int32), gt.astype(np.int32)


def dev(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).to(DEV)


def run_panoptic(pred, gt, C, is_thing, table=None):
    tp, fp, fn = (torch.zeros(C, dtype=torch.int64, device=DEV) for _ in range(3))
    iou = torch.zeros(C, dtype=torch.float64, device=DEV)
    ws = torch.empty(ops.workspace_bytes(pred.size), dtype=torch.uint8, device=DEV)
    ops.eval_panoptic(dev(pred).reshape(-1), dev(gt).reshape(-1), C, dev(is_thing, torch.uint8), ws, tp, fp, fn, iou,
                      None if table is None else dev(table, torch.int32))
    return [t.cpu().numpy() for t in (tp, fp, fn, iou)]


@pytest.mark.parametrize("C,H,W,table", [(1, 37, 101, None), (45, 120, 333, None), (64, 200, 257, None),
                                         (45, 77, 190, "partial"), (19, 64, 65, "full")])
def test_confusion_matrix_bit_exact(C, H, W, table):
    tab = None
    if table == "partial":       # dataset ids 0..59: some void (-1), some out of range, some channels never used
        g = np.random.default_rng(C)
        tab = np.where(g.random(60) < 0.2, -1, g.integers(0, C + 3, 60)).astype(np.int32)
    elif table == "full":
        tab = np.random.default_rng(1).permutation(C).astype(np.int32)
    is_thing = np.arange(C) % 3 == 1
    pred, gt = synth_frame(H, W, C, is_thing, seed=H * W, table=tab)
    assert (H * W) % 256 != 0
    conf = torch.zeros(C, C + 1, dtype=torch.int64, device=DEV)
    ops.eval_semantic(dev(pred).reshape(-1), dev(gt).reshape(-1), C, conf, None if tab is None else dev(tab))
    ref = RE.semantic_confusion(pred, gt, C, tab)
    assert ref[:, C].sum() > 0 and (C == 1 or ref.sum() < H * W)          # invalid predictions and void gt present
    assert np.array_equal(conf.cpu().numpy().astype(np.uint64), ref)
    ops.eval_semantic(dev(pred).reshape(-1), dev(gt).reshape(-1), C, conf, None if tab is None else dev(tab))
    assert np.array_equal(conf.cpu().numpy().astype(np.uint64), 2 * ref)  # accumulates


@pytest.mark.parametrize("C,H,W,block,table", [(45, 376, 1408, (8, 12), None), (19, 90, 131, (5, 7), None),
                                               (1, 33, 65, (4, 4), None), (64, 128, 200, (8, 8), "wide"),
                                               (45, 256, 320, (2, 2), None)])
def test_panoptic_tallies_exact(C, H, W, block, table):
    tab = None
    if table == "wide":          # large dataset ids (up to 2999 -> panoptic ids near 3e6) on a partial table
        g = np.random.default_rng(5)
        tab = np.where(g.random(3000) < 0.3, -1, g.integers(0, C, 3000)).astype(np.int32)
    is_thing = (np.arange(C) % 2 == 0) if C > 1 else np.array([True])
    pred, gt = synth_frame(H, W, C, is_thing, seed=C + H, table=tab, block=block)
    ref = RE.panoptic_frame(pred, gt, C, is_thing, tab)
    got = run_panoptic(pred, gt, C, is_thing, tab)
    assert ref[0].sum() > 0 and ref[1].sum() > 0 and ref[2].sum() > 0
    for name, a, b in zip(("tp", "fp", "fn"), got[:3], ref[:3]):
        assert np.array_equal(a, b), name
    np.testing.assert_allclose(got[3], ref[3], rtol=1e-12, atol=0)
    assert np.array_equal(got[3], ref[3])          # exact sum, rounded once: equal to math.fsum
    if block == (2, 2):
        keep = (RE.channels(gt, C, tab) >= 0) | (RE.channels(pred, C, tab) >= 0)
        assert len(np.unique(np.stack([gt.ravel()[keep.ravel()], pred.ravel()[keep.ravel()]]), axis=1)[0]) > 10_000


def test_workspace_too_small_is_refused():
    C = 3
    pred, gt = synth_frame(40, 50, C, [0, 1, 0], seed=0)
    args = [torch.zeros(C, dtype=torch.int64, device=DEV) for _ in range(3)] + [torch.zeros(C, dtype=torch.float64, device=DEV)]
    ws = torch.empty(ops.workspace_bytes(pred.size) - 16, dtype=torch.uint8, device=DEV)
    with pytest.raises(_capi.PnrError, match="workspace"):
        ops.eval_panoptic(dev(pred).reshape(-1), dev(gt).reshape(-1), C, dev([0, 1, 0], torch.uint8), ws, *args)
    assert all(int(t.abs().sum()) == 0 for t in args)


@pytest.mark.parametrize("n", [1, 1000, 376 * 1408, 1024 * 2048 + 3])
def test_image_sums_match_float64(n):
    g = torch.Generator().manual_seed(n)
    rgb, rgb_gt = torch.rand(n, 3, generator=g), torch.rand(n, 3, generator=g)
    depth = torch.rand(n, generator=g) * 80
    depth_gt = torch.where(torch.rand(n, generator=g) < 0.3, torch.zeros(n), torch.rand(n, generator=g) * 80)
    ws = torch.empty(ops.workspace_bytes(0), dtype=torch.uint8, device=DEV)
    s = torch.zeros(3, 6, dtype=torch.float64, device=DEV)
    ops.eval_image(s[0], ws, rgb.to(DEV), rgb_gt.to(DEV), depth.to(DEV), depth_gt.to(DEV))
    ops.eval_image(s[1], ws, rgb.to(DEV), rgb_gt.to(DEV))
    ops.eval_image(s[2], ws, depth_map=depth.to(DEV), depth_gt=depth_gt.to(DEV))
    ref = RE.image_sums(rgb.numpy(), rgb_gt.numpy(), depth.numpy(), depth_gt.numpy())
    got = s.cpu().numpy()
    np.testing.assert_allclose(got[0], ref, rtol=1e-12)
    assert got[1, 1] == n and got[0, 5] == int((depth_gt > 0).sum()) and got[2, 1] == 0 and got[1, 5] == 0
    np.testing.assert_allclose(got[1, :2], ref[:2], rtol=1e-12)
    np.testing.assert_allclose(got[2, 2:], ref[2:], rtol=1e-12)


def test_accumulators_are_deterministic():
    C, is_thing = 45, np.arange(45) % 2 == 0
    frames = [synth_frame(376, 1408, C, is_thing, seed=s) for s in range(3)]
    g = torch.Generator().manual_seed(0)
    rgb = [(torch.rand(376 * 1408, 3, generator=g).to(DEV), torch.rand(376 * 1408, 3, generator=g).to(DEV)) for _ in frames]

    def run():
        ev = Evaluator(num_classes=C, is_thing=is_thing)
        for (pred, gt), (a, b) in zip(frames, rgb):
            ev.evaluate({"rgb_map": a, "depth_map": a[:, 0].contiguous()},
                        {"panoptic_gt": dev(gt), "panoptic_pred": dev(pred), "rgb": b, "depth": b[:, 1].contiguous()})
        return [t.cpu().clone() for t in (ev.conf, ev.tp, ev.fp, ev.fn, ev.iou_sum, ev.frame_sums[:ev.frames])]
    a, b = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_argument_errors():
    lib = _capi.lib()
    x = torch.zeros(10, dtype=torch.int32, device=DEV)
    conf = torch.zeros(70 * 71, dtype=torch.int64, device=DEV)
    for C in (0, 65):
        assert lib.pnr_eval_semantic(x.data_ptr(), x.data_ptr(), 10, C, None, 0, conf.data_ptr(), None) == -1
        assert f"C={C}" in lib.pnr_last_error().decode()
    assert lib.pnr_eval_semantic(None, x.data_ptr(), 10, 3, None, 0, conf.data_ptr(), None) == -1
    assert lib.pnr_eval_semantic(x.data_ptr(), x.data_ptr(), 10, 3, x.data_ptr(), 0, conf.data_ptr(), None) == -1
    assert lib.pnr_eval_semantic(x.data_ptr(), x.data_ptr(), -1, 3, None, 0, conf.data_ptr(), None) == -1
    ws = torch.empty(ops.workspace_bytes(10), dtype=torch.uint8, device=DEV)
    assert lib.pnr_eval_panoptic(x.data_ptr(), x.data_ptr(), 10, 3, None, 0, None, ws.data_ptr(), ws.numel(),
                                 conf.data_ptr(), conf.data_ptr(), conf.data_ptr(), conf.data_ptr(), None) == -1
    assert "is_thing" in lib.pnr_last_error().decode()
    f = torch.zeros(30, device=DEV)
    s = torch.zeros(6, dtype=torch.float64, device=DEV)
    assert lib.pnr_eval_image(f.data_ptr(), None, None, None, 10, s.data_ptr(), ws.data_ptr(), ws.numel(), None) == -1
    assert lib.pnr_eval_image(f.data_ptr(), f.data_ptr(), None, None, 10, s.data_ptr(), ws.data_ptr(), 64, None) == -1
    with pytest.raises(_capi.PnrError, match="CUDA tensor"):
        ops.eval_semantic(x, x.cpu(), 3, torch.zeros(3, 4, dtype=torch.int64, device=DEV))
    with pytest.raises(_capi.PnrError, match="int32"):
        ops.eval_semantic(x, x.long(), 3, torch.zeros(3, 4, dtype=torch.int64, device=DEV))
    with pytest.raises(ValueError, match="pixels"):
        ops.eval_semantic(x, x[:5], 3, torch.zeros(3, 4, dtype=torch.int64, device=DEV))
    ev = Evaluator(num_classes=3)
    with pytest.raises(ValueError, match="CUDA|CPU"):
        ev.evaluate({}, {"panoptic_gt": x.cpu(), "panoptic_pred": x.cpu()})
    with pytest.raises(_capi.PnrError, match="CUDA tensor"):
        ev.evaluate({}, {"panoptic_gt": x, "panoptic_pred": x.cpu()})
    assert torch.count_nonzero(conf) == 0


def test_render_fuse_evaluate_end_to_end():
    import panopticnerf_b200 as PN
    from panopticnerf_b200 import synthetic as S
    from panopticnerf_b200.lib.visualizers import fuse_panoptic
    is_thing, inst_class = [0, 1, 1, 0, 0], [1, 1, 2, 2, 1, 2]
    cfg = PN.make_cfg("cfg1", num_classes=5, num_instances=6, max_hits=3, eval_is_thing=is_thing,
                      eval_inst_class=inst_class)
    from oracle import reference_renderer as O
    net = PN.make_network(cfg)
    net.load_state_dict(S.init_network_weights(O.make_network(cfg)).state_dict())
    net = net.to(DEV)
    ren = PN.make_renderer(cfg, net)
    ev = make_evaluator(cfg)
    g = np.random.default_rng(0)
    conf, tal, sums = 0, [0, 0, 0, 0], []
    for f in range(3):
        batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, seed=f, row0=8 * f, rows=24, num_boxes=32).items()}
        out = ren.render(batch)
        pred = fuse_panoptic(out, is_thing, inst_class)["panoptic"].cpu().numpy()
        R = pred.size
        gt = np.where(g.random(R) < 0.1, g.integers(0, 5, R) * 1000, pred)          # 10 % relabelled
        gt = np.where(g.random(R) < 0.05, -1, gt).astype(np.int32)                  # 5 % void
        rgb_gt, depth_gt = g.random((R, 3)).astype(np.float32), (g.random(R) * 60 - 10).astype(np.float32)
        ev.evaluate(out, {**batch, "panoptic_gt": dev(gt).reshape(6, -1), "rgb": dev(rgb_gt), "depth": dev(depth_gt)})
        conf = conf + RE.semantic_confusion(pred, gt, 5)
        tal = [a + b for a, b in zip(tal, RE.panoptic_frame(pred, gt, 5, is_thing))]
        sums.append(RE.image_sums(out["rgb_map"].cpu().numpy(), rgb_gt, out["depth_map"].cpu().numpy(), depth_gt))
    got = ev.summarize()
    ref = RE.summarize(conf, *tal, is_thing, np.stack(sums))
    assert got["frames"] == 3 and set(got) == set(ref)
    assert np.array_equal(ev.conf.cpu().numpy().astype(np.uint64), conf)
    for a, b in zip((ev.tp, ev.fp, ev.fn, ev.iou_sum), tal):
        assert np.array_equal(a.cpu().numpy(), b)
    assert tal[0].sum() > 0 and tal[1].sum() > 0 and tal[2].sum() > 0
    for k in ref:
        np.testing.assert_allclose(np.asarray(got[k], np.float64), np.asarray(ref[k], np.float64), rtol=1e-12, err_msg=k)
    ev.reset()
    assert ev.frames == 0 and int(ev.conf.sum()) == 0 and float(ev.iou_sum.abs().sum()) == 0.0
