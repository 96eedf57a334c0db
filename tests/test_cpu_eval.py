"""CPU: the evaluation rules of oracle/reference_eval.py on closed-form frames, the product's summary arithmetic against
the reference's, make_evaluator, the refusal of CPU tensors, and the KITTI-360 ground-truth PNG readers."""
import math

import numpy as np
import pytest
import torch

from oracle import reference_eval as RE

C = 4
THING = [0, 1, 1, 0]           # channels 1 and 2 have instances


def frame(rows):
    return np.array(rows, dtype=np.int64)


def pq_of(pred, gt, is_thing=THING, table=None):
    return RE.panoptic_frame(pred, gt, C, is_thing, table)


def test_perfect_prediction_scores_one():
    gt = frame([[0, 0, 1001, 1001, 1002], [3000, 3000, 2001, 2001, 2001]])
    tp, fp, fn, iou = pq_of(gt, gt)
    assert tp.tolist() == [1, 2, 1, 1] and fp.sum() == 0 and fn.sum() == 0 and iou.tolist() == [1.0, 2.0, 1.0, 1.0]
    s = RE.summarize(RE.semantic_confusion(gt, gt, C), tp, fp, fn, iou, THING, RE.image_sums(np.ones((10, 3)), np.ones((10, 3)))[None])
    for k in ("pq", "sq", "rq", "miou", "acc", "pq_th", "pq_st"):
        assert s[k] == 1.0, k
    assert s["psnr"] == math.inf


def test_split_segment_one_tp_one_fp():
    gt = frame([1001] * 10)
    tp, fp, fn, iou = pq_of(frame([1001] * 6 + [1002] * 4), gt)
    assert (tp[1], fp[1], fn[1]) == (1, 1, 0) and iou[1] == 0.6


def test_iou_of_exactly_one_half_is_not_a_match():
    gt = frame([1001] * 10)
    tp, fp, fn, iou = pq_of(frame([1001] * 5 + [1002] * 5), gt)
    assert (tp[1], fp[1], fn[1]) == (0, 2, 1) and iou[1] == 0.0


def test_merged_segments_two_fn():
    gt = frame([1001] * 5 + [1002] * 5)
    tp, fp, fn, _ = pq_of(frame([1003] * 10), gt)
    assert (tp[1], fp[1], fn[1]) == (0, 1, 2)
    tp, fp, fn, iou = pq_of(frame([1003] * 10), frame([1001] * 6 + [1002] * 4))
    assert (tp[1], fp[1], fn[1]) == (1, 0, 1) and iou[1] == 0.6


def test_void_is_taken_out_of_the_union_and_excuses_false_positives():
    # pred 1001 covers gt 1001 (4 px) and 4 void px: union = 8 + 4 - 4 - 4 = 4, IoU 1
    tp, fp, fn, iou = pq_of(frame([1001] * 8), frame([1001] * 4 + [-1] * 4))
    assert (tp[1], fp[1], fn[1], iou[1]) == (1, 0, 0, 1.0)
    # an unmatched prediction more than half on void is not an FP; exactly half is
    gt = frame([0] * 10 + [-1] * 6 + [0] * 4)
    tp, fp, fn, _ = pq_of(frame([0] * 10 + [3000] * 10), gt)
    assert fp[3] == 0 and tp[0] == 1
    gt = frame([0] * 10 + [-1] * 5 + [0] * 5)
    tp, fp, fn, _ = pq_of(frame([0] * 10 + [3000] * 10), gt)
    assert fp[3] == 1
    # ids that map to no channel are void too, on either side
    tp, fp, fn, _ = pq_of(frame([1001] * 8), frame([1001] * 4 + [9000] * 4))
    assert (tp[1], fp[1]) == (1, 0)


def test_crowd_regions_excuse_false_positives_of_their_class_and_are_never_fn():
    gt = frame([2000] * 6 + [0] * 4)                        # crowd of thing class 2, then stuff 0
    tp, fp, fn, _ = pq_of(frame([2001] * 10), gt)
    assert fp[2] == 0 and fn[2] == 0 and tp.sum() == 0      # 60 % of the prediction on its class's crowd
    assert fn[0] == 1                                       # the stuff segment it covers is missed
    tp, fp, fn, _ = pq_of(frame([1001] * 10), gt)            # another class: the crowd does not excuse it
    assert fp[1] == 1 and fn[0] == 1
    tp, fp, fn, _ = pq_of(frame([2000] * 6 + [0] * 4), gt)   # predicting the crowd id itself: no match, no FP
    assert tp[2] == 0 and fn[2] == 0 and fp[2] == 0 and tp[0] == 1
    tp, fp, fn, _ = pq_of(frame([3000] * 10), frame([3000] * 10), is_thing=[0, 1, 1, 1])
    assert tp[3] == 0 and fn[3] == 0 and fp[3] == 0       # n == 0 of a thing class is crowd on its own prediction too


def test_void_only_frame():
    gt = frame([-1] * 7 + [64000] * 3)
    pred = frame([0, 1001, 2002, 3000, -1, 5, 7, 8, 9, 10])
    assert RE.semantic_confusion(pred, gt, C).sum() == 0
    tp, fp, fn, iou = pq_of(pred, gt)
    assert tp.sum() == 0 and fn.sum() == 0 and iou.sum() == 0.0
    s = RE.summarize(RE.semantic_confusion(pred, gt, C), tp, fp, fn, iou, THING, np.zeros((1, 6)))
    assert math.isnan(s["miou"]) and math.isnan(s["acc"]) and math.isnan(s["psnr"]) and math.isnan(s["depth_mae"])


def test_semantic_confusion_and_id_table():
    gt = frame([0, 1001, 1002, 2000, 3000, -5, 7000])
    pred = frame([0, 1001, 2000, -1, 9000, 0, 0])
    conf = RE.semantic_confusion(pred, gt, C)
    want = np.zeros((C, C + 1), dtype=np.uint64)
    want[0, 0] = want[1, 1] = want[1, 2] = want[2, C] = want[3, C] = 1
    assert np.array_equal(conf, want)
    table = [2, -1, 0, 7]                 # dataset id 0 -> channel 2, 1 -> void, 2 -> 0, 3 -> out of range (void)
    conf = RE.semantic_confusion(pred, gt, C, table)
    want = np.zeros((C, C + 1), dtype=np.uint64)
    want[2, 2] = 1                        # (0, 0); 1001 and 3000 are void gt; pred 2000 -> channel 0 under gt 2000
    want[0, C] = 1                        # gt 2000 (channel 0) predicted -1
    assert np.array_equal(conf, want)


def test_two_frames_accumulate():
    g = np.random.default_rng(3)

    def blocky():        # runs of 25 pixels per segment; 20 % of the runs and 10 % of the pixels relabelled
        runs = g.integers(-1, 4, 40) * 1000 + g.integers(0, 3, 40)
        gt = np.repeat(runs, 25)
        pred = np.repeat(np.where(g.random(40) < 0.2, runs + 7, runs), 25)
        pred = np.where(g.random(gt.size) < 0.1, g.integers(0, 4, gt.size) * 1000 + 1, pred)
        return pred, gt
    f = [blocky(), blocky()]
    both = RE.semantic_confusion(np.concatenate([f[0][0], f[1][0]]), np.concatenate([f[0][1], f[1][1]]), C)
    assert np.array_equal(RE.semantic_confusion(*f[0], C) + RE.semantic_confusion(*f[1], C), both)
    # PQ is per frame: a sequence's tallies are the sums of its frames' tallies, and PQ_c comes from those sums
    a, b = pq_of(*f[0]), pq_of(*f[1])
    assert all(x.sum() > 0 for x in a[:3])
    tp, fp, fn, iou = (x + y for x, y in zip(a, b))
    s = RE.summarize(both, tp, fp, fn, iou, THING, np.zeros((2, 6)))
    for c in range(C):
        assert s["pq_per_class"][c] == pytest.approx(iou[c] / (tp[c] + 0.5 * fp[c] + 0.5 * fn[c]), rel=1e-15)


def test_product_summary_matches_the_reference():
    from panopticnerf_b200.lib.evaluators import summarize_counts
    g = np.random.default_rng(7)
    Cn = 19
    conf = g.integers(0, 1000, (Cn, Cn + 1)).astype(np.uint64)
    conf[4, :] = 0
    conf[:, 4] = 0                                          # a class absent on both sides: its IoU is undefined
    tp, fp, fn = (g.integers(0, 20, Cn) for _ in range(3))
    tp[2] = fp[2] = fn[2] = 0
    tp[5] = 0
    fp[5] = 3
    iou = tp * g.uniform(0.5, 1.0, Cn)
    thing = g.integers(0, 2, Cn)
    fs = np.abs(g.normal(size=(5, 6))) * 100
    fs[2, 1] = 0                                           # a frame without rgb
    a, b = summarize_counts(conf, tp, fp, fn, iou, thing, fs), RE.summarize(conf, tp, fp, fn, iou, thing, fs)
    assert set(a) == set(b)
    for k in a:
        np.testing.assert_allclose(np.asarray(a[k], dtype=np.float64), np.asarray(b[k], dtype=np.float64), rtol=1e-14, err_msg=k)


def test_make_evaluator_and_cpu_tensors_are_refused(tmp_path):
    import panopticnerf_b200 as PN
    from panopticnerf_b200.lib.evaluators import Evaluator, make_evaluator
    cfg = PN.make_cfg("cfg1", num_classes=5, eval_is_thing=[0, 1, 1, 0, 0])
    ev = make_evaluator(cfg)
    assert isinstance(ev, Evaluator) and ev.C == 5 and ev.is_thing.tolist() == [0, 1, 1, 0, 0]
    with pytest.raises(ValueError, match="CUDA|CPU"):
        ev.evaluate({}, {"panoptic_gt": torch.zeros(4, dtype=torch.int32), "panoptic_pred": torch.zeros(4, dtype=torch.int32)})
    plug = tmp_path / "my_eval.py"
    plug.write_text("class Evaluator:\n    def __init__(self, cfg):\n        self.cfg = cfg\n")
    cfg.evaluator_path = str(plug)
    assert make_evaluator(cfg).cfg is cfg
    with pytest.raises(ValueError, match="num_classes"):
        Evaluator(PN.make_cfg("cfg1"))
    with pytest.raises(ValueError, match="num_classes"):
        Evaluator(num_classes=65)
    with pytest.raises(ValueError, match="is_thing"):
        Evaluator(num_classes=3, is_thing=[1, 0])


def test_ground_truth_png_readers(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from panopticnerf_b200.lib.datasets.kitti360 import load_panoptic_gt, load_semantic_gt
    g = np.random.default_rng(0)
    inst = (g.integers(0, 46, (9, 13)) * 1000 + g.integers(0, 500, (9, 13))).astype(np.uint16)
    sem = g.integers(0, 46, (9, 13)).astype(np.uint8)
    cv2.imwrite(str(tmp_path / "inst.png"), inst)
    cv2.imwrite(str(tmp_path / "sem.png"), sem)
    cv2.imwrite(str(tmp_path / "rgb.png"), np.zeros((9, 13, 3), np.uint8))
    cv2.imwrite(str(tmp_path / "rgb16.png"), np.zeros((9, 13, 3), np.uint16))
    p = load_panoptic_gt(tmp_path / "inst.png")
    assert p.dtype == torch.int32 and p.shape == (9, 13) and np.array_equal(p.numpy(), inst.astype(np.int32))
    s = load_semantic_gt(tmp_path / "sem.png")
    assert s.dtype == torch.int32 and np.array_equal(s.numpy(), sem.astype(np.int32) * 1000)
    with pytest.raises(ValueError, match="16-bit"):
        load_panoptic_gt(tmp_path / "sem.png")
    with pytest.raises(ValueError, match="8-bit"):
        load_semantic_gt(tmp_path / "inst.png")
    with pytest.raises(ValueError, match="single-channel"):
        load_semantic_gt(tmp_path / "rgb.png")
    with pytest.raises(ValueError, match="single-channel"):
        load_panoptic_gt(tmp_path / "rgb16.png")
    with pytest.raises(FileNotFoundError):
        load_panoptic_gt(tmp_path / "missing.png")
