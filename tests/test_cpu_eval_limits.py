"""The first value outside every range of the evaluation entry points (pnr_eval_semantic / pnr_eval_panoptic /
pnr_eval_image) is refused with PNR_ERR_ARG and an error that names it, and pnr_eval_workspace_bytes follows the
layout eval_kernels.cu documents.  The checks run before any CUDA call, so this needs no GPU: the pointers passed are
placeholders that are never dereferenced.  tests/test_gpu_eval_limits.py runs the same entry points at the last
accepted values."""
import pytest

from panopticnerf_b200 import _capi

X = 64          # a non-null, 16-byte aligned placeholder pointer (never dereferenced: the argument checks refuse first)
ERR_ARG = -1
IMAGE_BYTES = 8 * 256 * 6      # image partials: 256 blocks x 6 doubles (a multiple of 256 already)


def _refused(rc, needle):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg, msg


def _align(b):
    return (b + 255) // 256 * 256


def _layout_bytes(n):
    """[image partials][pair_key u64 | gt_key u32 | pr_key u32][7 u32 count words per slot][iou_acc u64 [64][2]], each
    part aligned to 256 bytes, with S = 1024 slots or the next power of two >= 2n."""
    S = 1024
    while S < 2 * n:
        S *= 2
    return IMAGE_BYTES + _align(S * 16) + _align(S * 28) + _align(8 * 2 * 64)


@pytest.mark.parametrize("n,S", [(0, 1024), (1, 1024), (511, 1024), (512, 1024), (513, 2048), (2**31 - 1, 2**32)])
def test_workspace_bytes_follow_the_layout(n, S):
    got = _capi.lib().pnr_eval_workspace_bytes(n)
    assert got == _layout_bytes(n)
    assert got == IMAGE_BYTES + S * 44 + 1024


def _semantic(n=10, C=4, table=None, n_ids=0):
    return _capi.lib().pnr_eval_semantic(X, X, n, C, table, n_ids, X, None)


def _panoptic(n=10, C=4, table=None, n_ids=0, is_thing=X, ws=X, ws_bytes=None):
    ws_bytes = _capi.lib().pnr_eval_workspace_bytes(max(n, 0)) if ws_bytes is None else ws_bytes
    return _capi.lib().pnr_eval_panoptic(X, X, n, C, table, n_ids, is_thing, ws, ws_bytes, X, X, X, X, None)


@pytest.mark.parametrize("fn", [_semantic, _panoptic])
@pytest.mark.parametrize("kw,needle", [({"C": 0}, "C=0"), ({"C": 65}, "C=65"), ({"n": -1}, "n=-1"),
                                       ({"n": 2**31}, "n=2147483648"), ({"table": X, "n_ids": 0}, "n_ids > 0")])
def test_semantic_and_panoptic_refuse_out_of_range(fn, kw, needle):
    _refused(fn(**kw), needle)


def test_panoptic_refuses_a_null_is_thing():
    _refused(_panoptic(is_thing=None), "is_thing")


@pytest.mark.parametrize("n", [1, 512, 513, 10**6])
def test_panoptic_refuses_a_workspace_one_byte_short(n):
    need = _capi.lib().pnr_eval_workspace_bytes(n)
    _refused(_panoptic(n=n, ws_bytes=need - 1), f"workspace of {need - 1} bytes")


def test_panoptic_refuses_a_misaligned_workspace():
    _refused(_panoptic(ws=X + 8), "16-byte aligned")


def _image(n=10, rgb=X, rgb_gt=X, depth=X, depth_gt=X, ws_bytes=IMAGE_BYTES):
    return _capi.lib().pnr_eval_image(rgb, rgb_gt, depth, depth_gt, n, X, X, ws_bytes, None)


@pytest.mark.parametrize("kw,needle", [({"n": -1}, "n=-1"), ({"rgb_gt": None}, "rgb_map and rgb_gt"),
                                       ({"rgb": None}, "rgb_map and rgb_gt"),
                                       ({"depth_gt": None}, "depth_map and depth_gt"),
                                       ({"depth": None}, "depth_map and depth_gt"),
                                       ({"ws_bytes": IMAGE_BYTES - 1}, f"needs {IMAGE_BYTES}")])
def test_image_refuses_out_of_range(kw, needle):
    _refused(_image(**kw), needle)
