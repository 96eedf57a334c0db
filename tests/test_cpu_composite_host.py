"""The host rules every compositing call shares (raw2outputs, its backward, Network.forward_composite and the fused
renderer): which maps a call produces, in which order, and how the primitive tables reach the kernels.  No GPU: these
are decided before any launch."""
import itertools

import pytest
import torch

from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P


def _expected_keys(C, K, sample_box, box_sem, box_inst):
    """The maps raw2outputs returned, as its rule was written out in it."""
    keys = ["rgb_map", "depth_map", "acc_map", "disp_map", "weights"]
    if C > 0:
        keys.append("semantic_map")
    if K > 0:
        keys.append("instance_map")
    if sample_box is not None and box_sem is not None and C > 0:
        keys.append("fixed_semantic_map")
    if sample_box is not None and box_inst is not None and K > 0:
        keys.append("fixed_instance_map")
    return keys


@pytest.mark.parametrize("C,K,fsem,finst", list(itertools.product((0, 5), (0, 7), (False, True), (False, True))))
def test_map_keys_follow_the_raw2outputs_rule(C, K, fsem, finst):
    tab = torch.zeros(4, dtype=torch.int32)
    want = _expected_keys(C, K, tab, tab if fsem else None, tab if finst else None)
    assert P.composite_map_keys(C, K, fsem, finst) == want
    maps = P.empty_composite_maps(3, 64, C, K, fsem, finst, "cpu")
    assert list(maps) == want
    shapes = {"rgb_map": (3, 3), "weights": (3, 64), "semantic_map": (3, C), "instance_map": (3, K),
              "fixed_semantic_map": (3, C), "fixed_instance_map": (3, K)}
    for k, t in maps.items():
        assert tuple(t.shape) == shapes.get(k, (3,)) and t.dtype == torch.float32, k


def test_primitive_tables_refuse_id_tables_of_different_lengths():
    ref, sb = torch.zeros(2), torch.zeros(2, 8, dtype=torch.int64)
    with pytest.raises(ValueError, match=r"box_sem and box_inst must have one entry per primitive each, got lengths \[3, 10\]"):
        P.primitive_tables(ref, sb, torch.zeros(3, dtype=torch.int64), torch.zeros(10, dtype=torch.int64))


@pytest.mark.parametrize("name", ["sample_box", "box_sem", "box_inst"])
def test_primitive_tables_refuse_another_device(name):
    tables = {"sample_box": torch.zeros(2, 8, dtype=torch.int32), "box_sem": torch.zeros(4, dtype=torch.int32),
              "box_inst": torch.zeros(4, dtype=torch.int32)}
    tables[name] = tables[name].to("meta")
    with pytest.raises(_capi.PnrError, match=f"{name} is on meta, expected cpu"):
        P.primitive_tables(torch.zeros(2), **tables)


def test_primitive_tables_give_int32_tables_and_their_bound():
    ref = torch.zeros(2)
    sb = torch.arange(16, dtype=torch.int64).reshape(8, 2).t()          # not contiguous
    bs, bi = torch.arange(5, dtype=torch.int64), torch.arange(5, dtype=torch.int16)
    out = P.primitive_tables(ref, sb, bs, bi)
    for t, src in zip(out[:3], (sb, bs, bi)):
        assert t.dtype == torch.int32 and t.is_contiguous() and torch.equal(t.long(), src.long())
    assert out[3] == 5
    assert P.primitive_tables(ref, sb, None, bi)[3] == 5
    assert P.primitive_tables(ref, sb, None, None)[3] == 0
    # without per-sample ids nothing indexes the id tables: B = 0 and their lengths are not compared
    assert P.primitive_tables(ref, None, bs[:3], bi)[3] == 0
    assert P.primitive_tables(ref, None, None, None) == (None, None, None, 0)
