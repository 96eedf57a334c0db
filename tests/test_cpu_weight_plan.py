"""CPU tier: the packing plan of a fused-MLP program.  The builder reads the configuration and the shapes, never a weight
value, and the values enter through one packer that applies the plan: the fp16 range check runs on what it packs (the
weights after the feature_linear fold), and programs over different values of the same shapes are the same program."""
import ctypes as C

import pytest
import torch

import test_cpu_hashgrid_network as H
from oracle_hashgrid import hash_cfg
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as S
from test_cpu_program import PROGRAM_BACKWARD, build

ERR_UNSUPPORTED = -4    # PNR_ERR_UNSUPPORTED


def _net(cfg, seed=3):
    return S.init_network_weights(make_network(cfg), seed=seed)


WEIGHTS = [1e5, float("nan"), 65504.0, -65504.0, 65505.0, -65505.0, float("inf"), float("-inf")]


@pytest.mark.parametrize("value", WEIGHTS, ids=["1e5", "nan", "65504", "-65504", "65505", "-65505", "inf", "-inf"])
@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_trunk_weight_outside_fp16_is_refused(precision, value):
    """|w| <= 65504 is packed; 65505, +-Inf and NaN are refused (the host twin of pnr_update_weights' bit 1)."""
    cfg = make_cfg("cfg2", precision=precision)
    net = _net(cfg)
    with torch.no_grad():
        net.pts_linears[3].weight[5, 7] = value
    if abs(value) <= 65504.0:
        build(cfg, net)
        return
    with pytest.raises(_capi.PnrError, match=rf"rc={ERR_UNSUPPORTED}\).*outside the fp16 range"):
        build(cfg, net)
    build(make_cfg("cfg2", precision="bf16x3"), net)          # the bf16 range holds it


def test_fold_overflow_is_refused_though_every_input_is_in_range():
    """feature_linear and the view layer's h columns are each well inside the fp16 range, their fold is not: the check
    is on the packed (folded) weights, not on the tensors given."""
    cfg = make_cfg("cfg2", precision="fp16x3")
    net = _net(cfg)
    with torch.no_grad():
        net.feature_linear.weight.fill_(300.0)
        net.views_linears[0].weight[:, :cfg.W].fill_(300.0)             # folded: 256 * 300 * 300 = 2.3e7
    assert max(float(p.detach().abs().max()) for p in net.parameters()) <= 300.0
    with pytest.raises(_capi.PnrError, match=rf"rc={ERR_UNSUPPORTED}\).*outside the fp16 range"):
        build(cfg, net)
    build(make_cfg("cfg2", precision="bf16x3"), net)


@pytest.mark.parametrize("flags", [0, PROGRAM_BACKWARD], ids=["forward", "backward"])
@pytest.mark.parametrize("encoding", ["frequency", "hashgrid"])
def test_program_depends_on_the_shapes_only(encoding, flags):
    if encoding == "frequency":
        cfg, make = make_cfg("cfg3"), build
    else:
        cfg, make = hash_cfg("cfg3", hash_levels=16, hash_features=2, hash_log2_size=12), H.build
    (p1, w1, c1), (p2, w2, c2) = (make(cfg, _net(cfg, seed), flags=flags) for seed in (1, 2))
    assert C.string_at(C.addressof(p1), C.sizeof(p1)) == C.string_at(C.addressof(p2), C.sizeof(p2))
    assert len(w1) == len(w2) and len(c1) == len(c2)
    assert (w1 != w2).any() and (c1 != c2).any()                 # the values did reach the stream and the constants
