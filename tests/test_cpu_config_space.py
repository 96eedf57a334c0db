"""CPU tier: the configuration space `pnr_create` accepts (check_config in csrc/pnr_api.cu), at its edges.  Every
value at the edge of a range, alone and combined with the other extremes, must build a forward program that stays
inside the program's limits, keeps its schedule consistent and, replayed from the packed bytes, computes the float64
oracle network; the first value outside each range must be refused by name.  The same for the backward programs
(x3 modes, D <= 9) and for hash grids whose E = L*F pads the embedding operand."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import test_cpu_hashgrid_network as H
from oracle import reference_renderer as O
from oracle_hashgrid import hash_cfg, oracle_like
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as S
from test_cpu_hazards import unordered_conflicts
from test_cpu_program import (A_EMB, EPI_GRAD_OUT, EPI_LOGITS, EPI_MASK_TO_A, EPI_RELU_TO_A, EPI_VIEW_RGB, K_MAX_STAGES, K_MAX_STEPS,
                              PROGRAM_BACKWARD, assert_grad_close, build, check_invariants, replay, trunk_grad_oracle)
from util import assert_close, rms

K_MAX_CONSTS = 65536        # mlp_program.h: what the uint16_t constant offsets of EpiDesc address
# replay with exact activations: only the 16-bit split of the weights separates it from fp32 (as in test_cpu_program)
TOL = {"fp16x3": 2e-5, "bf16x3": 1e-4, "fp16": 4e-3, "bf16": 3e-2}
PRECISIONS = ["fp16x3", "bf16x3", "fp16", "bf16"]
HEADS = [(0, 0), (1, 0), (0, 128), (1, 1), (17, 113), (128, 128)]
ENCODINGS = [(0, 0), (10, 4), (0, 4), (10, 0)]          # (xyz_res, view_res)


def _case(D, W, heads, enc, precision):
    return dict(D=D, W=W, num_classes=heads[0], num_instances=heads[1], xyz_res=enc[0], view_res=enc[1],
                precision=precision)


# Every D edge x every width, the heads, encodings and precisions rotated over them so that each meets every width;
# then the corners: the widest, deepest network with the largest heads, and each edge value alone on cfg2.
FORWARD = [_case(D, W, HEADS[i % 6], ENCODINGS[i % 4], PRECISIONS[(i // 2) % 4])
           for i, (D, W) in enumerate(itertools.product([3, 4, 9, 10, 13, 16], [64, 128, 256]))]
FORWARD += [_case(16, 256, (128, 128), (0, 0), "bf16x3"),
            _case(12, 256, (128, 128), (10, 4), "fp16x3"), _case(16, 64, (128, 128), (10, 4), "bf16x3"),
            _case(16, 128, (128, 128), (0, 4), "fp16"), _case(3, 64, (1, 1), (0, 0), "bf16")]
FORWARD += [dict(D=3), dict(D=16), dict(W=64), dict(W=128), dict(num_classes=1), dict(num_instances=1),
            dict(num_classes=128), dict(num_instances=128), dict(xyz_res=0), dict(view_res=0)]
FORWARD += [dict(precision=p) for p in PRECISIONS[1:]]


def _id(over):
    return "-".join(f"{k[:4]}{v}" for k, v in over.items())


def _inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(n, 3, generator=g) * 2 - 1) * 4
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    return pts, vd


def _check_limits(prog, consts, stages_of):
    """The program fits its tables, and every constant it addresses lies inside the table its offsets can reach."""
    assert 0 < prog.n_stages <= K_MAX_STAGES and 0 < prog.n_steps <= K_MAX_STEPS
    assert prog.n_consts == len(consts) <= K_MAX_CONSTS
    for s in range(prog.n_steps):
        ed = prog.ep[s]
        if ed.kind not in (EPI_GRAD_OUT, EPI_MASK_TO_A):          # the gradient epilogues read no bias
            assert ed.bias_off % 4 == 0 and ed.bias_off + ed.n <= len(consts), s
        if ed.kind == EPI_RELU_TO_A and ed.sigma:
            assert ed.aux_off + ed.n <= len(consts), s
        if ed.kind == EPI_VIEW_RGB:
            assert ed.aux_off + 3 * ed.n <= len(consts), s
    assert len(stages_of) == prog.n_steps


def _oracle64(cfg, net):
    onet = O.Network(cfg).double()
    onet.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    return onet


def _compare(got, ref, cfg, what, tol):
    C_, K_ = cfg.num_classes, cfg.num_instances
    for name, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4)), ("sem", slice(4, 4 + C_)), ("inst", slice(4 + C_, 4 + C_ + K_))):
        if ref[:, sl].numel():
            assert_close(got[:, sl], ref[:, sl], rms(ref[:, sl]), f"{what} {name}", rel=tol)


@pytest.mark.parametrize("over", FORWARD, ids=[_id(o) for o in FORWARD])
def test_accepted_config_builds_and_replays_against_float64(over):
    cfg = make_cfg("cfg2", **over)
    net = S.init_network_weights(make_network(cfg), seed=3)
    prog, w16, consts = build(cfg, net)
    pts, vd = _inputs(257, seed=5)
    got, stages_of = replay(prog, w16, consts, cfg, pts, vd)
    _check_limits(prog, consts, stages_of)
    check_invariants(prog, stages_of)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20 and not bad, f"{over}: unordered conflicts, e.g. {bad[:3]}"
    with torch.no_grad():
        ref = _oracle64(cfg, net)(pts.double(), vd.double())
    _compare(torch.from_numpy(got), ref, cfg, str(over), TOL[cfg.precision])


def test_merged_heads_with_unequal_halves_address_their_own_biases():
    """C = 17, K = 113: the merged logits step's halves are 32 and 128 columns wide; each half's bias block and output
    channel offset belong to its own head."""
    cfg = make_cfg("cfg2", num_classes=17, num_instances=113)
    prog, _, consts = build(cfg, S.init_network_weights(make_network(cfg), seed=3))
    logits = [prog.ep[s] for s in range(prog.n_steps) if prog.ep[s].kind == EPI_LOGITS]
    assert len(logits) == 1
    e = logits[0]
    assert (e.n0, e.n, e.n_valid, e.n_valid1, e.out_off, e.out_off1) == (32, 160, 17, 113, 4, 21)
    assert np.all(consts[e.bias_off + 17:e.bias_off + 32] == 0) and np.all(consts[e.bias_off + 32 + 113:e.bias_off + 160] == 0)


def test_largest_networks_need_more_than_4096_constants():
    """The configurations whose constant tables outgrew the old 4096-float cap: they load now."""
    for over in (dict(D=13), dict(D=14), dict(D=16), dict(D=12, num_classes=128, num_instances=128)):
        cfg = make_cfg("cfg2", **over)
        prog, _, consts = build(cfg, S.init_network_weights(make_network(cfg), seed=0))
        assert 4096 < len(consts) <= K_MAX_CONSTS, over


def _program_host_error(pc):
    L = _capi.lib()
    w = torch.zeros(4, 4)
    ptrs = (C.c_void_p * 2)(w.data_ptr(), w.data_ptr())
    shp = (C.c_int64 * 4)(4, 4, 4, 1)
    pb, wb, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
    rc = L.pnr_program_host(C.byref(pc), ptrs, shp, 2, 0, None, 0, C.byref(pb), None, 0, C.byref(wb), None, 0, C.byref(nc))
    return rc, L.pnr_last_error().decode()


REFUSED = [(dict(D=2), "D=2"), (dict(D=17), "D=17"), (dict(W=32), "W=32"), (dict(num_classes=129), "num_classes=129"),
           (dict(num_instances=129), "num_instances=129"), (dict(xyz_res=11), "xyz_res=11"), (dict(view_res=5), "view_res=5"),
           (dict(xyz_res=-1), "xyz_res=-1"), (dict(num_classes=-1), "num_classes=-1")]
REFUSED_GRID = [(dict(hash_features=3), "hash_features=3"), (dict(hash_levels=9, hash_features=8), "E=72 > 64"),
                (dict(hash_levels=33, hash_features=1), "hash_levels=33"), (dict(hash_levels=0), "hash_levels=0")]


@pytest.mark.parametrize("over,msg", REFUSED + REFUSED_GRID, ids=[m for _, m in REFUSED + REFUSED_GRID])
def test_first_value_outside_each_range_is_refused_by_name(over, msg):
    if any(k.startswith("hash_") for k in over):
        base = hash_cfg("cfg2", hash_log2_size=12)
        pc = H.pnr_config(base)
        for k, v in over.items():
            setattr(pc, k, v)
    else:
        pc = H.pnr_config(make_cfg("cfg2", **over))
    rc, err = _program_host_error(pc)
    assert rc != 0 and msg in err, (over, err)


# ---------------------------------------------------------------------------------------------------------- backward
BACKWARD = [dict(D=9), dict(D=9, W=64, precision="bf16x3", xyz_res=0), dict(D=3), dict(D=3, W=64, xyz_res=0),
            dict(D=9, W=128, precision="bf16x3"), dict(D=4, W=64, xyz_res=10), dict(D=3, W=256, xyz_res=0, precision="bf16x3")]


@pytest.mark.parametrize("over", BACKWARD, ids=[_id(o) for o in BACKWARD])
def test_backward_program_edges_replay_against_float64_autograd(over):
    cfg = make_cfg("cfg2", **over)
    net = S.init_network_weights(make_network(cfg), seed=4)
    prog, w16, consts = build(cfg, net, flags=PROGRAM_BACKWARD)
    assert prog.n_steps == 2 * cfg.D + 1
    g = torch.Generator().manual_seed(6)
    pts = (torch.rand(200, 3, generator=g) * 2 - 1) * 4
    grad_h = torch.randn(200, cfg.W, generator=g)
    got, stages_of = replay(prog, w16, consts, cfg, pts, torch.zeros_like(pts), grad_in=grad_h.double().numpy())
    _check_limits(prog, consts, stages_of)
    check_invariants(prog, stages_of)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20 and not bad, f"{over}: unordered conflicts, e.g. {bad[:3]}"
    ref, min_z = trunk_grad_oracle(cfg, net, pts, grad_h)
    assert got.shape == ref.shape
    tol = {"fp16x3": 2e-5, "bf16x3": 1e-4}[cfg.precision]
    kink = {"fp16x3": 1e-6, "bf16x3": 2e-5}[cfg.precision]
    assert_grad_close(torch.from_numpy(got), ref, min_z, f"{over} d_emb", tol, kink)


def test_backward_program_is_refused_past_the_sign_pattern_slots():
    """D = 9 keeps 8 sign patterns, the most shared memory holds; D = 10 is refused by name (the forward builds)."""
    for W in (64, 256):
        cfg = make_cfg("cfg2", D=10, W=W)
        net = S.init_network_weights(make_network(cfg), seed=0)
        build(cfg, net)
        with pytest.raises(_capi.PnrError, match="slots"):
            build(cfg, net, flags=PROGRAM_BACKWARD)


# --------------------------------------------------------------------------------------------------------- hash grids
GRIDS = [(1, 1), (8, 1), (5, 2), (3, 8), (8, 8), (32, 2), (16, 4)]          # E = 1, 8, 10, 24, 64, 64, 64
GRID_MODES = ["fp16x3", "bf16x3", "fp16", "fp16x3", "bf16x3", "bf16", "fp16x3"]
GRID_SHAPES = [dict(D=8, W=256), dict(D=3, W=64), dict(D=9, W=128, num_classes=17, num_instances=113), dict(D=5, W=256),
               dict(D=4, W=128), dict(D=16, W=256, num_classes=128, num_instances=128), dict(D=9, W=64, num_classes=1)]


def _grid_cfg(k, **extra):
    L, F = GRIDS[k]
    return hash_cfg("cfg2", hash_levels=L, hash_features=F,
                    **{"hash_log2_size": 12, "precision": GRID_MODES[k], **GRID_SHAPES[k], **extra})


def _grid_points(n, seed):
    return H._points(n, seed)


@pytest.mark.parametrize("k", range(len(GRIDS)), ids=[f"L{L}F{F}" for L, F in GRIDS])
def test_hashgrid_edges_replay_forward_against_float64(k):
    cfg = _grid_cfg(k)
    E = cfg.hash_levels * cfg.hash_features
    net = S.init_network_weights(make_network(cfg), seed=3)
    prog, w16, consts = H.build(cfg, net)
    emb = [prog.st[i] for i in range(prog.n_stages) if prog.st[i].a_kind == A_EMB]
    assert emb and all(sd.ksteps * 16 == (E + 15) // 16 * 16 for sd in emb)         # K = E padded to 16, zero columns
    pts, vd = _grid_points(300, seed=5)
    on64 = oracle_like(net, cfg, torch.float64)
    with torch.no_grad():
        hx = on64.xyz_encoder(pts)
        ref = on64(pts.double(), vd.double())
    got, stages_of = H.replay(prog, w16, consts, cfg, hx.numpy(), vd)
    _check_limits(prog, consts, stages_of)
    check_invariants(prog, stages_of)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20 and not bad, f"L{cfg.hash_levels} F{cfg.hash_features}: unordered conflicts, e.g. {bad[:3]}"
    _compare(torch.from_numpy(got), ref, cfg, f"L{cfg.hash_levels} F{cfg.hash_features}", TOL[cfg.precision])


@pytest.mark.parametrize("k", range(len(GRIDS)), ids=[f"L{L}F{F}" for L, F in GRIDS])
def test_hashgrid_edges_replay_backward_against_float64_autograd(k):
    cfg = _grid_cfg(k, D=min(GRID_SHAPES[k]["D"], 9), precision="bf16x3" if "bf16" in GRID_MODES[k] else "fp16x3")
    E = cfg.hash_levels * cfg.hash_features
    net = S.init_network_weights(make_network(cfg), seed=4)
    prog, w16, consts = H.build(cfg, net, flags=PROGRAM_BACKWARD)
    grad_out = [prog.ep[s] for s in range(prog.n_steps) if prog.ep[s].kind == EPI_GRAD_OUT]
    assert len(grad_out) == 2 and all(e.n_valid == E and e.n == (E + 15) // 16 * 16 for e in grad_out)
    pts, _ = _grid_points(200, seed=6)
    grad_h = torch.randn(200, cfg.W, generator=torch.Generator().manual_seed(7))
    on64 = oracle_like(net, cfg, torch.float64)
    with torch.no_grad():
        hx = on64.xyz_encoder(pts)
    got, stages_of = H.replay(prog, w16, consts, cfg, hx.numpy(), torch.zeros_like(pts), grad_in=grad_h.double().numpy())
    check_invariants(prog, stages_of)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20 and not bad, f"L{cfg.hash_levels} F{cfg.hash_features}: unordered conflicts, e.g. {bad[:3]}"
    ex = hx.clone().requires_grad_(True)
    h, min_z = ex, torch.full((200,), float("inf"), dtype=torch.float64)
    for i, lin in enumerate(on64.pts_linears):
        pre = lin(h)
        min_z = torch.minimum(min_z, pre.detach().abs().min(dim=1).values)
        h = torch.relu(pre)
        if i == on64.skip:
            h = torch.cat([ex, h], -1)
    h.backward(grad_h.double())
    tol = {"fp16x3": 2e-5, "bf16x3": 1e-4}[cfg.precision]
    kink = {"fp16x3": 1e-6, "bf16x3": 2e-5}[cfg.precision]
    assert_grad_close(torch.from_numpy(got), ex.grad, min_z, f"L{cfg.hash_levels} F{cfg.hash_features} dL/dh(x)", tol, kink)
