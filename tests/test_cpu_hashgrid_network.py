"""CPU tier of the hash-grid trunk input (cfg.xyz_encoding = "hashgrid"): the programs `pnr_program_host` builds for a
hash-grid network, replayed on the host from the packed bytes with h(x) as the embedding operand, against the oracle
hash-grid network (tests/oracle_hashgrid.py); the hazard check of their schedule; the state_dict drop-in; argument
rejection; and the ctypes layout of pnr_config against the header."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import reference_renderer as O
from panopticnerf_b200 import _capi, make_network, synthetic as S
from oracle_hashgrid import SCENE_AABB, hash_cfg, mlp_flops_per_sample, oracle_like
from test_cpu_hazards import unordered_conflicts
from test_cpu_program import (A_EMB, A_TMEM, COL_A_HI, COL_HEAD_HI, EPI_GRAD_OUT, EPI_LOADG_TO_A, EPI_LOGITS, EPI_MASK_TO_A,
                              EPI_RELU_TO_A, EPI_VIEW_RGB, F_FIRST, F_WAIT_E0, MlpProgram, PROGRAM_BACKWARD,
                              PROGRAM_VIEW_PRODUCERS, assert_grad_close, check_invariants, to_f32)
from util import assert_close, rms

ROOT = Path(__file__).resolve().parent.parent

# E = 32 (L16 F2), 16 (L8 F2: no padding), 64 (L16 F4); tables of 2^12 entries keep the CPU oracle fast
GRIDS = [dict(hash_levels=16, hash_features=2, hash_log2_size=12), dict(hash_levels=8, hash_features=2, hash_log2_size=12),
         dict(hash_levels=16, hash_features=4, hash_log2_size=12)]
MODES = [("cfg2", {}), ("cfg3", dict(precision="bf16x3")), ("cfg1", dict(precision="fp16"))]


def pnr_config(cfg):
    pc = _capi.PnrConfig(cfg.D, cfg.W, cfg.xyz_res, cfg.view_res, cfg.num_classes, cfg.num_instances,
                         _capi.PREC[cfg.precision], 0)
    if getattr(cfg, "xyz_encoding", "frequency") == "hashgrid":
        pc.xyz_encoding = _capi.XYZ_ENCODING["hashgrid"]
        pc.hash_levels, pc.hash_features, pc.hash_log2_size = cfg.hash_levels, cfg.hash_features, cfg.hash_log2_size
        pc.hash_base_resolution, pc.hash_per_level_scale = cfg.hash_base_resolution, cfg.hash_per_level_scale
        if cfg.hash_aabb is not None:
            pc.hash_aabb[:] = [float(v) for v in torch.as_tensor(cfg.hash_aabb).reshape(6)]
    return pc


def build(cfg, net, flags=0):
    host, shapes = [], []
    for lin in net._linears():
        w, b = lin.weight.detach().float().contiguous(), lin.bias.detach().float().contiguous()
        host += [w, b]
        shapes += [w.shape[0], w.shape[1], b.shape[0], 1]
    L = _capi.lib()
    pc = pnr_config(cfg)
    ptrs = (C.c_void_p * len(host))(*[t.data_ptr() for t in host])
    shp = (C.c_int64 * len(shapes))(*shapes)
    pb, wb, nc = C.c_size_t(), C.c_size_t(), C.c_size_t()
    _capi.check(L.pnr_program_host(C.byref(pc), ptrs, shp, len(host), flags, None, 0, C.byref(pb), None, 0,
                                   C.byref(wb), None, 0, C.byref(nc)), "pnr_program_host (sizes)")
    prog = MlpProgram()
    w16 = np.zeros(wb.value // 2, dtype=np.uint16)
    consts = np.zeros(nc.value, dtype=np.float32)
    _capi.check(L.pnr_program_host(C.byref(pc), ptrs, shp, len(host), flags, C.byref(prog), pb.value, C.byref(pb),
                                   w16.ctypes.data, wb.value, C.byref(wb), consts.ctypes.data, nc.value, C.byref(nc)),
                "pnr_program_host")
    return prog, w16, consts


def replay(prog, w16, consts, cfg, emb_x, viewdirs, grad_in=None):
    """What the kernel computes from the packed program (float64, exact activations) with emb_x [S, E] as the
    embedding operand (h(x), zero-padded to the program's K)."""
    S_ = emb_x.shape[0]
    bf16 = cfg.precision.startswith("bf16")
    emb = np.zeros((S_, 64)); emb[:, :emb_x.shape[1]] = emb_x
    dirs = np.zeros((S_, 32)); dirs[:, :3 + 6 * cfg.view_res] = O.embed(viewdirs, cfg.view_res).double().numpy()
    act = {COL_A_HI: np.zeros((S_, 256)), COL_HEAD_HI: np.zeros((S_, 128))}
    acc = np.zeros((S_, 256))
    out = np.zeros((S_, 4 + cfg.num_classes + cfg.num_instances if grad_in is None else emb_x.shape[1]))
    sig, masks, stages_of = np.zeros(S_), {}, []
    for i in range(prog.n_stages):
        if prog.st[i].flags & F_WAIT_E0:
            stages_of.append([])
        stages_of[-1].append(i)
    for s, idxs in enumerate(stages_of):
        ed = prog.ep[s]
        for i in idxs:
            sd = prog.st[i]
            n, kc, base = sd.n, sd.ksteps * 2, sd.gofs // 2
            hi = to_f32(w16[base:base + n * kc * 8], bf16).reshape(kc, n, 8).astype(np.float64)
            lo = np.zeros_like(hi)
            if prog.passes == 3:
                lo0 = base + sd.lo_off16 * 8
                lo = to_f32(w16[lo0:lo0 + n * kc * 8], bf16).reshape(kc, n, 8).astype(np.float64)
            Wm = (hi + lo).transpose(1, 0, 2).reshape(n, kc * 8)
            if sd.a_kind == A_TMEM:
                region = COL_A_HI if sd.a_off >= COL_A_HI else COL_HEAD_HI
                k0 = (sd.a_off - region) * 2
                A = act[region][:, k0:k0 + kc * 8]
            elif sd.a_kind == A_EMB:
                A = emb[:, sd.a_off * 2:sd.a_off * 2 + kc * 8]
            else:
                A = dirs[:, sd.a_off * 2:sd.a_off * 2 + kc * 8]
            if sd.flags & F_FIRST:
                acc[:, sd.acc_col:sd.acc_col + n] = 0.0
            acc[:, sd.acc_col:sd.acc_col + n] += A @ Wm.T
        n = ed.n
        v = acc[:, ed.acc_col:ed.acc_col + n] + consts[ed.bias_off:ed.bias_off + n][None]
        if ed.kind == EPI_MASK_TO_A:
            v = acc[:, ed.acc_col:ed.acc_col + n]
            act[ed.dst_col][:, :n] = np.where(masks[ed.n_valid - 1][:, :n], v, 0.0) if ed.n_valid else v
        elif ed.kind == EPI_LOADG_TO_A:
            act[ed.dst_col][:, :n] = np.where(v > 0.0, grad_in[:, :n], 0.0)
        elif ed.kind == EPI_GRAD_OUT:
            v = acc[:, ed.acc_col:ed.acc_col + ed.n_valid]
            out[:, :ed.n_valid] = v + (out[:, :ed.n_valid] if ed.n_valid1 else 0.0)
        elif ed.kind == EPI_RELU_TO_A:
            v = np.maximum(v, 0.0)
            if ed.sigma:
                sig = v @ consts[ed.aux_off:ed.aux_off + n].astype(np.float64)
            if grad_in is not None and ed.n_valid:
                masks[ed.n_valid - 1] = v > 0.0
            act[ed.dst_col][:, :n] = v
        elif ed.kind == EPI_VIEW_RGB:
            v = np.maximum(v, 0.0)
            wr = consts[ed.aux_off:ed.aux_off + 3 * n].astype(np.float64).reshape(3, n)
            out[:, :3] = v @ wr.T + consts[prog.rgb_bias_off:prog.rgb_bias_off + 3][None]
            out[:, 3] = sig + consts[prog.sigma_bias_off]
        else:
            assert ed.kind == EPI_LOGITS
            out[:, ed.out_off:ed.out_off + ed.n_valid] = v[:, :ed.n_valid]
            if ed.n_valid1:
                out[:, ed.out_off1:ed.out_off1 + ed.n_valid1] = v[:, ed.n0:ed.n0 + ed.n_valid1]
    return out, stages_of


def _points(n, seed):
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(SCENE_AABB[:3]), torch.tensor(SCENE_AABB[3:])
    pts = lo + (hi - lo) * (torch.rand(n, 3, generator=g) * 1.1 - 0.05)        # a few points outside the box
    vd = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    return pts, vd


@pytest.mark.parametrize("grid", GRIDS, ids=["E32", "E16", "E64"])
@pytest.mark.parametrize("preset,over", MODES, ids=["cfg2-fp16x3", "cfg3-bf16x3", "cfg1-fp16"])
def test_hashgrid_program_replay_matches_oracle(preset, over, grid):
    cfg = hash_cfg(preset, **over, **grid)
    net = S.init_network_weights(make_network(cfg), seed=3)
    E = cfg.hash_levels * cfg.hash_features
    assert net.in_dim == E and net.pts_linears[0].weight.shape == (cfg.W, E)
    prog, w16, consts = build(cfg, net)
    assert prog.Lx == 0
    emb_stages = [prog.st[i] for i in range(prog.n_stages) if prog.st[i].a_kind == A_EMB]
    assert emb_stages and all(sd.ksteps * 16 == (E + 15) // 16 * 16 for sd in emb_stages)   # K = E padded to 16
    pts, vd = _points(300, seed=5)
    onet = oracle_like(net, cfg)
    with torch.no_grad():
        hx = onet.xyz_encoder(pts)
        ref = onet(pts, vd).double()
    got, stages_of = replay(prog, w16, consts, cfg, hx.double().numpy(), vd)
    check_invariants(prog, stages_of)
    tol = {"fp16x3": 2e-5, "bf16x3": 1e-4, "fp16": 4e-3}[cfg.precision]
    got = torch.from_numpy(got)
    C_, K_ = cfg.num_classes, cfg.num_instances
    for name, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4)), ("sem", slice(4, 4 + C_)), ("inst", slice(4 + C_, 4 + C_ + K_))):
        if ref[:, sl].numel():
            assert_close(got[:, sl], ref[:, sl], rms(ref[:, sl]), f"{preset} {grid} {name}", rel=tol)


@pytest.mark.parametrize("grid", GRIDS, ids=["E32", "E16", "E64"])
@pytest.mark.parametrize("preset,over", [("cfg2", {}), ("cfg3", dict(precision="bf16x3")), ("cfg1", dict(D=5, W=128))],
                         ids=["cfg2-fp16x3", "cfg3-bf16x3", "cfg1-D5W128"])
def test_hashgrid_backward_program_replay_matches_autograd(preset, over, grid):
    """dL/dh(x) through the trunk from the backward program, against float64 autograd through the oracle's trunk."""
    cfg = hash_cfg(preset, **over, **grid)
    net = S.init_network_weights(make_network(cfg), seed=4)
    prog, w16, consts = build(cfg, net, flags=PROGRAM_BACKWARD)
    E = cfg.hash_levels * cfg.hash_features
    grad_out = [prog.ep[s] for s in range(prog.n_steps) if prog.ep[s].kind == EPI_GRAD_OUT]
    assert len(grad_out) == 2 and all(e.n_valid == E and e.n == (E + 15) // 16 * 16 for e in grad_out)
    pts, _ = _points(200, seed=6)
    grad_h = torch.randn(200, cfg.W, generator=torch.Generator().manual_seed(7))
    onet = oracle_like(net, cfg, torch.float64)
    with torch.no_grad():
        hx = onet.xyz_encoder(pts)
    got, stages_of = replay(prog, w16, consts, cfg, hx.numpy(), torch.zeros_like(pts), grad_in=grad_h.double().numpy())
    check_invariants(prog, stages_of)
    ex = hx.clone().requires_grad_(True)
    h, min_z = ex, torch.full((200,), float("inf"), dtype=torch.float64)
    for i, lin in enumerate(onet.pts_linears):
        pre = lin(h)
        min_z = torch.minimum(min_z, pre.detach().abs().min(dim=1).values)
        h = torch.relu(pre)
        if i == onet.skip:
            h = torch.cat([ex, h], -1)
    h.backward(grad_h.double())
    tol = {"fp16x3": 2e-5, "bf16x3": 1e-4}[cfg.precision]
    assert_grad_close(torch.from_numpy(got), ex.grad, min_z, f"{preset} {grid} dL/dh(x)", tol, 1e-6)


HAZARD_CASES = [("cfg2", dict(hash_levels=16, hash_features=2)), ("cfg2", dict(hash_levels=8, hash_features=2, precision="fp16")),
                ("cfg3", dict(hash_levels=16, hash_features=4)), ("cfg1", dict(hash_levels=8, hash_features=8, precision="bf16x3"))]


@pytest.mark.parametrize("preset,over", HAZARD_CASES)
@pytest.mark.parametrize("flags", [0, PROGRAM_BACKWARD, PROGRAM_VIEW_PRODUCERS])
def test_hashgrid_program_conflicts_are_ordered(preset, over, flags):
    """The happens-before check of tests/test_cpu_hazards.py on the hash-grid programs (the embedding operand is
    narrower, so layer 0 and the skip layer have fewer stages)."""
    cfg = hash_cfg(preset, hash_log2_size=12, **over)
    if flags == PROGRAM_BACKWARD and not cfg.precision.endswith("x3"):
        pytest.skip("backward programs are x3 only")
    if flags == PROGRAM_VIEW_PRODUCERS and cfg.num_classes:
        pytest.skip("view on producers: networks without heads")
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=0), flags=flags)
    checked, bad = unordered_conflicts(prog)
    assert checked > 20
    assert not bad, f"{preset} {over} flags={flags}: unordered conflicts, e.g. {bad[:3]}"


def test_frequency_programs_are_unchanged_by_the_new_fields():
    """An all-zero tail of pnr_config is today's network: same program bytes as an explicit 'frequency' config."""
    from panopticnerf_b200 import make_cfg
    cfg = make_cfg("cfg3")
    net = S.init_network_weights(make_network(cfg), seed=0)
    assert not net.hashgrid and net.in_dim == 63
    a = build(cfg, net)
    b = build(make_cfg("cfg3", xyz_encoding="frequency", hash_aabb=SCENE_AABB), net)
    assert bytes(a[0]) == bytes(b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.parametrize("preset", ["cfg1", "cfg2", "cfg3"])
def test_hashgrid_state_dict_is_drop_in(preset):
    import oracle_hashgrid as OH
    cfg = hash_cfg(preset, hash_log2_size=12)
    a, b = make_network(cfg), OH.Network(cfg)
    assert [(k, tuple(v.shape)) for k, v in a.state_dict().items()] == [(k, tuple(v.shape)) for k, v in b.state_dict().items()]
    assert a.state_dict()["xyz_encoder.table"].shape == (16, 1 << 12, 2)
    assert torch.equal(a.state_dict()["xyz_encoder.aabb"], torch.tensor(SCENE_AABB))
    S.init_network_weights(b, seed=2)
    a.load_state_dict(b.state_dict())
    assert all(torch.equal(x, y) for x, y in zip(a.state_dict().values(), b.state_dict().values()))
    assert 2 * sum(p.numel() for n, p in a.named_parameters() if n.endswith("weight")) == mlp_flops_per_sample(cfg)
    # the table is drawn U(-1, 1) after the linears (features of O(1))
    t = b.xyz_encoder.table.detach()
    assert float(t.min()) >= -1.0 and float(t.max()) <= 1.0 and float(t.abs().mean()) > 0.4


def test_hashgrid_arguments_are_rejected():
    cfg = hash_cfg("cfg1")
    net = S.init_network_weights(make_network(hash_cfg("cfg1", hash_log2_size=12)), seed=0)
    with pytest.raises(ValueError, match="> 64"):
        make_network(hash_cfg("cfg1", hash_levels=16, hash_features=8))
    with pytest.raises(ValueError, match="hash_features=3"):
        make_network(hash_cfg("cfg1", hash_features=3))
    with pytest.raises(ValueError, match="hash_aabb"):
        make_network(hash_cfg("cfg1", hash_aabb=None))
    with pytest.raises(ValueError, match="xyz_encoding"):
        make_network(hash_cfg("cfg1", xyz_encoding="sh"))
    # the C ABI makes the same checks (pnr_program_host here; pnr_create shares them)
    for over, msg in ((dict(hash_levels=16, hash_features=8), b"E=128 > 64"), (dict(hash_features=3), b"hash_features=3"),
                      (dict(hash_aabb=None), b"hash_aabb"), (dict(hash_log2_size=30), b"hash_log2_size=30"),
                      (dict(hash_base_resolution=1e5), b"finest resolution")):
        c = hash_cfg("cfg1", **{**dict(hash_log2_size=12), **over})
        with pytest.raises(_capi.PnrError) as e:
            build(c, net)
        assert msg.decode() in str(e.value), (over, str(e.value))
    assert cfg.hash_levels * cfg.hash_features == 32


def test_pnr_config_ctypes_layout_matches_the_header(tmp_path):
    """Offsets of every pnr_config field (the ctypes mirror vs offsetof in a host program built against include/pnr.h)."""
    import shutil
    if not shutil.which("g++"):
        pytest.skip("no host compiler")
    fields = [f for f, _ in _capi.PnrConfig._fields_]
    src = tmp_path / "offsets.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(pnr_config, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(pnr_config));\n  return 0;\n}\n')
    exe = tmp_path / "offsets"
    subprocess.check_call(["g++", "-x", "c++", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got[:-1] == [getattr(_capi.PnrConfig, f).offset for f in fields]
    assert got[-1] == C.sizeof(_capi.PnrConfig)
