"""GPU tier of the fixed-point hash-grid table gradient (pnr_hashgrid_backward_fixed, cfg.hash_grad = "fixed"): the
kernel against the numpy oracle (tests/oracle_hashgrid_fixed.py) bit for bit across shapes, sizes, point layouts,
magnitudes and non-finite gradients; independence of the order of the points, of the launch, of the process and of
graph capture; the derived error bound against float64; and hash-grid training that is reproducible bit for bit, on
one GPU, in the one-process shard simulation and on two ranks (tests/dp2_hashfixed_worker.py)."""
import hashlib
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import panopticnerf_b200 as PN
from oracle import reference_panoptic as OP
from oracle_hashgrid_fixed import F32, corners, level_scale, table_grad_fixed
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.train import FusedAdam, NetworkWrapper

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = Path(__file__).resolve().parent


def fixed_grad(x, aabb, g, L, F, T_log2, base, scale, grad_table=None):
    """pnr_hashgrid_backward_fixed on the device; x, g, aabb CPU or CUDA tensors; returns the CUDA grad_table."""
    xd = torch.as_tensor(x, dtype=torch.float32).reshape(-1, 3).contiguous().to(DEV)
    gd = torch.as_tensor(g, dtype=torch.float32).contiguous().to(DEV)
    ad = None if aabb is None else torch.as_tensor(aabb, dtype=torch.float32).reshape(6).contiguous().to(DEV)
    gt = (torch.zeros(L, 1 << T_log2, F) if grad_table is None else torch.as_tensor(grad_table)).contiguous().to(DEV)
    Lib = _capi.lib()
    nb = Lib.pnr_hashgrid_fixed_workspace_bytes(L, F, T_log2)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    _capi.check(Lib.pnr_hashgrid_backward_fixed(xd.data_ptr(), xd.shape[0], _capi.ptr(ad), gd.data_ptr(), L, F, T_log2,
                                                base, scale, gt.data_ptr(), ws.data_ptr(), nb, _capi.stream_ptr()),
                "pnr_hashgrid_backward_fixed")
    return gt


def assert_same_bits(got, ref, what=""):
    """Bit-identical, NaN exactly where the reference has NaN (any payload)."""
    got = got.detach().cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    gn, rn = np.isnan(got), np.isnan(ref)
    assert np.array_equal(gn, rn), f"{what}: NaN at {int(gn.sum())} entries, the oracle at {int(rn.sum())}"
    diff = got[~gn].view(np.uint32) != ref[~rn].view(np.uint32)
    assert not diff.any(), f"{what}: {int(diff.sum())} entries differ in their bits"


def points(layout, n, seed):
    g = torch.Generator().manual_seed(seed)
    if layout == "rays":                     # 256 coherent samples per ray through the unit cube, as in training
        R = (n + 255) // 256
        o = torch.rand(R, 1, 3, generator=g) * 0.2 + 0.4
        d = torch.nn.functional.normalize(torch.randn(R, 1, 3, generator=g), dim=-1) * 0.5
        t = torch.linspace(0, 1, 256)
        return (o + d * t[None, :, None]).reshape(-1, 3)[:n].clamp(0, 1).contiguous()
    if layout == "random":
        return torch.rand(n, 3, generator=g)
    return torch.full((n, 3), 0.3183) + torch.rand(n, 3, generator=g) * 1e-6      # one cell at every level


def check_case(x, aabb, g, L, F, T_log2, base, scale, grad_table=None, what=""):
    got = fixed_grad(x, aabb, g, L, F, T_log2, base, scale, grad_table)
    ref = table_grad_fixed(x, aabb, g, L, F, T_log2, base, scale, grad_table)
    assert_same_bits(got, ref, what)
    return got, ref


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("L,F,T_log2,base,scale,n", [(16, 2, 19, 16.0, 1.3819, 20000), (8, 4, 12, 4.0, 2.0, 5000),
                                                     (4, 1, 10, 2.0, 1.5, 300), (5, 8, 11, 3.0, 1.9, 999)])
def test_matches_the_oracle_at_the_atomic_paths_shapes(L, F, T_log2, base, scale, n):
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    gen = torch.Generator().manual_seed(n)
    x = torch.rand(n, 3, generator=gen) * 2.4 - 1.2
    up = torch.randn(n, L * F, generator=gen)
    check_case(x, aabb, up, L, F, T_log2, base, scale, what=f"L={L} F={F}")


@pytest.mark.parametrize("L,F,T_log2,base,scale", [(32, 1, 12, 2.0, 1.3), (8, 2, 14, 4.0, 1.8), (6, 4, 10, 2.0, 2.0),
                                                   (3, 8, 6, 2.0, 1.5), (32, 2, 4, 1.0, 1.2)])
def test_matches_the_oracle_across_features_levels_and_table_sizes(L, F, T_log2, base, scale):
    """F = 1, 2, 4, 8, L = 32, T = 2^4; every case has levels on both sides of the dense / hash switch."""
    dense = [(r + 1) ** 3 <= 1 << T_log2 for r in OP.hashgrid_resolutions(L, base, scale)]
    assert any(dense) and not all(dense)
    n = 3001
    x = points("random", n, seed=L + F)
    g = torch.randn(n, L * F, generator=torch.Generator().manual_seed(F))
    check_case(x, None, g, L, F, T_log2, base, scale, what=f"L={L} F={F} T=2^{T_log2}")


@pytest.mark.parametrize("layout", ["rays", "random", "one_cell"])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1 << 20])
def test_matches_the_oracle_across_sizes_and_layouts(n, layout):
    x = points(layout, n, seed=n)
    g = torch.randn(n, 32, generator=torch.Generator().manual_seed(n + 1)) * 1e-3
    check_case(x, None, g, 16, 2, 19, 16.0, 1.3819, what=f"n={n} {layout}")


@pytest.mark.parametrize("mag", [1e-30, 1e-7, 1e30, "subnormal"])
def test_magnitudes_from_subnormal_to_1e30(mag):
    n = 4099
    gen = torch.Generator().manual_seed(5)
    x = points("rays", n, seed=6)
    g = torch.randn(n, 16, generator=gen)
    if mag == "subnormal":
        g = g * 1e-40                                        # every value subnormal in fp32
        assert bool((g.abs() < torch.finfo(torch.float32).tiny).all())
    else:
        g = g * mag
    check_case(x, None, g, 8, 2, 14, 8.0, 1.5, what=f"|g| ~ {mag}")


def test_accumulates_onto_a_non_zero_table_as_one_fp32_add():
    n, L, F, T_log2 = 5000, 8, 2, 12
    gen = torch.Generator().manual_seed(9)
    x = points("random", n, seed=10)
    g = torch.randn(n, L * F, generator=gen) * 1e-2
    base = (torch.randn(L, 1 << T_log2, F, generator=gen) * 0.3).numpy()
    base[0, :5] = -0.0
    got, ref = check_case(x, None, g, L, F, T_log2, 4.0, 1.7, grad_table=base, what="onto a table")
    zero = table_grad_fixed(x, None, g, L, F, T_log2, 4.0, 1.7)
    assert np.array_equal(ref, (base + zero).astype(F32))


def test_non_finite_gradients_mark_their_corners_and_nothing_else():
    n, L, F = 3000, 8, 4
    gen = torch.Generator().manual_seed(12)
    x = points("rays", n, seed=13)
    g = torch.randn(n, L * F, generator=gen)
    idx = torch.randperm(n * L * F, generator=gen)[:30]
    g.view(-1)[idx[:10]] = float("nan")
    g.view(-1)[idx[10:20]] = float("inf")
    g.view(-1)[idx[20:]] = -float("inf")
    g[7, 3 * F:4 * F] = float("nan")                          # a whole level of one point
    got, ref = check_case(x, None, g, L, F, 11, 4.0, 1.6, what="NaN / Inf")
    assert 0 < int(np.isnan(ref).sum()) <= 34 * 8
    finite = table_grad_fixed(x, None, torch.where(torch.isfinite(g), g, torch.zeros_like(g)), L, F, 11, 4.0, 1.6)
    keep = ~np.isnan(ref)
    # the finite entries are the rule over the finite contributions (the scales ignore non-finite values)
    assert np.array_equal(ref[keep], finite[keep])


# ------------------------------------------------------------------------------------------------ order independence
def _case(seed=21, n=200_000):
    x = points("rays", n, seed=seed)
    g = torch.randn(n, 32, generator=torch.Generator().manual_seed(seed + 1)) * 1e-4
    return x, g


def test_independent_of_the_order_of_the_points_and_of_the_launch():
    x, g = _case()
    a = fixed_grad(x, None, g, 16, 2, 19, 16.0, 1.3819)
    b = fixed_grad(x, None, g, 16, 2, 19, 16.0, 1.3819)
    perm = torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(3))
    c = fixed_grad(x[perm], None, g[perm], 16, 2, 19, 16.0, 1.3819)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(a.view(torch.int32), c.view(torch.int32))


_CHILD = """
import hashlib, sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_hashgrid_fixed as T
x, g = T._case()
print(hashlib.sha256(T.fixed_grad(x, None, g, 16, 2, 19, 16.0, 1.3819).cpu().numpy().tobytes()).hexdigest())
"""


def test_a_second_process_gets_the_same_bytes():
    x, g = _case()
    mine = hashlib.sha256(fixed_grad(x, None, g, 16, 2, 19, 16.0, 1.3819).cpu().numpy().tobytes()).hexdigest()
    r = subprocess.run([sys.executable, "-c", _CHILD.format(root=str(HERE.parent), tests=str(HERE))],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.split()[-1] == mine


def test_a_cuda_graph_replay_equals_the_eager_call():
    x, g = _case(seed=31, n=50_000)
    eager = fixed_grad(x, None, g, 16, 2, 19, 16.0, 1.3819)
    xd, gd = x.to(DEV), g.to(DEV)
    gt = torch.zeros_like(eager)
    Lib = _capi.lib()
    nb = Lib.pnr_hashgrid_fixed_workspace_bytes(16, 2, 19)
    ws = torch.full((nb,), 0xAB, dtype=torch.uint8, device=DEV)          # garbage: the call zeroes what it uses
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        gt.zero_()
        _capi.check(Lib.pnr_hashgrid_backward_fixed(xd.data_ptr(), xd.shape[0], None, gd.data_ptr(), 16, 2, 19, 16.0, 1.3819,
                                                    gt.data_ptr(), ws.data_ptr(), nb, _capi.stream_ptr()))
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(gt.view(torch.int32), eager.view(torch.int32))


# ------------------------------------------------------------------------------------------------ error against float64
def test_within_the_derived_error_bound_of_float64_autograd():
    """Per entry: |got - ref| <= sum over its contributions of (2^-24 |w_k g| + 2^-(s_l + 1)), plus the final
    int64 -> double and double -> float roundings (2^-52 + 2^-24 of the result); ref = float64 autograd through the
    reference encoder (the same fp32 corner weights, float64 products and sums)."""
    L, F, T_log2, base, scale, n = 16, 2, 19, 16.0, 1.3819, 20000
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    gen = torch.Generator().manual_seed(n)
    x = torch.rand(n, 3, generator=gen) * 2.4 - 1.2
    up = torch.randn(n, L * F, generator=gen, dtype=torch.float64).float()
    t_ref = torch.zeros(L, 1 << T_log2, F, dtype=torch.float64, requires_grad=True)
    (OP.hashgrid_encode(x, aabb, t_ref, base, scale) * up.double()).sum().backward()
    ref = t_ref.grad.numpy()
    got = fixed_grad(x, aabb, up, L, F, T_log2, base, scale).cpu().numpy().astype(np.float64)
    gl = up.numpy().reshape(n, L, F).astype(np.float64)
    worst = 0.0
    for l, (w, idx) in enumerate(corners(x, aabb, L, 1 << T_log2, base, scale)):
        s = level_scale(float(np.abs(gl[:, l]).max()), n)
        mass = np.zeros((1 << T_log2, F))
        cnt = np.zeros(1 << T_log2)
        for k in range(8):
            np.add.at(mass, idx[:, k], np.abs(w[:, k, None].astype(np.float64) * gl[:, l]))
            np.add.at(cnt, idx[:, k], 1.0)
        bound = 2.0 ** -24 * mass + cnt[:, None] * 2.0 ** -(s + 1) + (2.0 ** -24 + 2.0 ** -52) * np.abs(got[l])
        err = np.abs(got[l] - ref[l])
        assert (err <= bound * (1 + 1e-9) + 1e-300).all(), f"level {l}"
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    print(f"fixed-point table gradient vs float64: worst error / bound = {worst:.3f}")


# ------------------------------------------------------------------------------------------------ training
def _cfg3_fixed():
    from test_gpu_data_parallel import cfg3
    cfg = cfg3("hashgrid")
    cfg.hash_grad = "fixed"
    return cfg


def _nets(cfg, shared, seed):
    net = S.init_network_weights(PN.make_network(cfg), seed=seed).to(DEV)
    fine = None if shared else S.init_network_weights(PN.make_network(cfg), seed=seed + 1).to(DEV)
    assert net.xyz_encoder.grad == "fixed"
    return net, fine


def _params(net, fine):
    return list(net.parameters()) + ([] if fine is None else list(fine.parameters()))


@pytest.mark.parametrize("shared", [False, True])
def test_two_training_runs_hold_identical_parameters_and_moments(shared):
    from test_gpu_data_parallel import train_batch
    cfg = _cfg3_fixed()
    runs = []
    for _ in range(2):
        net, fine = _nets(cfg, shared, seed=71)
        w = NetworkWrapper(cfg, net, fine)
        opt = FusedAdam(_params(net, fine), lr=1e-3)
        for s in range(5):
            batch = train_batch(cfg, 256, seed=80 + s, step=4)
            opt.zero_grad()
            _, loss, _, _ = w(batch)
            loss.backward()
            opt.step()
        runs.append(opt._flat)
    for fa, fb in zip(*runs):
        for k in ("param", "exp_avg", "exp_avg_sq"):
            assert torch.equal(fa[k].view(torch.int32), fb[k].view(torch.int32)), k


@pytest.mark.parametrize("shared,G,R", [(False, 4, 150), (True, 8, 42), (False, 2, 161)])
def test_shard_simulation_is_reproducible_and_sums_to_the_whole_batch(shared, G, R):
    from test_gpu_data_parallel import simulate_shards, train_batch
    cfg = _cfg3_fixed()
    net, fine = _nets(cfg, shared, seed=51)
    batch = train_batch(cfg, R, seed=9)
    params = _params(net, fine)
    opt = FusedAdam(params)
    opt.zero_grad()
    _, loss_w, _, _ = NetworkWrapper(cfg, net, fine)(batch)
    loss_w.backward()
    g_whole = opt.flat_grads()[0].clone()
    stacks = [simulate_shards(cfg, net, fine, batch, G, opt)[1][0].clone() for _ in range(2)]
    assert torch.equal(stacks[0].view(torch.int32), stacks[1].view(torch.int32))
    g_sum = stacks[0].sum(0)
    tol = 2e-4 if net.precision == "bf16x3" else 1e-4
    worst = 0.0
    for p, off in zip(params, opt._flat[0]["offsets"]):
        ref, got = g_whole[off:off + p.numel()], g_sum[off:off + p.numel()]
        rms = float(ref.pow(2).mean().sqrt())
        if rms == 0.0:
            assert torch.equal(got, ref)
            continue
        e = float((got - ref).abs().max()) / rms
        worst = max(worst, e)
        assert e <= tol, f"{tuple(p.shape)}: {e:.2e} of the RMS"
    print(f"hash_grad=fixed shared={shared} G={G} R={R}: max |sum of shards - whole| = {worst:.2e} of the RMS")


def test_thirty_steps_lower_the_loss():
    from test_gpu_data_parallel import train_batch
    cfg = _cfg3_fixed()
    net, fine = _nets(cfg, False, seed=41)
    w = NetworkWrapper(cfg, net, fine)
    opt = FusedAdam(_params(net, fine), lr=1e-3)
    batch = train_batch(cfg, 512, seed=12, step=2)
    gen = torch.Generator().manual_seed(13)
    losses = []
    for _ in range(30):
        batch["u"] = torch.rand(512, int(cfg.N_samples), generator=gen).to(DEV)
        batch["u_fine"] = torch.rand(512, int(cfg.N_importance), generator=gen).to(DEV)
        opt.zero_grad()
        _, loss, _, _ = w(batch)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    # the jitter is redrawn every step, so the loss is compared over three steps at either end (the run is reproducible
    # bit for bit: the margin is that of one fixed sequence of losses)
    assert np.mean(losses[-3:]) < 0.98 * np.mean(losses[:3]), losses


def test_two_ranks_equal_the_one_process_simulation():
    """tests/dp2_hashfixed_worker.py on two GPUs: with hash_grad = "fixed" the two ranks hold, after 5 steps, the
    parameters and moments of the one-process simulation of their shards, bit for bit."""
    import socket
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(HERE / "dp2_hashfixed_worker.py")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "DP2 HASHFIXED OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
