"""GPU tier of data-parallel training: pnr_adam_step bit for bit against a float32 restatement of its documented order;
FusedAdam against torch.optim.Adam, its state_dict both ways and the repack of the network it updates; G shards run one
after another against the whole batch; a real one-rank communicator against NetworkWrapper + FusedAdam bit for bit;
and two ranks on two GPUs (tests/dp2_worker.py)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import panopticnerf_b200 as PN
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.train import DataParallelWrapper, FusedAdam, NetworkWrapper

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32


# ------------------------------------------------------------------------------------------------ the kernel
def restate_adam(slices, p, m, v, beta1, beta2, eps, wd, lr, t):
    """The documented order of pnr_adam_step (include/pnr.h) in numpy float32, one rounding per operation."""
    with np.errstate(all="ignore"):
        g = slices[0].copy()
        for s in slices[1:]:
            g = g + s
        gsum = g.copy()
        if wd != 0:
            g = g + F32(wd) * p
        w1 = F32(1.0 - beta1)
        d = g - m
        m = m + w1 * d if w1 < 0.5 else g - d * (F32(1) - w1)
        v = v * F32(beta2) + (F32(1.0 - beta2) * g) * g
        step_size, bc2 = F32(lr / (1.0 - beta1 ** t)), F32((1.0 - beta2 ** t) ** 0.5)
        denom = np.sqrt(v) / bc2 + F32(eps)
        p = p + (-step_size) * (m / denom)
    return p, m, v, gsum


def adam_call(grads, p, m, v, G, P, ld, beta1, beta2, eps, wd, lr, t, grad_sum=None):
    a = _capi.PnrAdamArgs()
    a.P, a.ld_grad, a.G, a.beta1, a.beta2, a.eps, a.weight_decay = P, ld, G, beta1, beta2, eps, wd
    a.step_size, a.bc2_sqrt = lr / (1.0 - beta1 ** t), (1.0 - beta2 ** t) ** 0.5
    _capi.check(_capi.lib().pnr_adam_step(grads.data_ptr(), p.data_ptr(), m.data_ptr(), v.data_ptr(), C.byref(a),
                                          grad_sum.data_ptr() if grad_sum is not None else None, _capi.stream_ptr()),
                "pnr_adam_step")


def _same_bits(got, ref):
    """Bit-identical, NaN where the reference has NaN (any payload)."""
    got = got.cpu().numpy()
    gn, rn = np.isnan(got), np.isnan(ref)
    return bool((gn == rn).all() and (got[~gn].view(np.uint32) == ref[~rn].view(np.uint32)).all())


def _adam_case(P, G, ld, seed, poison=False):
    rng = np.random.default_rng(seed)
    grads = rng.standard_normal((G, ld)).astype(F32)
    if poison and P:
        idx = rng.choice(P, size=min(P, 12), replace=False)
        grads[1 % G, idx[0::3]] = np.nan
        grads[1 % G, idx[1::3]] = np.inf
        grads[1 % G, idx[2::3]] = -np.inf
    p = rng.standard_normal(P).astype(F32)
    m = (rng.standard_normal(P) * 0.1).astype(F32)
    v = np.abs(rng.standard_normal(P) * 1e-2).astype(F32)
    return grads, p, m, v


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("P", [0, 1, 3, 4, 5, (1 << 20) + 3, (1 << 24) + 1])
def test_adam_step_matches_the_float32_restatement(P, G):
    ld = P + (0, 3, 4)[(P + G) % 3]                        # ld_grad > P, on both the 16-byte and the scalar path
    wd = 0.01 if G % 2 else 0.0
    t = 10 ** 4 if P % 2 else 1
    beta1 = 0.3 if G == 3 else 0.9                         # 1 - beta1 >= 0.5: the other branch of torch's lerp
    hp = dict(beta1=beta1, beta2=0.999, eps=1e-8, wd=wd, lr=1e-3, t=t)
    grads, p, m, v = _adam_case(P, G, ld, seed=P * 31 + G)
    ref = restate_adam([grads[g, :P] for g in range(G)], p, m, v, **hp)
    outs = []
    for _ in range(2):                                    # two runs are bit-identical
        d = [torch.from_numpy(x.copy()).to(DEV) for x in (grads, p, m, v)]
        gs = torch.full((P,), 7.0, device=DEV)
        adam_call(d[0], d[1], d[2], d[3], G, P, ld, grad_sum=gs, **hp)
        outs.append(d[1:] + [gs])
    torch.cuda.synchronize()
    for got, want, name in zip(outs[0], ref, ("param", "exp_avg", "exp_avg_sq", "grad_sum")):
        assert _same_bits(got, want), name
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("G,ld", [(3, 1003), (8, 1006)])
def test_adam_step_propagates_nan_and_inf_as_the_restatement(G, ld):
    P = 1003
    hp = dict(beta1=0.9, beta2=0.999, eps=1e-8, wd=0.01, lr=1e-3, t=7)
    grads, p, m, v = _adam_case(P, G, ld, seed=G, poison=True)
    ref = restate_adam([grads[g, :P] for g in range(G)], p, m, v, **hp)
    assert np.isnan(ref[0]).sum() >= 8
    d = [torch.from_numpy(x.copy()).to(DEV) for x in (grads, p, m, v)]
    gs = torch.empty(P, device=DEV)
    adam_call(d[0], d[1], d[2], d[3], G, P, ld, grad_sum=gs, **hp)
    for got, want, name in zip(d[1:] + [gs], ref, ("param", "exp_avg", "exp_avg_sq", "grad_sum")):
        assert _same_bits(got, want), name


# ------------------------------------------------------------------------------------------------ FusedAdam
SHAPES = [(300, 37), (513,), (7, 3, 5), (64, 64)]


def _pairs(seed):
    g = torch.Generator().manual_seed(seed)
    init = [torch.randn(s, generator=g) for s in SHAPES]
    a = [torch.nn.Parameter(x.clone().to(DEV)) for x in init]
    b = [torch.nn.Parameter(x.clone().to(DEV)) for x in init]
    return a, b


def _groups(ps):
    return [{"params": ps[:2]}, {"params": ps[2:], "lr": 3e-3, "weight_decay": 0.0}]


def _set_grads(pa, pb, fused, gen):
    grads = [torch.randn(p.shape, generator=gen).to(DEV) for p in pa]
    for p, g in zip(pa, grads):
        p.grad = g.clone()
    fused.zero_grad()
    for p, g in zip(pb, grads):
        p.grad.copy_(g)


def _bound(p_ref, lr_sum, steps):
    return lr_sum * 2.0 ** -16 + steps * torch.finfo(torch.float32).eps * (p_ref.abs() + 4 * lr_sum)


def test_fused_adam_follows_torch_adam_with_a_scheduler():
    """50 steps of the same gradients with ExponentialLR(0.95), weight decay 0.01 on one group and 0 on the other.

    Bound per element: both optimisers compute the same formulas in fp32 and differ only in rounding: torch contracts
    some products into FMAs and divides by bc2_sqrt through its reciprocal, the kernel rounds every operation.  So a
    step's update differs by at most ~10 roundings of its own size, and that size is at most 4 lr_t for these betas
    (Cauchy-Schwarz over the exponential weights: |m_hat| / sqrt(v_hat) <= sqrt(1 - beta2) / (1 - beta1) *
    (1 - beta1) / sqrt((1 - beta2) (1 - beta1^2 / beta2)) < 2.3, with the bias corrections of t <= 50).  The moments' earlier
    differences enter the update too, damped by beta1 each step (<= 10 steps' worth) and under the square root of v
    (<= 50 steps' worth, halved).  All of this stays under 64 roundings of 4 lr_t = 2^-16 lr_t per step.  Once the
    parameters differ, each step's p + u can also round apart, by one ulp of |p| <= |p_torch| + 4 sum(lr_t).
    Sum over the steps: sum(lr_t) 2^-16 + 50 eps (|p_torch| + 4 sum(lr_t))."""
    pa, pb = _pairs(1)
    ta = torch.optim.Adam(_groups(pa), lr=1e-3, weight_decay=0.01, foreach=False)
    fb = FusedAdam(_groups(pb), lr=1e-3, weight_decay=0.01)
    sa, sb = (torch.optim.lr_scheduler.ExponentialLR(o, 0.95) for o in (ta, fb))
    gen = torch.Generator().manual_seed(2)
    lr_sum = [0.0, 0.0]
    for _ in range(50):
        _set_grads(pa, pb, fb, gen)
        lr_sum = [s + gr["lr"] for s, gr in zip(lr_sum, ta.param_groups)]
        ta.step()
        fb.step()
        sa.step()
        sb.step()
    assert [gr["lr"] for gr in ta.param_groups] == [gr["lr"] for gr in fb.param_groups]
    worst = 0.0
    for i, (a, b) in enumerate(zip(pa, pb)):
        err = (a.detach() - b.detach()).abs()
        bound = _bound(a.detach(), lr_sum[0 if i < 2 else 1], 50)
        worst = max(worst, float((err / bound).max()))
        assert (err <= bound).all(), f"parameter {i}: max error {float(err.max()):.3e}"
        assert not torch.equal(a.detach(), _pairs(1)[0][i].detach())      # they moved
    print(f"FusedAdam vs torch.optim.Adam after 50 steps: max error / bound = {worst:.3f}")

    # state_dict both ways, then one more step each
    pc = [torch.nn.Parameter(p.detach().clone()) for p in pb]
    tc = torch.optim.Adam(_groups(pc), lr=1e-3, foreach=False)
    tc.load_state_dict(fb.state_dict())
    pd = [torch.nn.Parameter(p.detach().clone()) for p in pa]
    fd = FusedAdam(_groups(pd), lr=1e-3)
    fd.load_state_dict(ta.state_dict())
    assert [gr["lr"] for gr in fd.param_groups] == [gr["lr"] for gr in ta.param_groups]
    assert float(fd.state[pd[0]]["step"]) == 50.0
    _set_grads(pa, pb, fb, gen)
    for p, q in zip(pc, pb):
        p.grad = q.grad.clone()
    fd.zero_grad()
    for p, q in zip(pd, pa):
        p.grad.copy_(q.grad)
    before = [p.detach().clone() for p in pb]
    for o in (ta, fb, tc, fd):
        o.step()
    lr1 = max(gr["lr"] for gr in ta.param_groups)
    for x, y in ((pc, pb), (pd, pa)):
        for i, (a, b) in enumerate(zip(x, y)):
            err = (a.detach() - b.detach()).abs()
            assert (err <= _bound(b.detach(), lr_sum[0] + lr1, 51)).all(), i
    assert not torch.equal(before[0], pb[0].detach())


def test_fused_adam_refuses_a_replaced_or_sparse_gradient():
    p = torch.nn.Parameter(torch.zeros(8, device=DEV))
    opt = FusedAdam([p])
    p.grad = torch.ones(8, device=DEV)                  # not the view into the flat gradient
    with pytest.raises(RuntimeError, match="view"):
        opt.step()
    p.grad = torch.ones(8, device=DEV).to_sparse()
    with pytest.raises(ValueError, match="sparse"):
        opt.step()
    opt.zero_grad(set_to_none=True)                   # zeroes in place; the views stay
    p.grad = None
    with pytest.raises(RuntimeError, match="None"):
        opt.step()
    opt.zero_grad()
    p.grad = opt._flat[0]["views"][0]
    p.data = torch.zeros(8, device=DEV)              # what module.to() or load_state_dict(assign=True) does
    with pytest.raises(RuntimeError, match="flat parameter buffer"):
        opt.step()


def _render_cfg(kind):
    if kind == "hashgrid":
        from oracle_hashgrid import hash_cfg
        return hash_cfg("cfg1", num_classes=5, num_instances=6, N_importance=8, hash_log2_size=14)
    return PN.make_cfg("cfg1", num_classes=5, num_instances=6, N_importance=8)


def _fresh_render(cfg, net, batch):
    """The render of a network built anew from `net`'s state_dict (packed from scratch)."""
    fresh = PN.make_network(cfg)
    fresh.load_state_dict({k: v.cpu() for k, v in net.state_dict().items()})
    return PN.make_renderer(cfg, fresh.to(DEV)).render(batch)


@pytest.mark.parametrize("kind", ["frequency", "hashgrid"])
def test_a_render_after_a_step_equals_a_fresh_network_with_the_same_state(kind):
    """The network is packed before FusedAdam moves its parameters (and a hash-grid network's table) into the flat
    buffers, packed again on those buffers, then stepped twice with a render between the steps.  Each step leaves
    every data_ptr() as it was, so only the version bump after the kernel's write makes the next render repack: a
    missing bump renders the weights of the previous step."""
    cfg = _render_cfg(kind)
    net = S.init_network_weights(PN.make_network(cfg), seed=5).to(DEV)
    ren = PN.make_renderer(cfg, net)
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, row0=20, rows=4).items()}
    before = ren.render(batch)                           # packs the weights and binds the table
    opt = FusedAdam(net.parameters(), lr=1e-2)
    moved = ren.render(batch)                            # repacked from the flat buffers, the table rebound
    for k in before:
        assert torch.equal(moved[k], before[k]), k
    g = torch.Generator().manual_seed(6)
    prev = moved
    for step in range(2):
        opt.zero_grad()
        for p in net.parameters():
            p.grad.copy_(torch.randn(p.shape, generator=g).to(DEV))
        opt.step()
        got = ren.render(batch)
        ref = _fresh_render(cfg, net, batch)
        assert not torch.equal(got["rgb_map"], prev["rgb_map"]), f"step {step}: the render did not change"
        for k in ref:
            assert torch.equal(got[k], ref[k]), f"step {step}: {k}"
        prev = got


class _FromRoot:
    """A one-rank stand-in for rank r > 0: broadcast(t) writes rank 0's tensors into t in place, in call order."""

    rank, world = 1, 2

    def __init__(self, root_tensors):
        self._src = iter(root_tensors)

    def broadcast(self, t):
        return t.copy_(next(self._src))


def test_the_wrapper_broadcast_repacks_a_network_already_packed():
    """A replica whose network was packed on its own parameters, inside FusedAdam's flat buffers, renders rank 0's
    parameters after the wrapper's broadcast wrote them in place (same data_ptr(): only the version bump repacks)."""
    cfg = _render_cfg("frequency")
    net = S.init_network_weights(PN.make_network(cfg), seed=7).to(DEV)
    root = S.init_network_weights(PN.make_network(cfg), seed=8).to(DEV)
    FusedAdam(net.parameters())
    batch = {k: v.to(DEV) for k, v in S.make_batch(cfg, row0=20, rows=4).items()}
    ren = PN.make_renderer(cfg, net)
    own = ren.render(batch)
    DataParallelWrapper(cfg, net, device=DEV, comm=_FromRoot([p.detach() for p in root.parameters()]))
    got = ren.render(batch)
    ref = PN.make_renderer(cfg, root).render(batch)
    assert not torch.equal(got["rgb_map"], own["rgb_map"])
    for k in ref:
        assert torch.equal(got[k], ref[k]), k


@pytest.mark.parametrize("F", [2, 4])
def test_a_hash_table_off_its_vector_alignment_is_refused(F):
    """FusedAdam places every parameter 256 bytes apart in its flat buffer; a table that is not aligned to one corner's
    features (read as a float2 / float4) is refused by name instead of being read."""
    from oracle_hashgrid import hash_cfg
    cfg = hash_cfg("cfg1", hash_log2_size=10, hash_levels=4, hash_features=F)
    net = S.init_network_weights(PN.make_network(cfg), seed=1).to(DEV)
    ctx = net.pack()
    L = _capi.lib()
    table = net.xyz_encoder.table
    assert L.pnr_bind_hashgrid_table(C.c_void_p(ctx), table.data_ptr() + 4) == -1
    assert "not aligned" in L.pnr_last_error().decode()
    x = torch.rand(5, 3, device=DEV)
    out = torch.empty(5, 4 * F, device=DEV)
    e = net.xyz_encoder
    assert L.pnr_hashgrid_encode(x.data_ptr(), 5, None, table.data_ptr() + 4, e.L, e.F, e.T_log2, e.base, e.scale,
                                 out.data_ptr(), _capi.stream_ptr()) == -1
    assert "not aligned" in L.pnr_last_error().decode()
    assert L.pnr_bind_hashgrid_table(C.c_void_p(ctx), table.data_ptr()) == 0


# ------------------------------------------------------------------------------------------------ sharded training
class SimComm:
    """Rank `rank` of `world` whose exchanges the test performs itself (by stacking); nothing is broadcast."""

    def __init__(self, rank, world):
        self.rank, self.world = rank, world

    def broadcast(self, t):
        return t

    def allgather(self, t):
        raise AssertionError("the one-process simulation stacks the exchanges itself")


def cfg3(kind):
    kw = dict(render_path="staged", bound_by_primitives=True, perturb=1.0)
    if kind == "hashgrid":
        from oracle_hashgrid import hash_cfg
        return hash_cfg("cfg3", hash_log2_size=16, **kw)
    return PN.make_cfg("cfg3", **kw)


def train_batch(cfg, R, seed, step=8):
    """R rays of one synthetic frame with its primitives, supplied jitter u / u_fine and targets, on the device."""
    b = S.make_batch(cfg, seed=seed, row0=150, rows=(R * step + int(cfg.W_img) - 1) // int(cfg.W_img))
    b["rays"] = b["rays"][::step][:R].contiguous()
    g = torch.Generator().manual_seed(seed + 100)
    b.update(u=torch.rand(R, int(cfg.N_samples), generator=g), u_fine=torch.rand(R, int(cfg.N_importance), generator=g),
             rgb=torch.rand(R, 3, generator=g),
             depth=torch.where(torch.rand(R, generator=g) < 0.7, torch.rand(R, generator=g) * 40 + 5, torch.zeros(R)),
             pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    return {k: v.to(DEV) for k, v in b.items()}


def simulate_shards(cfg, net, fine, batch, G, opt, device=DEV):
    """One G-rank step's phases, shard after shard in this process, with the exchanges done by stacking.  Returns
    [(output, loss, stats)] per rank and each group's gradient slices stacked [G, P] (what the all-gather yields)."""
    ws = [DataParallelWrapper(cfg, net, fine, device=device, comm=SimComm(g, G)) for g in range(G)]
    shards = [w.shard(batch) for w in ws]
    counts = torch.stack([w.local_counts(s) for w, s in zip(ws, shards)]).sum(0).tolist()
    steps = [w.forward_local(s, counts) for w, s in zip(ws, shards)]
    gathered = torch.stack([s["exchange"] for s in steps])
    stacks = [torch.empty(G, g.numel(), device=device) for g in opt.flat_grads()]
    results = []
    for g, (w, s) in enumerate(zip(ws, steps)):
        loss, stats = w.finish(s, gathered)
        opt.zero_grad()
        loss.backward()
        for st, fg in zip(stacks, opt.flat_grads()):
            st[g].copy_(fg)
        results.append((s["output"], loss.detach(), stats))
    return results, stacks


def _nets(cfg, shared, seed):
    net = S.init_network_weights(PN.make_network(cfg), seed=seed).to(DEV)
    fine = None if shared else S.init_network_weights(PN.make_network(cfg), seed=seed + 1).to(DEV)
    return net, fine


def _params(net, fine):
    return list(net.parameters()) + ([] if fine is None else list(fine.parameters()))


@pytest.mark.parametrize("kind,shared,G,R", [
    ("frequency", False, 2, 161), ("frequency", False, 3, 160), ("frequency", False, 4, 150),
    ("frequency", False, 8, 42),                        # ceil(42 / 8) = 6 rays per shard: the last shard is empty
    ("frequency", True, 3, 160), ("frequency", True, 8, 42),
    ("hashgrid", False, 4, 150), ("hashgrid", True, 8, 42)])
def test_sharded_step_equals_the_whole_batch(kind, shared, G, R):
    cfg = cfg3(kind)
    net, fine = _nets(cfg, shared, seed=51)
    batch = train_batch(cfg, R, seed=9)
    params = _params(net, fine)
    opt = FusedAdam(params)
    whole = NetworkWrapper(cfg, net, fine)
    opt.zero_grad()
    _, loss_w, stats_w, _ = whole(batch)
    loss_w.backward()
    g_whole = opt.flat_grads()[0].clone()
    results, stacks = simulate_shards(cfg, net, fine, batch, G, opt)
    g_sum = stacks[0].sum(0)
    assert float(results[-1][1]) == pytest.approx(float(loss_w.detach()), rel=1e-5)
    tol = 2e-4 if net.precision == "bf16x3" else 1e-4
    worst = 0.0
    for p, off in zip(params, opt._flat[0]["offsets"]):
        n = p.numel()
        ref, got = g_whole[off:off + n].view_as(p), g_sum[off:off + n].view_as(p)
        rms = float(ref.pow(2).mean().sqrt())
        if rms == 0.0:
            assert torch.equal(got, ref)
            continue
        if p.dim() == 3:
            # the hash table: a few entries, gathered by many samples, lie far above the rest, and its fp32
            # atomics add in an order that varies from run to run, so one rounding of such an entry exceeds 1e-4 of
            # the RMS.  It is held elementwise to the tolerance form of the path's table-gradient test:
            # |got - ref| <= 1e-4 max(|ref|, RMS).
            e = float(((got - ref).abs() / ref.abs().clamp(min=rms)).max())
        else:
            e = float((got - ref).abs().max()) / rms
        worst = max(worst, e)
        assert e <= tol, f"{tuple(p.shape)}: {e:.2e} of the RMS"
    print(f"{kind} shared={shared} G={G} R={R}: max |sum of shards - whole| = {worst:.2e} of the RMS (table: of "
          f"max(|ref|, RMS))")
    for out, loss, stats in results:                 # global values, identical on every rank
        assert torch.equal(loss, results[0][1])
        assert int(stats["n_inst"]) == int(stats_w["n_inst"])
        for k, v in stats_w.items():
            if k != "n_inst":
                assert float(stats[k]) == pytest.approx(float(v), rel=1e-5, abs=1e-7), k
    assert int(stats_w["n_inst"]) > 0


def test_one_rank_communicator_equals_network_wrapper_and_fused_adam():
    """World = 1 through a real pnr_comm (NCCL all-gather and broadcast of one rank) is bit for bit the one-GPU step."""
    import torch.distributed as dist
    from panopticnerf_b200 import parallel
    cfg = cfg3("frequency")
    net_a, fine_a = _nets(cfg, False, seed=61)
    net_b, fine_b = copy.deepcopy(net_a), copy.deepcopy(fine_a)
    wa = NetworkWrapper(cfg, net_a, fine_a)
    oa = FusedAdam(_params(net_a, fine_a), lr=1e-3)
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        tg = parallel.TileGather(DEV)
        wb = DataParallelWrapper(cfg, net_b, fine_b, comm=tg)
        ob = FusedAdam(_params(net_b, fine_b), lr=1e-3, comm=tg)
        for s in range(5):
            batch = train_batch(cfg, 256, seed=70 + s, step=4)
            for w, o in ((wa, oa), (wb, ob)):
                o.zero_grad()
                _, loss, stats, _ = w(batch)
                loss.backward()
                o.step()
            for a, b in zip(_params(net_a, fine_a), _params(net_b, fine_b)):
                assert torch.equal(a.detach(), b.detach()), f"step {s}"
        for fa, fb in zip(oa._flat, ob._flat):
            assert torch.equal(fa["exp_avg_sq"], fb["exp_avg_sq"])
        tg.close()
    finally:
        dist.destroy_process_group()


def test_two_ranks_hold_identical_replicas():
    """tests/dp2_worker.py on two GPUs: broadcast at construction, replica identity after 5 steps for frequency and
    hash-grid networks, and for the frequency network equality with the one-process simulation of the two shards."""
    import socket
    import subprocess
    import sys
    from pathlib import Path
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    worker = Path(__file__).parent / "dp2_worker.py"
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(worker)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "DP2 OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
