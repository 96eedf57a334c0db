"""One `NetworkWrapper` iteration per case against the float64 oracle chain pinned to the device's own decisions
(tests/oracle_pinned.py), every link element by element.

The decisions are the ones the backward pass took, collected per pass from the rays, depths and network the wrapper
used: trunk layers 0 .. D-2 from the activations `backward_trunk(..., stash=True)` keeps, the last trunk layer from
`trunk_forward`, the view and head ReLUs from the `_lin` calls of `mlp_backward._tail` on that h, the density from
`forward_rays` (+ the batch's noise), the depth sign, clamp branch and instance target from the wrapper's outputs.
`network_backward` is wrapped (pytest's monkeypatch) to record each pass's d(loss)/d(raw); one pass's gradients are
recomputed from it bit for bit, which shows these calls repeat what the wrapper's backward did.

The float64 chain runs on the device (float64 is not touched by TF32) and is checked in this order, so a failure
names its link:
  maps     coarse and fine, per ray at the compositing stage's tolerances (tests/test_gpu_stage_limits.py) against
           the float64 compositing of the pass's raw from `forward_rays` (the compositing link: the float64 chain's
           own raw differs from the device's by the MLP forward's error, which moved a weight by 1.1e-4 of its ray's
           largest on the mesh case's first H100 run);
  loss     the total and each term within 1e-4;
  d_raw    each pass per sample within 1e-4 of the ray's largest |ref| per channel group, plus the fp32
           transmittance floor derived in `oracle_pinned.d_raw_bound`, against the float64 compositing and loss
           backward of the pass's own raw (the links alone, as for the maps);
  params   every gradient of every network, the hash table included, element by element against the float64
           network backward (pinned) of the device's own recorded d_raw: |got - ref| <= tol max(|ref|, RMS(ref)),
           tol = 1e-4 (fp16x3) / 2e-4 (bf16x3), the per-network contract as
           `test_network_backward_every_parameter` asserts it; a zero reference exactly zero.  The atomic hash-table
           gradient adds (n + 1) 2^-24 sum |term| per entry, the bound of an fp32 sum of n terms in any order.
With the decisions pinned the chain is linear in d_raw, so the whole chain's gradient differs from the params
reference exactly by the float64 backward of (device d_raw - float64 d_raw): the links above account for all of the
end-to-end difference.  Its ratio to tol RMS(ref) is printed, not asserted: measured on the H100 it reaches 8.5 on the
layers fed gamma(x) (columns of |x| up to ~60 m), the density bias and the hash table, where d_raw differences of
~1e-5 of each ray's largest add up over 30 000 samples with cancellation; and tol RMS(ref) alone is not met by the
network backward either on elements far above the RMS (layer 0's x columns, the skip layer, coarse hash levels).
Each check prints its largest error as a share of its bound, and each pass its number of pinned flips.
The compositing backward has no softmax semantics (it refuses sem_activation = "softmax" by name), so the case with
white background, noise and label weights trains on semantic logits, and the refusal is asserted."""
import pytest
import torch

import oracle_pinned as OPN
from oracle import reference_renderer as O
import panopticnerf_b200 as PN
from panopticnerf_b200 import _capi, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from panopticnerf_b200.lib.train import NetworkWrapper
from panopticnerf_b200.lib.train import mlp_backward as MB

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
TOL = {"fp16x3": 1e-4, "bf16x3": 2e-4}


def _dev(b):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()}


def _oracle_net(cfg, net):
    """The float64 oracle of a product network, on the device (a hash grid's encoder stays on the CPU, where the
    oracle encoder runs)."""
    if getattr(net, "hashgrid", False):
        from oracle_hashgrid import oracle_like
        onet = oracle_like(net, cfg, F64)
        for name, mod in onet.named_children():
            if name != "xyz_encoder":
                mod.to(DEV)
        return onet
    onet = O.Network(cfg).double()
    onet.load_state_dict({k: v.detach().cpu().double() for k, v in net.state_dict().items()})
    return onet.to(DEV)


def _batch(cfg, R, seed, step=8, depth=True, labels=True):
    """R rays of one synthetic frame with its primitives, jitter and targets: some rays without a depth target, some
    ignored labels."""
    b = S.make_batch(cfg, seed=seed, row0=150, rows=(R * step + int(cfg.W_img) - 1) // int(cfg.W_img))
    b["rays"] = b["rays"][::step][:R].contiguous()
    g = torch.Generator().manual_seed(seed + 100)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    b.update(u=torch.rand(R, N, generator=g), u_fine=torch.rand(R, Ni, generator=g), rgb=torch.rand(R, 3, generator=g))
    if depth:
        b["depth"] = torch.where(torch.rand(R, generator=g) < 0.7, torch.rand(R, generator=g) * 40 + 5, torch.zeros(R))
    if labels:
        b["pseudo_label"] = torch.randint(-1, int(cfg.num_classes), (R,), generator=g)
    return b


def device_decisions(net, rays, z, noise=None, std=0.0):
    """The ReLU and density decisions the backward pass of one pass takes, from the calls it makes; and the pass's
    raw (`forward_rays`, what the compositing kernel composited)."""
    D, W = net.D, net.W
    R, N = z.shape
    with torch.no_grad():
        _, st = net.backward_trunk(torch.zeros(R * N, W, device=DEV), rays=rays, z=z, stash=True)
        pins = {f"pts_linears.{i}": st[i] > 0 for i in range(D - 1)}
        del st
        h = net.trunk_forward(rays=rays, z=z)
        pins[f"pts_linears.{D - 1}"] = h > 0
        pr = net.precision if net.precision in ("fp16x3", "bf16x3") else "fp16x3"
        vd = (rays[:, 3:] / rays[:, 3:].norm(dim=-1, keepdim=True))[:, None, :].expand(-1, N, -1).reshape(-1, 3)
        ed = P.embed(vd.contiguous(), net.Ld)
        feat = MB._lin(net.feature_linear, h, pr)
        pad = (-(feat.shape[1] + ed.shape[1])) % 4
        parts = [feat, ed] + ([feat.new_zeros(feat.shape[0], pad)] if pad else [])
        pins["views_linears.0"] = MB._lin(net.views_linears[0], torch.cat(parts, -1), pr) > 0
        if net.C > 0:
            pins["semantic_linears.0"] = MB._lin(net.semantic_linears[0], h, pr) > 0
        if net.K > 0:
            pins["instance_linears.0"] = MB._lin(net.instance_linears[0], h, pr) > 0
        raw = net.forward_rays(rays, z)
        s = raw[..., 3:4] + noise[..., None] * std if std > 0.0 else raw[..., 3:4]
        pins["sigma"] = s[..., 0] > 0
    return pins, raw


@pytest.fixture
def record_d_raw(monkeypatch):
    """{(id(net), samples per ray): d_raw} of every network_backward call the wrapper's backward makes."""
    rec = {}
    orig = MB.network_backward

    def spy(net, d_raw, **kw):
        rec[(id(net), kw["z"].shape[1])] = d_raw.detach().clone()
        return orig(net, d_raw, **kw)
    monkeypatch.setattr(MB, "network_backward", spy)
    rec["orig"] = orig
    return rec


def _grads(net):
    return {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in net.named_parameters()}


def _atomic(cfg, ref):
    """The table gradient's fp32 atomics: (n + 1) 2^-24 sum |term| per entry (`oracle_pinned.network_grads`) on top
    of the contract; the fixed-point path is order-free and gets nothing."""
    a = ref.get("xyz_encoder.table:atomic")
    return {"xyz_encoder.table": a} if a is not None and str(getattr(cfg, "hash_grad", "atomic")) == "atomic" else None


def run_chain(cfg, net, fine, b, rec, what):
    """One wrapper iteration on batch b, the pinned oracle of it and every check.  Returns (device gradients per
    distinct network, the oracle's result, the oracle's inputs and pins) for further use."""
    prec = str(cfg.precision)
    onet = _oracle_net(cfg, net)
    onet_f = None if int(cfg.N_importance) == 0 else (onet if fine is None else _oracle_net(cfg, fine))
    db = _dev(b)
    wrapper = NetworkWrapper(cfg, net, fine)
    out, loss, stats, _ = wrapper(db)
    loss.backward()
    assert net.range_status() == 0 and (fine is None or fine.range_status() == 0)
    fnet = net if fine is None else fine
    std = float(getattr(cfg, "raw_noise_std", 0.0))
    inst = "instance_map" in out and "fixed_instance_map" in out
    rays = db["rays"]
    roles = ["coarse", "fine"] if onet_f is not None else ["coarse"]
    zs = {"coarse": out["z_vals_0"] if onet_f is not None else out["z_vals"], "fine": out["z_vals"]}
    ob = dict(rays=b["rays"], C=net.C, K=net.K, white_bkgd=bool(cfg.white_bkgd), mask_outside=bool(cfg.mask_outside),
              raw_noise_std=std, sem_activation=str(cfg.sem_activation), rgb=b["rgb"], depth=b.get("depth"),
              pseudo_label=b.get("pseudo_label"), pseudo_weight=b.get("pseudo_weight"),
              weights=wrapper.weights if inst else wrapper.weights[:4], inst_min_weight=wrapper.inst_min_weight)
    has_boxes = "box_id" in out
    if has_boxes:
        ob.update(box_sem=b["box_sem"], box_inst=b["box_inst"])
    pins, raws = {}, {}
    for role, n in zip(roles, [net, fnet]):
        z = zs[role]
        ob[f"z_{role}"] = z.cpu()
        if has_boxes:
            ob[f"sb_{role}"] = (out["sample_box"] if role == roles[-1] else
                                O.tag_samples(z.cpu(), *(out[k].cpu() for k in ("box_id", "t_in", "t_out")))).to(DEV)
        nz = db.get("noise" if role == "coarse" else "noise_fine")
        if std > 0.0:
            ob[f"noise_{role}"] = nz
        pins[role], raws[role] = device_decisions(n, rays, z, nz, std)
    m1 = {k: out[k] for k in out}
    if "depth" in b:
        pins["depth_sign"] = torch.sign(m1["depth_map"].detach() - db["depth"])
    if "pseudo_label" in b and net.C > 0:
        lab = db["pseudo_label"].clamp(0, net.C - 1).long()[:, None]
        if "fixed_semantic_map" in m1:
            pins["fix_clamp"] = m1["fixed_semantic_map"].detach().gather(1, lab)[:, 0] >= 1e-8
        if str(cfg.sem_activation) == "softmax":
            pins["sem_clamp"] = m1["semantic_map"].detach().gather(1, lab)[:, 0] >= 1e-8
    if inst:
        pins["inst_label"] = out["inst_label"]
    ref = OPN.iteration((onet, onet_f), ob, pins=pins, precision=prec)
    print(f"{what}: pinned flips {ref['flips']}")
    # maps: the compositing link, float64 compositing of the device's own raw
    for role in roles:
        got = {k[:-2]: v for k, v in out.items() if k.endswith("_0")} if (role == "coarse" and len(roles) == 2) else out
        raw64, z64 = raws[role].cpu().double(), zs[role].cpu().double()
        sb = ob.get(f"sb_{role}")
        nz = ob.get(f"noise_{role}")
        m64 = O.raw2outputs(raw64, z64, b["rays"][:, 3:].double(), raw_noise_std=std,
                            noise=None if nz is None else nz.cpu().double(), white_bkgd=bool(cfg.white_bkgd),
                            num_classes=net.C, num_instances=net.K, sem_activation=str(cfg.sem_activation),
                            sample_box=None if sb is None else sb.cpu(), box_sem=ob.get("box_sem"),
                            box_inst=ob.get("box_inst"), mask_outside=bool(cfg.mask_outside))
        worst = OPN.maps_ratio(got, m64, raw64, z64, net.C, net.K, bool(cfg.white_bkgd),
                               str(cfg.sem_activation) == "softmax")
        print(f"{what} {role} maps: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
        assert max(worst.values()) <= 1.0, (role, worst)
    # loss
    terms = ["rgb", "depth", "sem", "fix"] + (["inst"] if inst else [])
    got_t = torch.stack([stats[t + "_loss"].double() for t in terms]).to(DEV)
    e_t = (got_t - ref["terms"]).abs()
    assert bool((e_t[ref["terms"] == 0] == 0).all()), "a term the float64 chain has as 0 is not 0"
    r_t = float((e_t / (1e-4 * ref["terms"].abs())).nan_to_num(0.0).max())
    r_l = abs(float(loss.detach()) - float(ref["total"])) / (1e-4 * abs(float(ref["total"])))
    print(f"{what} loss: total {r_l:.2e}, terms {r_t:.2e} of the bound")
    assert r_l <= 1.0 and r_t <= 1.0
    # d_raw
    own = OPN.iteration((onet, onet_f), ob, pins=pins, precision=prec, raw_from=raws)
    for role, n in zip(roles, [net, fnet]):
        got = rec[(id(n), zs[role].shape[1])]
        e = OPN.d_raw_ratio(got, own, role, net.C, net.K)
        print(f"{what} {role} d_raw: largest error / bound = {e:.3e}")
        assert e <= 1.0, role
    # every parameter: the network-backward link on the device's own d_raw; end to end reported
    mine = [_grads(net)] + ([_grads(fine)] if fine is not None else [])
    up = {role: rec[(id(n), zs[role].shape[1])] for role, n in zip(roles, [net, fnet])}
    link = OPN.network_grads((onet, onet_f), ob, pins, up, prec)
    for i, (g, r, r_e2e) in enumerate(zip(mine, link, ref["grads"])):
        ratios = OPN.param_ratios(g, r, TOL[prec], extra=_atomic(cfg, r))
        print(f"{what} network {i} network backward, largest error / bound: " + ", ".join(f"{k} {v:.2e}" for k, v in ratios.items()))
        e2e = OPN.param_ratios(g, r_e2e, TOL[prec], floor_only=True)
        k = max(e2e, key=e2e.get)
        print(f"{what} network {i} end to end, largest error / (tol RMS): {k} {e2e[k]:.2e}")
        bad = {k: v for k, v in ratios.items() if not v <= 1.0}
        assert not bad, bad
    ref["up"], ref["raws"] = up, raws
    return mine, ref, ob, pins, out


# ------------------------------------------------------------------------------------------------ the cases
def _cfg3(**over):
    kw = dict(render_path="staged", bound_by_primitives=True, perturb=1.0, check_range=True)
    kw.update(over)
    return PN.make_cfg("cfg3", **kw)


def _weighted(b, seed):
    g = torch.Generator().manual_seed(seed)
    b["pseudo_weight"] = 0.25 + torch.rand(b["rays"].shape[0], generator=g)
    return b


@pytest.mark.parametrize("shared,precision", [(False, "fp16x3"), (True, "fp16x3"), (False, "bf16x3")],
                         ids=["separate", "shared", "bf16x3"])
def test_cfg3_iteration_every_link(shared, precision, record_d_raw):
    """Cases 1 - 3: cfg3 networks, 64 + 128 samples, primitives, fixed maps, all five terms, rays without a depth
    target and ignored labels; separate or shared fine network; fp16x3 and bf16x3."""
    cfg = _cfg3(precision=precision)
    net = S.init_network_weights(PN.make_network(cfg), seed=21).to(DEV)
    fine = None if shared else S.init_network_weights(PN.make_network(cfg), seed=22).to(DEV)
    b = _batch(cfg, 160, seed=7)
    assert bool((b["depth"] == 0).any()) and bool((b["pseudo_label"] < 0).any())
    mine, ref, ob, pins, out = run_chain(cfg, net, fine, b, record_d_raw, f"cfg3 {precision} shared={shared}")
    assert int((out["inst_label"] >= 0).sum()) >= 20
    if not shared:      # the decisions collected again are the ones the backward took: one pass recomputed, same bits
        again = record_d_raw["orig"](fine, record_d_raw[(id(fine), out["z_vals"].shape[1])], rays=_dev(b)["rays"],
                                     z=out["z_vals"])
        for n, p in fine.named_parameters():
            assert torch.equal(again[n], p.grad), n


def test_cfg2_without_heads_on_the_128_row_kernel(record_d_raw):
    """Case 4: cfg2 (no heads: its forward program runs on the 128-sample tiles), colour and depth terms."""
    cfg = PN.make_cfg("cfg2", render_path="staged", N_importance=128, perturb=1.0, check_range=True)
    net = S.init_network_weights(PN.make_network(cfg), seed=23).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=24).to(DEV)
    b = _batch(cfg, 256, seed=8, labels=False)
    run_chain(cfg, net, fine, b, record_d_raw, "cfg2")


@pytest.mark.parametrize("hash_grad", ["atomic", "fixed"])
def test_hash_grid_iteration_every_link(hash_grad, record_d_raw):
    """Case 5: a cfg3 hash-grid network (shared), both table-gradient paths."""
    from oracle_hashgrid import hash_cfg
    cfg = hash_cfg("cfg3", render_path="staged", bound_by_primitives=True, perturb=1.0, hash_log2_size=15,
                   hash_grad=hash_grad, check_range=True)
    net = S.init_network_weights(PN.make_network(cfg), seed=41).to(DEV)
    b = _batch(cfg, 160, seed=12)
    mine, ref, *_ = run_chain(cfg, net, None, b, record_d_raw, f"hash grid {hash_grad}")
    assert float(mine[0]["xyz_encoder.table"].abs().sum()) > 0


def test_mesh_primitives_with_mask_outside(record_d_raw):
    """Case 6: the mesh-primitive batch of test_gpu_mesh_primitives.py with bound_by_primitives, mask_outside and
    perturb = 1."""
    from test_gpu_mesh_primitives import _mesh_batch
    cfg = _cfg3(mask_outside=True)
    net = S.init_network_weights(PN.make_network(cfg), seed=31).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=32).to(DEV)
    R = 400
    b = _mesh_batch(cfg, R, seed=3, row0=230, step=4)
    g = torch.Generator().manual_seed(9)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    b.update(u=torch.rand(R, N, generator=g), u_fine=torch.rand(R, Ni, generator=g), rgb=torch.rand(R, 3, generator=g),
             depth=torch.rand(R, generator=g) * 40 + 5, pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    b["box_inst"] = torch.arange(b["box_center"].shape[0], dtype=torch.int32) % int(cfg.num_instances)
    _, _, ob, _, out = run_chain(cfg, net, fine, b, record_d_raw, "meshes")
    assert bool((out["box_id"] >= 64).any()) and bool((ob["sb_fine"] < 0).any())


def test_white_background_noise_and_label_weights(record_d_raw):
    """Case 7: white_bkgd, raw_noise_std > 0 with the batch's noise / noise_fine and pseudo_weight; the compositing
    backward's refusal of softmax semantics by name."""
    cfg = _cfg3(white_bkgd=True, raw_noise_std=0.3)
    net = S.init_network_weights(PN.make_network(cfg), seed=51).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=52).to(DEV)
    R = 160
    b = _weighted(_batch(cfg, R, seed=9), 10)
    g = torch.Generator().manual_seed(11)
    b.update(noise=torch.randn(R, int(cfg.N_samples), generator=g),
             noise_fine=torch.randn(R, int(cfg.N_samples) + int(cfg.N_importance), generator=g))
    run_chain(cfg, net, fine, b, record_d_raw, "white noise weights")
    soft = _cfg3(sem_activation="softmax")
    w = NetworkWrapper(soft, S.init_network_weights(PN.make_network(soft), seed=1).to(DEV))
    _, loss, _, _ = w(_dev(_batch(soft, 32, seed=1)))
    with pytest.raises(_capi.PnrError, match="softmax"):
        loss.backward()


def test_sequence_table_with_a_moving_box(record_d_raw):
    """Case 8: a sequence table (static boxes + per-frame dynamic blocks) and ray_frame, the setup of
    test_gpu_sequence_primitives.py."""
    from test_gpu_sequence_primitives import _seq_batch
    cfg = _cfg3()
    net = S.init_network_weights(PN.make_network(cfg), seed=61).to(DEV)
    fine = S.init_network_weights(PN.make_network(cfg), seed=62).to(DEV)
    R = 200
    b = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in _seq_batch(cfg, R, seed=11).items()}
    g = torch.Generator().manual_seed(12)
    b.update(rgb=torch.rand(R, 3, generator=g), depth=torch.rand(R, generator=g) * 40 + 5,
             pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    _, _, _, _, out = run_chain(cfg, net, fine, b, record_d_raw, "sequence")
    assert bool((out["box_id"] >= 48).any()), "no ray met a dynamic box"


# ------------------------------------------------------------------------------------------------ power
def test_the_element_wise_check_rejects_each_deliberate_change(record_d_raw):
    """The device's iteration against a reference built with one deliberate change at a time (w_inst x 1.01; the
    coarse colour term dropped for a shared network; mask_outside left out of the backward; half of a head's rows
    1 % off): each is rejected by the link it changes - d_raw of a pass, or the network backward on the tensor it
    affects.  Also prints whether cosine >= 0.999 with the norm within 1 % (end to end) would have accepted it."""
    cfg = _cfg3(mask_outside=True)
    net = S.init_network_weights(PN.make_network(cfg), seed=71).to(DEV)
    b = _batch(cfg, 160, seed=13)
    mine, ref, ob, pins, _ = run_chain(cfg, net, None, b, record_d_raw, "power: unchanged")
    onet = _oracle_net(cfg, net)
    for edit in OPN.EDITS:
        bad = OPN.iteration((onet, onet), ob, pins=pins, edit=edit)
        bad_links = OPN.iteration((onet, onet), ob, pins=pins, edit=edit, raw_from=ref["raws"])
        d_raw = {role: OPN.d_raw_ratio(ref["up"][role], bad_links, role, net.C, net.K) for role in ("coarse", "fine")}
        link = OPN.network_grads((onet, onet), ob, pins, ref["up"], edit=edit)[0]
        rejected = {k: v for k, v in OPN.param_ratios(mine[0], link, TOL["fp16x3"]).items() if v > 1.0}
        old = OPN.old_criterion_accepts(mine[0], bad["grads"][0])
        print(f"power: {edit}: d_raw {d_raw['coarse']:.1f} / {d_raw['fine']:.1f} x the bound, network backward rejected "
              f"on {sorted(rejected)}; the cosine / norm criterion would have {'accepted' if old else 'rejected'} it")
        if edit == "head_rows":
            assert "instance_linears.1.weight" in rejected
        else:
            assert max(d_raw.values()) > 1.0, edit


def check_single_pass(cfg, net, rays, z, batch, weights, total, rec, what):
    """`training_step` (one pass, no primitives) against the pinned float64 chain: the total within 1e-4, d_raw per
    ray, and every parameter's gradient (in p.grad) against the float64 network backward of the step's own recorded
    d_raw (rec: the `record_d_raw` fixture), as `run_chain` checks them.  rays, z, batch: the step's device inputs."""
    onet = _oracle_net(cfg, net)
    pins = {"coarse": device_decisions(net, rays, z)[0]}
    if "depth" in batch:
        out = P.raw2outputs(net.forward_rays(rays, z), z, rays, num_classes=net.C, num_instances=net.K)
        pins["depth_sign"] = torch.sign(out["depth_map"] - batch["depth"])
    ob = dict(rays=rays.cpu(), z_coarse=z.cpu(), rgb=batch["rgb"], depth=batch.get("depth"),
              pseudo_label=batch.get("pseudo_label"), weights=tuple(weights))
    prec = str(cfg.precision)
    ref = OPN.iteration((onet, None), ob, pins=pins, precision=prec)
    print(f"{what}: pinned flips {ref['flips']}")
    assert abs(float(total) - float(ref["total"])) <= 1e-4 * abs(float(ref["total"]))
    up = rec[(id(net), z.shape[1])]
    own = OPN.iteration((onet, None), ob, pins=pins, precision=prec, raw_from={"coarse": net.forward_rays(rays, z)})
    e = OPN.d_raw_ratio(up, own, "coarse", net.C, net.K)
    print(f"{what} d_raw: largest error / bound = {e:.3e}")
    assert e <= 1.0
    link = OPN.network_grads((onet, None), ob, pins, {"coarse": up}, prec)[0]
    ratios = OPN.param_ratios(_grads(net), link, TOL[prec], extra=_atomic(cfg, link))
    print(f"{what} network backward, largest error / bound: " + ", ".join(f"{k} {v:.2e}" for k, v in ratios.items()))
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, bad
