"""CPU tier of the pinned training-chain oracle (tests/oracle_pinned.py).

- No-op pinning: with every decision taken from its own float64 value, the pinned chain is the plain oracle chain -
  autograd through O.Network, O.raw2outputs, reference_losses.losses and oracle_instance.instance_loss - bit for bit,
  for every parameter's gradient and for d(loss)/d(raw) of both passes.
- Point formation: the fp32 points and view directions equal numpy float32 mul-then-add (and sqrt, divide) bit for bit.
- Stand-in device: the same chain run in fp32 autograd plays the device.  Its own ReLU, density, depth-sign, clamp
  and instance decisions pin the float64 chain, which then meets the element-wise checks of
  tests/test_gpu_train_chain.py; at the size of its first case the fp32 run flips at least one unit, which is why
  pinning is needed.  A flipped unit far from zero is refused by the margin guard.
- Power: the deliberate changes of the reference (w_inst x 1.01, the coarse colour term dropped for a shared network,
  mask_outside left out of the backward, half of a head's rows 1 % off) are each rejected by the element-wise check."""
import numpy as np
import pytest
import torch

import oracle_pinned as OPN
import oracle_instance as OI
from oracle import reference_losses as OL
from oracle import reference_renderer as O
from panopticnerf_b200 import make_cfg, make_network, synthetic as S

TOL = 1e-4


def _nets(cfg, shared, dtype, seed=21):
    out = []
    for s in (seed, None if shared else seed + 1):
        if s is None:
            out.append(out[0])
            continue
        net = S.init_network_weights(make_network(cfg), seed=s)
        onet = O.Network(cfg).to(dtype)
        onet.load_state_dict({k: v.detach().to(dtype) for k, v in net.state_dict().items()})
        out.append(onet)
    return out


def _batch(cfg, R, seed, nets32, mask_outside=False, noise=False):
    """The inputs a device iteration hands the oracle, made on the CPU: rays of a synthetic frame and its primitives,
    coarse depths with jitter and fine depths sampled from the fp32 coarse weights (the oracle renderer), tags, targets
    (some rays without depth, some ignored labels, label weights)."""
    full = S.make_batch(cfg, seed=seed, row0=150, rows=(R * 8 + int(cfg.W_img) - 1) // int(cfg.W_img))
    rays = full["rays"][::8][:R].contiguous()
    g = torch.Generator().manual_seed(seed + 100)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    b = dict(full, rays=rays, u=torch.rand(R, N, generator=g), u_fine=torch.rand(R, Ni, generator=g), perturb=1.0)
    with torch.no_grad():
        out = O.Renderer(cfg, *nets32).render(b)
    C, K = int(cfg.num_classes), int(cfg.num_instances)
    box = (out["box_id"], out["t_in"], out["t_out"])
    res = dict(rays=rays, z_coarse=out["z_vals_0"], z_fine=out["z_vals"], sb_coarse=O.tag_samples(out["z_vals_0"], *box),
               sb_fine=out["sample_box"], box_sem=full["box_sem"], box_inst=full["box_inst"], mask_outside=mask_outside,
               rgb=torch.rand(R, 3, generator=g),
               depth=torch.where(torch.rand(R, generator=g) < 0.7, torch.rand(R, generator=g) * 40 + 5, torch.zeros(R)),
               pseudo_label=torch.randint(-1, C, (R,), generator=g), pseudo_weight=0.5 + torch.rand(R, generator=g),
               weights=(1.0, 0.1, 0.5, 2.0, 0.7), inst_min_weight=0.5)
    if noise:
        res.update(raw_noise_std=0.5, noise_coarse=torch.randn(R, N, generator=g), noise_fine=torch.randn(R, N + Ni, generator=g))
    assert K > 0 and int((res["sb_fine"] >= 0).sum()) > 0
    return res


def _plain(nets, b):
    """The plain float64 chain through the oracle's own modules: (total, grads per distinct network, d_raw)."""
    rays = b["rays"]
    raws, maps = {}, {}
    for role, net in zip(("coarse", "fine"), nets):
        pts, vd = OPN.form_points(rays, b[f"z_{role}"])
        R, N = b[f"z_{role}"].shape
        raws[role] = net(pts.double(), vd.double()).reshape(R, N, -1)
        maps[role] = O.raw2outputs(raws[role], b[f"z_{role}"].double(), rays[:, 3:].double(),
                                   raw_noise_std=float(b.get("raw_noise_std", 0.0)), noise=b.get(f"noise_{role}"),
                                   num_classes=net.C, num_instances=net.K, sample_box=b[f"sb_{role}"],
                                   box_sem=b["box_sem"], box_inst=b["box_inst"], mask_outside=bool(b["mask_outside"]))
    m1, m0, w = maps["fine"], maps["coarse"], b["weights"]
    total, _ = OL.losses(m1["rgb_map"], m0["rgb_map"], m1["depth_map"], m1["semantic_map"], m1["fixed_semantic_map"],
                         b["rgb"], b["depth"], b["pseudo_label"], b["pseudo_weight"].double(), w[:4])
    inst, _, _, _ = OI.instance_loss(m1["instance_map"], m1["fixed_instance_map"], b["inst_min_weight"])
    total = total + w[4] * inst
    uniq = [nets[0]] + ([nets[1]] if nets[1] is not nets[0] else [])
    params = [p for n in uniq for p in n.parameters()]
    g = torch.autograd.grad(total, params + [raws["coarse"], raws["fine"]])
    grads, k = [], 0
    for n in uniq:
        names = [name for name, _ in n.named_parameters()]
        grads.append(dict(zip(names, g[k:k + len(names)])))
        k += len(names)
    return total.detach(), grads, {"coarse": g[-2], "fine": g[-1]}


@pytest.mark.parametrize("shared,noise", [(False, False), (True, True)])
def test_no_op_pinning_is_the_plain_oracle_bit_for_bit(shared, noise):
    cfg = make_cfg("cfg1", D=4, W=64, num_classes=5, num_instances=6, N_samples=16, N_importance=16,
                   bound_by_primitives=True, perturb=1.0)
    nets = _nets(cfg, shared, torch.float64)
    b = _batch(cfg, 96, seed=3, nets32=_nets(cfg, shared, torch.float32), mask_outside=noise, noise=noise)
    total, grads, d_raw = _plain(nets, b)
    got = OPN.iteration(nets, b)
    assert got["flips"] == {} and torch.equal(got["total"], total)
    for mine, ref in zip(got["grads"], grads):
        assert set(mine) == set(ref)
        for name in ref:
            assert torch.equal(mine[name], ref[name]), name
    for role in ("coarse", "fine"):
        assert torch.equal(got["d_raw"][role], d_raw[role]), role
    # the chain's own decisions fed back as pins give the same bits again, with no flip
    again = OPN.iteration(nets, b, pins=got["own"])
    assert again["flips"] == {"coarse": 0, "fine": 0, "loss": 0} and torch.equal(again["total"], total)
    for mine, ref in zip(again["grads"], grads):
        for name in ref:
            assert torch.equal(mine[name], ref[name]), name


def test_points_and_view_directions_are_numpy_float32_mul_then_add():
    g = torch.Generator().manual_seed(0)
    R, N = 300, 70
    rays = torch.cat([torch.randn(R, 3, generator=g) * 30, torch.randn(R, 3, generator=g) * 2], -1)
    z = torch.rand(R, N, generator=g) * 80
    pts, vd = OPN.form_points(rays, z)
    r, zz = rays.numpy(), z.numpy()
    want = (r[:, None, :3] + np.multiply(r[:, None, 3:], zz[..., None], dtype=np.float32)).reshape(-1, 3)
    assert want.dtype == np.float32 and np.array_equal(pts.numpy(), want)
    d = r[:, 3:]
    n2 = d[:, 0] * d[:, 0]
    n2 = n2 + d[:, 1] * d[:, 1]
    n2 = n2 + d[:, 2] * d[:, 2]
    want_vd = np.repeat((d / np.sqrt(n2)[:, None])[:, None, :], N, 1).reshape(-1, 3)
    assert want_vd.dtype == np.float32 and np.array_equal(vd.numpy(), want_vd)


@pytest.fixture(scope="module")
def standin():
    """Case 1's shape (cfg3 networks, 160 rays of 64 + 128 samples, primitives, fixed maps, five terms) with a
    shared network and mask_outside, so that every deliberate change of the power test applies: the fp32 chain as the
    device, and the float64 chain pinned to its decisions."""
    cfg = make_cfg("cfg3", bound_by_primitives=True, perturb=1.0)
    n32, n64 = _nets(cfg, True, torch.float32), _nets(cfg, True, torch.float64)
    b = _batch(cfg, 160, seed=7, nets32=n32, mask_outside=True)
    dev = OPN.iteration(n32, b)
    ref = OPN.iteration(n64, b, pins=dev["own"])
    return cfg, n64, b, dev, ref


def _rejections(dev, ref):
    return {k: v for k, v in OPN.param_ratios(dev["grads"][0], ref["grads"][0], TOL, floor_only=True).items() if v > 1.0}


def test_the_fp32_stand_in_meets_every_check_once_pinned(standin):
    cfg, _, b, dev, ref = standin
    C, K = int(cfg.num_classes), int(cfg.num_instances)
    print(f"pinned flips: {ref['flips']}")
    assert ref["flips"]["coarse"] + ref["flips"]["fine"] >= 1, "the fp32 run took every ReLU branch float64 took"
    for role in ("coarse", "fine"):
        worst = OPN.maps_ratio(dev["maps"][role], ref["maps"][role], ref["raw"][role], b[f"z_{role}"], C, K)
        print(f"{role} maps: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
        assert max(worst.values()) <= 1.0, worst
        e = OPN.d_raw_ratio(dev["d_raw"][role], ref, role, C, K)
        print(f"{role} d_raw: largest error / bound = {e:.3e}")
        assert e <= 1.0
    assert float((dev["total"].double() - ref["total"]).abs()) <= 1e-4 * float(ref["total"].abs())
    assert bool(((dev["terms"].double() - ref["terms"]).abs() <= 1e-4 * ref["terms"].abs()).all())
    ratios = OPN.param_ratios(dev["grads"][0], ref["grads"][0], TOL, floor_only=True)
    print("largest error / bound: " + ", ".join(f"{k} {v:.2e}" for k, v in ratios.items()))
    assert max(ratios.values()) <= 1.0


def test_the_margin_guard_refuses_a_flip_far_from_zero(standin):
    cfg, n64, b, dev, _ = standin
    pins = {k: (dict(v) if isinstance(v, dict) else v) for k, v in dev["own"].items()}
    name = "pts_linears.3"
    m = pins["fine"][name].clone()
    pre_far = m.nonzero()[0]                       # a unit the fp32 run kept on; flip it off
    m[pre_far[0], pre_far[1]] = False
    pins["fine"][name] = m
    with pytest.raises(OPN.PinError, match="beyond the margin"):
        OPN.iteration(n64, b, pins=pins)
    sign = pins["depth_sign"].clone()
    ok = b["depth"] > 0
    i = int(ok.nonzero()[0])
    sign[i] = -sign[i]
    pins = dict(dev["own"], depth_sign=sign)
    with pytest.raises(OPN.PinError, match="depth sign"):
        OPN.iteration(n64, b, pins=pins)


@pytest.mark.parametrize("edit", OPN.EDITS)
def test_each_deliberate_change_of_the_reference_is_rejected(standin, edit):
    cfg, n64, b, dev, _ = standin
    bad = OPN.iteration(n64, b, pins=dev["own"], edit=edit)
    rejected = _rejections(dev, bad)
    old = OPN.old_criterion_accepts(dev["grads"][0], bad["grads"][0])
    print(f"{edit}: rejected on {len(rejected)} tensors (largest {max(rejected.values(), default=0):.1f} x the bound); "
          f"cosine >= 0.999 and norm within 1 % would have {'accepted' if old else 'rejected'} it")
    assert rejected, f"{edit}: the element-wise check accepted a changed reference"
    affected = {"w_inst": "instance_linears.1.weight", "head_rows": "instance_linears.1.weight",
                "drop_coarse_rgb": "rgb_linear.weight", "mask_forward_only": "alpha_linear.weight"}[edit]
    assert affected in rejected, (edit, sorted(rejected))
