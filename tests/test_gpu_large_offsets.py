"""The render and training kernels on buffers whose element offsets pass 2^31 (and 2^32 where the entry point allows
it), through the C ABI.  Every other test of these kernels runs at a few thousand rows, where a 32-bit product in a
row offset cannot show.

Method, the same for every kernel:
  1. One large launch, sized so that one buffer's element offsets cross 2^31, with the cheapest shape (wide channels
     or many levels rather than many rays).  Each case prints the largest element offset of that buffer.
  2. Whole output, bit for bit: the large launch's outputs against small launches over row ranges of the same inputs
     (pointer offsets into the same buffers, each small buffer under 2^31 elements).  The other limits tests pin the
     small launches to their oracles, so this compares every row with little extra memory.
  3. Boundary rows against float64 (or the bit-exact oracle), with the tolerance model of the kernel's limits test:
     the rows whose element range holds 2^31 - 1, 2^31, 2^32 - 1 or 2^32, the first and last rows and random rows.
     This catches a large launch and small launches that are wrong in the same way.
  4. Reductions over rows (n_inst of pnr_losses, stash_absmax, pnr_wgrad's split-K sums) depend on the launch, so
     they are compared with float64 (or exact integer) sums over all rows, computed on the device.
  5. Every output buffer is filled with the byte 0xA5 and has a poisoned tail of at least one row, which must stay
     unchanged.
Inputs are built on the device with cheap structure: a small random block repeated with a period prime to every chunk
size, plus per-row values (ids, directions, depth offsets) so that no two rows of a launch repeat each other.
A case that does not fit in the free device memory skips, naming the GiB it needs and the GiB free; none needs more
than 31.3 GiB (the 128-row kernel's case, counting 2 GiB kept free).
The float64 check of step 3 takes 1000 random rows in every case but the rays-mode MLP, which takes 40 random rays
of 192 samples each."""
import ctypes as C
import gc

import pytest
import torch

from oracle import reference_panoptic as OP
from oracle import reference_renderer as O
from oracle_bound import VIEWDIR_REL, forward_bound, view_encoding
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as SY
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from panopticnerf_b200.lib.train.mlp_backward import _pow2_scale
from test_cpu_operand_split import default_grad_scale, ratio, trunk_input
from test_gpu_backward_bound import check_within, pinned_bound
from test_gpu_render_limits import _per_ray_ratio
from test_gpu_stage_limits import _abs_sums, _composite_case, _ratio, _report
from test_gpu_train_limits import _check_linear, _check_wgrad, _linear, _ref_wgrad, _wgrad

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32, F64, I32 = torch.float32, torch.float64, torch.int32
B31, B32 = 1 << 31, 1 << 32
GIB = float(1 << 30)
MARGIN = 2 << 30                  # device memory kept free beyond a case's own buffers
SMALL = 1 << 28                   # elements of the widest buffer of one small launch (1 GiB of fp32)
POISON = 0xA5
_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Each case starts and ends with the caching allocator emptied: the next one measures what is really free."""
    gc.collect()
    torch.cuda.empty_cache()
    yield
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _need(nbytes, what):
    free = torch.cuda.mem_get_info(DEV)[0]
    if free < nbytes + MARGIN:
        pytest.skip(f"{what} needs {(nbytes + MARGIN) / GIB:.1f} GiB of device memory; {free / GIB:.1f} GiB free")


def _small(n_wide=1):
    """Bytes one small launch adds: n_wide fp32 outputs of its widest row size (SMALL elements each) and the bool mask
    of their comparison (_same_bits compares contiguous row ranges in place)."""
    return n_wide * SMALL * 4 + SMALL


def _crossing(what, elems):
    """Report the largest element offset of the buffer that crosses 2^31."""
    top = elems - 1
    print(f"{what}: largest element offset {top} = 2^31 + {top - B31}" + (" (past 2^32)" if top >= B32 else ""))
    assert top >= B31, f"{what}: the buffer does not cross 2^31"


def _poisoned(shape, dtype=F32, tail=1):
    """(rows view, whole buffer): a buffer of shape[0] + tail rows, every byte POISON."""
    buf = torch.empty((shape[0] + tail,) + tuple(shape[1:]), dtype=dtype, device=DEV)
    buf.view(-1).view(torch.uint8).fill_(POISON)
    return buf[:shape[0]], buf


def _tail_intact(buf, rows, what):
    assert bool((buf[rows:].reshape(-1).view(torch.uint8) == POISON).all()), f"{what}: written past its last row"


def _same_bits(a, b, what, r0=0):
    assert a.shape == b.shape, f"{what}: {tuple(a.shape)} vs {tuple(b.shape)}"
    x, y = a.contiguous(), b.contiguous()
    if x.dtype != torch.bool:
        x, y = x.view(_INT[x.element_size()]), y.view(_INT[y.element_size()])
    diff = x != y
    if bool(diff.any()):
        rows = diff.reshape(diff.shape[0], -1).any(1).nonzero()[:, 0]
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ, in {rows.numel()} rows, the first row "
                             f"{r0 + int(rows[0])}")


def _check_chunks(what, R, row_elems, run, full):
    """Step 2: run(r0, r1) launches over rows [r0, r1) of the same inputs and returns {name: its output rows}; each
    must equal full[name][r0:r1] bit for bit.  Rows per small launch: SMALL // row_elems (row_elems: elements per row
    of the widest buffer)."""
    step = max(1, SMALL // row_elems)
    n = 0
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        got = run(r0, r1)
        for k, v in got.items():
            _same_bits(v, full[k][r0:r1], f"{what} {k} rows [{r0}, {r1})", r0)
        n += 1
    print(f"{what}: {n} small launches of up to {step} rows equal the large launch bit for bit")


def _rows(R, row_elems, n_random=1000, seed=0):
    """Step 3's rows (sorted, CPU int64): the first and last rows, those whose elements [r row_elems, (r+1) row_elems)
    hold 2^31 - 1, 2^31, 2^32 - 1 or 2^32, and n_random random rows."""
    s = {0, R - 1}
    s.update(b // row_elems for b in (B31 - 1, B31, B32 - 1, B32) if b < R * row_elems)
    g = torch.Generator().manual_seed(seed)
    s.update(torch.randint(0, R, (n_random,), generator=g).tolist())
    return torch.tensor(sorted(s), dtype=torch.int64)


def _tile(block, R):
    """[R, ...] on the device: row r = block[r % len(block)]."""
    b = block.to(DEV)
    P_ = b.shape[0]
    out = torch.empty((R,) + tuple(b.shape[1:]), dtype=b.dtype, device=DEV)
    q = R // P_
    out[:q * P_].view((q,) + tuple(b.shape)).copy_(b[None].expand((q,) + tuple(b.shape)))
    out[q * P_:] = b[:R - q * P_]
    return out


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# ------------------------------------------------------------------------------------------------ compositing
COMP_MAPS = {"rgb_map": 3, "depth_map": 0, "acc_map": 0, "disp_map": 0, "weights": "N", "semantic_map": "C",
             "instance_map": "K", "fixed_semantic_map": "C", "fixed_instance_map": "K"}


def _map_shape(k, R, N, Cn, Kn):
    w = COMP_MAPS[k]
    w = {"N": N, "C": Cn, "K": Kn}.get(w, w)
    return (R, w) if w else (R,)


def _composite_call(raw, z, rays, sb, bs, bi, Cn, Kn, out):
    R, N = z.shape
    co = _capi.ptr_struct(_capi.PnrCompositeOut, out)
    _capi.check(_capi.lib().pnr_composite(raw.data_ptr(), z.data_ptr(), rays.data_ptr(), R, N, Cn, Kn, 0, 0, 0,
                                          sb.data_ptr(), bs.data_ptr(), bi.data_ptr(), bs.shape[0], C.byref(co),
                                          _capi.stream_ptr()), "pnr_composite")


def _composite_backward_call(raw, z, rays, sb, bs, bi, Cn, Kn, grads, d_raw):
    R, N = z.shape
    cg = _capi.ptr_struct(_capi.PnrCompositeGrads, grads)
    _capi.check(_capi.lib().pnr_composite_backward(raw.data_ptr(), z.data_ptr(), rays.data_ptr(), R, N, Cn, Kn, 0, 0, 0,
                                                   sb.data_ptr(), bs.data_ptr(), bi.data_ptr(), bs.shape[0],
                                                   C.byref(cg), d_raw.data_ptr(), _capi.stream_ptr()),
                "pnr_composite_backward")


def test_composite_forward_and_backward_past_2_31():
    """pnr_composite and pnr_composite_backward at C = K = 128 (260 channels), N = 256, R = 33 000 rays: raw and d_raw
    hold 2.2e9 elements.  raw repeats a block of 252 rays of test_gpu_stage_limits' four regimes (logits of 1e4,
    surface-like and empty rays, duplicated depths, ids outside the tables); every ray has its own direction length
    and its own sample ids, so every ray's outputs differ.  Boundary rays against float64 as
    test_composite_per_ray_against_float64 and test_composite_backward_per_ray_against_float64 hold them."""
    R, N, Cn, Kn = 33000, 256, 128, 128
    CH = 4 + Cn + Kn
    row = N * CH
    _need(2 * R * row * 4 + _small(), "pnr_composite at 2.2e9 raw elements")
    raw_b, z_b, d_b, sb_b, bs, bi = _composite_case(252, N, Cn, Kn, seed=31, big_on_surface=False)
    raw = _tile(raw_b, R)
    z = _tile(z_b, R)
    r = torch.arange(R, device=DEV)
    d = _tile(d_b, R) * (1.0 + (r % 1021).float() * 2.0 ** -10)[:, None]
    rays = torch.cat([torch.zeros(R, 3, device=DEV), d], 1).contiguous()
    g = _gen(32)
    sb = torch.randint(-3, 23, (R, N), generator=g, device=DEV, dtype=I32)
    bs, bi = bs.to(DEV), bi.to(DEV)
    _crossing("pnr_composite raw", R * row)
    # forward
    full, bufs = {}, {}
    for k in COMP_MAPS:
        full[k], bufs[k] = _poisoned(_map_shape(k, R, N, Cn, Kn))
    _composite_call(raw, z, rays, sb, bs, bi, Cn, Kn, full)
    for k in COMP_MAPS:
        _tail_intact(bufs[k], R, f"pnr_composite {k}")

    def fwd(r0, r1):
        out = {k: torch.empty(_map_shape(k, r1 - r0, N, Cn, Kn), device=DEV) for k in COMP_MAPS}
        _composite_call(raw[r0:r1], z[r0:r1], rays[r0:r1], sb[r0:r1], bs, bi, Cn, Kn, out)
        return out
    _check_chunks("pnr_composite", R, row, fwd, full)
    idx = _rows(R, row)
    n = idx.numel()
    r64, z64, d64, sbs = raw[idx.to(DEV)].cpu().double(), z[idx.to(DEV)].cpu().double(), d[idx.to(DEV)].cpu().double(), sb[idx.to(DEV)].cpu()
    kw = dict(num_classes=Cn, num_instances=Kn, sample_box=sbs, box_sem=bs.cpu(), box_inst=bi.cpu())
    ref = O.raw2outputs(r64, z64, d64, **kw)
    w64 = ref["weights"]
    S = _abs_sums(r64, z64, w64, Cn, Kn, sbs, bs.cpu(), bi.cpu(), False)
    w_max = w64.max(1).values
    worst = 0.0
    for k, s in S.items():
        per_ray = s.reshape(n, -1).max(1).values
        if k.startswith("fixed_"):
            per_ray = torch.maximum(per_ray, w_max)
        err = (full[k][idx.to(DEV)].cpu().double() - ref[k]).abs().reshape(n, -1)
        worst = max(worst, _ratio(err, 1e-4 * per_ray[:, None] + 2.0 ** -24 * ref[k].abs().reshape(n, -1)))
    worst = max(worst, _ratio((full["weights"][idx.to(DEV)].cpu().double() - w64).abs(), 1e-4 * w_max[:, None].expand(n, N)))
    dg, dr = full["disp_map"][idx.to(DEV)].cpu().double(), ref["disp_map"]
    assert torch.equal(torch.isnan(dg), torch.isnan(dr))
    ok = ~torch.isnan(dr)
    worst = max(worst, _ratio((dg - dr)[ok].abs(), 2e-4 * dr[ok].abs()))
    _report(f"pnr_composite R={R} boundary rays ({n})", worst)
    del full, bufs, ref, S
    # backward: upstream gradients on every map
    grads = {k: torch.randn(_map_shape(k, R, N, Cn, Kn), generator=g, device=DEV) for k in COMP_MAPS if k != "disp_map"}
    d_raw, dbuf = _poisoned((R, N, CH))
    _composite_backward_call(raw, z, rays, sb, bs, bi, Cn, Kn, grads, d_raw)
    _tail_intact(dbuf, R, "pnr_composite_backward d_raw")
    _crossing("pnr_composite_backward d_raw", R * row)

    def bwd(r0, r1):
        out = torch.empty(r1 - r0, N, CH, device=DEV)
        _composite_backward_call(raw[r0:r1], z[r0:r1], rays[r0:r1], sb[r0:r1], bs, bi, Cn, Kn,
                                 {k: v[r0:r1] for k, v in grads.items()}, out)
        return {"d_raw": out}
    _check_chunks("pnr_composite_backward", R, row, bwd, {"d_raw": d_raw})
    ref = O.raw2outputs_backward(r64, z64, d64, {k: v[idx.to(DEV)].cpu().double() for k, v in grads.items()}, **kw)
    got = d_raw[idx.to(DEV)].cpu().double()
    assert torch.isfinite(ref).all() and torch.isfinite(got).all()
    worst = 0.0
    for name, sl in (("rgb", slice(0, 3)), ("sigma", slice(3, 4)), ("sem", slice(4, 4 + Cn)), ("inst", slice(4 + Cn, CH))):
        rr, a = ref[..., sl], got[..., sl]
        floor = 1e-6 * float(rr.pow(2).mean().sqrt())
        per_ray = rr.abs().reshape(n, -1).max(1).values.clamp(min=floor)
        worst = max(worst, _ratio((a - rr).abs().reshape(n, -1), 1e-4 * per_ray[:, None].expand(n, a[0].numel())))
    _report(f"pnr_composite_backward R={R} boundary rays ({n})", worst)


# ------------------------------------------------------------------------------------------------ losses
def _loss_call(R, Cn, Kn, t, out, r0=0, r1=None, w=(1.0, 0.1, 0.5, 2.0), w_inst=0.7):
    """pnr_losses over rows [r0, r1) of the inputs t (pointer offsets), into out (already those rows)."""
    r1 = R if r1 is None else r1
    sl = lambda k: None if t.get(k) is None else _capi.ptr(t[k][r0:r1])
    o = lambda k: None if out.get(k) is None else _capi.ptr(out[k])
    a = _capi.PnrLossArgs()
    a.R, a.C, a.sem_is_prob, a.K = r1 - r0, Cn, int(t["prob"]), Kn
    a.rgb_map, a.rgb_map0, a.rgb_gt = sl("rgb"), sl("rgb0"), sl("rgb_gt")
    a.depth_map, a.depth_gt = sl("depth"), sl("depth_gt")
    a.semantic_map, a.fixed_semantic_map, a.label, a.label_weight = sl("sem"), sl("fix"), sl("label"), sl("conf")
    a.w_rgb, a.w_depth, a.w_sem, a.w_fix = w
    a.inv_n_rgb, a.inv_n_depth, a.inv_n_sem, a.eps = t["inv_n"] + (EPS,)
    a.per_ray, a.d_rgb_map, a.d_rgb_map0, a.d_depth_map = o("per_ray"), o("d_rgb"), o("d_rgb0"), o("d_depth")
    a.d_semantic_map, a.d_fixed_semantic_map = o("d_sem"), o("d_fix")
    if Kn:
        a.instance_map = a.fixed_instance_map = sl("inst")          # the logits are also the primitive weights
        a.w_inst, a.inst_min_weight = w_inst, 0.5
        a.per_ray_inst, a.inst_label, a.n_inst, a.d_instance_map = o("per_ray_inst"), o("inst_label"), o("n_inst"), o("d_inst")
    _capi.check(_capi.lib().pnr_losses(C.byref(a), _capi.stream_ptr()), "pnr_losses")


EPS = 2.0 ** -20                   # exact in fp32: p == eps on both sides


@pytest.mark.parametrize("term", ["semantic", "probability", "instance"])
def test_losses_past_2_31(term):
    """pnr_losses at R = 65 600 rays with 32767 channels: each [R, C] map and gradient holds 2.15e9 elements.  Every
    case has the photometric term of both colour maps (rgb_map and rgb_map0) and the depth term.
    - semantic: softmax cross-entropy of C = 32767 logits, repeating a block of 61 rows with logits up to +-1e4 on
      40% of them.
    - probability: sem_is_prob = 1 with the same [R, C] probabilities as semantic_map and fixed_semantic_map, so both
      -log(max(p, eps)) terms read it and write d_semantic_map and d_fixed_semantic_map; the labelled probability is
      exactly 0, eps or 2 eps on three rays of seven.
    - instance: K = 32767 instance logits (one block row all negative, so not counted).  Its gradient is normalised
      by the launch's count of counted rays, so small launches scale it differently: it is held to float64 alone
      (step 3), and the count itself must equal the count over all rows, exactly.
    Labels, confidences, colours and depths are per ray."""
    R, W_ = 65600, 32767
    wide = {"semantic": (2, 1), "probability": (3, 2), "instance": (2, 0)}[term]    # [R, C] buffers: whole, per launch
    _need(wide[0] * R * W_ * 4 + _small(wide[1]), f"pnr_losses {term} at 2.15e9 elements")
    g = torch.Generator().manual_seed(41)
    if term == "probability":
        blk = torch.rand(61, W_, generator=g)
        blk /= blk.sum(1, keepdim=True)
    else:
        blk = torch.randn(61, W_, generator=g) * 3
        big = torch.rand(61, generator=g) < 0.4
        blk[big] = torch.sign(blk[big]) * 1e4 * torch.rand(int(big.sum()), W_, generator=g)
    if term == "instance":
        blk[5] = -blk[5].abs() - 1.0                                   # row maximum < inst_min_weight: not counted
    x = _tile(blk, R)
    gd = _gen(42)
    t = dict(rgb=torch.rand(R, 3, generator=gd, device=DEV), rgb0=torch.rand(R, 3, generator=gd, device=DEV),
             rgb_gt=torch.rand(R, 3, generator=gd, device=DEV), depth=torch.rand(R, generator=gd, device=DEV) * 50 + 1,
             prob=term == "probability")
    t["depth_gt"] = torch.where(torch.rand(R, generator=gd, device=DEV) > 0.3, t["depth"] + 1, torch.zeros(R, device=DEV))
    lab = (torch.arange(R, device=DEV) * 5) % (W_ + 2) - 1                       # -1 and C: ignored
    has_d = (lab >= 0) & (lab < W_)
    n_depth = int((t["depth_gt"] > 0).sum())
    if term == "instance":
        Cn, Kn, n_sem = 0, W_, 1
        t["inst"] = x
    else:
        Cn, Kn = W_, 0
        t.update(sem=x, label=lab.to(I32), conf=torch.rand(R, generator=gd, device=DEV))
        n_sem = int(has_d.sum())
        if t["prob"]:
            t["fix"] = x
            for m, p in enumerate((0.0, EPS, 2 * EPS)):             # the labelled probability at 0, eps and 2 eps
                rows = torch.arange(m, R, 7, device=DEV)
                rows = rows[has_d[rows]]
                x[rows, lab[rows]] = p
    t["inv_n"] = (1.0 / (3 * R), 1.0 / n_depth, 1.0 / n_sem)
    _crossing(f"pnr_losses {term} map and gradient", R * W_)
    out, bufs = {}, {}
    shapes = dict(per_ray=((R, 4), F32), d_rgb=((R, 3), F32), d_rgb0=((R, 3), F32), d_depth=((R,), F32))
    if Kn:
        shapes.update(d_inst=((R, Kn), F32), per_ray_inst=((R,), F32), inst_label=((R,), I32), n_inst=((1,), I32))
    else:
        shapes.update(d_sem=((R, Cn), F32))
        if t["prob"]:
            shapes.update(d_fix=((R, Cn), F32))
    for k, (s, dt) in shapes.items():
        out[k], bufs[k] = _poisoned(s, dt)
    _loss_call(R, Cn, Kn, t, out)
    for k, (s, _) in shapes.items():
        _tail_intact(bufs[k], s[0], f"pnr_losses {k}")
    per_launch = ("d_inst", "n_inst")

    def run(r0, r1):
        o = {k: torch.empty((r1 - r0,) + s[1:], dtype=dt, device=DEV) for k, (s, dt) in shapes.items() if k not in per_launch}
        if Kn:
            o["n_inst"] = torch.empty(1, dtype=I32, device=DEV)
        _loss_call(R, Cn, Kn, t, o, r0, r1)
        o.pop("n_inst", None)
        return o
    _check_chunks(f"pnr_losses {term}", R, W_, run, {k: v for k, v in out.items() if k not in per_launch})
    idx = _rows(R, W_, seed=43)
    n = idx.numel()
    ix = idx.to(DEV)
    s64 = x[ix].cpu().double()
    rgb, rgb0, gt = t["rgb"][ix].cpu().double(), t["rgb0"][ix].cpu().double(), t["rgb_gt"][ix].cpu().double()
    dep, dgt = t["depth"][ix].cpu().double(), t["depth_gt"][ix].cpu().double()
    w_rgb, w_depth, w_sem, w_fix, w_inst = 1.0, 0.1, 0.5, 2.0, 0.7
    z64 = torch.zeros(n, dtype=F64)
    ref_pr = torch.stack([((rgb - gt) ** 2).sum(1) + ((rgb0 - gt) ** 2).sum(1),
                          torch.where(dgt > 0, (dep - dgt).abs(), z64), z64, z64], 1)
    slack = torch.zeros(n, 4, dtype=F64)
    slack[:, 1] = 2.0 ** -23 * torch.maximum(dep.abs(), dgt.abs())
    grads = {"d_rgb": 2 * (rgb - gt) * w_rgb / (3 * R), "d_rgb0": 2 * (rgb0 - gt) * w_rgb / (3 * R),
             "d_depth": torch.where(dgt > 0, torch.sign(dep - dgt), z64) * w_depth / n_depth}
    if term != "instance":
        label, conf = lab[ix].cpu(), t["conf"][ix].cpu().double()
        has = (label >= 0) & (label < Cn)
        k = label.clamp(0, Cn - 1)
        onehot = torch.nn.functional.one_hot(k, Cn).double()
        p = s64.gather(1, k[:, None])[:, 0]
        if t["prob"]:
            # -log(max(p, eps)) of both maps (the same probabilities); the gradient passes at p == eps, not below
            l = torch.where(has, -torch.log(p.clamp_min(EPS)) * conf, z64)
            ref_pr[:, 2], ref_pr[:, 3] = l, l
            live = has & (p >= EPS)
            for name, wt in (("d_sem", w_sem), ("d_fix", w_fix)):
                grads[name] = torch.where(live[:, None], -onehot * (conf * wt / n_sem / p.clamp_min(EPS))[:, None],
                                          torch.zeros_like(s64))
            # over all rays: p == eps passes a gradient, p == 0 passes none
            for m, live_at in ((0, False), (1, True)):
                rows = torch.arange(m, R, 7, device=DEV)
                rows = rows[has_d[rows] & (t["conf"][rows] > 0)]
                for name in ("d_sem", "d_fix"):
                    gl = out[name][rows, lab[rows]]
                    assert bool((gl != 0).all()) if live_at else bool((gl == 0).all()), (name, m)
        else:
            lse = torch.logsumexp(s64, 1)
            ref_pr[:, 2] = torch.where(has, (lse - p) * conf, z64)
            slack[:, 2] = torch.where(has, 2.0 ** -23 * s64.abs().max(1).values * conf, z64)
            grads["d_sem"] = torch.where(has[:, None], (torch.softmax(s64, 1) - onehot) * (conf * w_sem / n_sem)[:, None],
                                         torch.zeros_like(s64))
    else:
        n_all = int((x.amax(1) >= 0.5).sum())                          # every row: no NaN in these logits
        assert int(out["n_inst"][0]) == n_all, (int(out["n_inst"][0]), n_all)
        print(f"pnr_losses instance: n_inst = {n_all} of {R} rays, exactly")
        lse = torch.logsumexp(s64, 1)
        k = OP._argmax_first(s64.float())
        cnt = s64.max(1).values >= 0.5
        assert torch.equal(out["inst_label"][ix].cpu().long(), torch.where(cnt, k, torch.full_like(k, -1)))
        li = torch.where(cnt, lse - s64.gather(1, k[:, None])[:, 0], z64)
        r = _ratio((out["per_ray_inst"][ix].cpu().double() - li).abs(),
                   1e-4 * li.abs() + torch.where(cnt, 2.0 ** -23 * s64.abs().max(1).values, z64))
        _report("pnr_losses per_ray_inst boundary rays", r)
        onehot = torch.nn.functional.one_hot(k, Kn).double()
        grads["d_inst"] = torch.where(cnt[:, None], (torch.softmax(s64, 1) - onehot) * (w_inst / n_all),
                                      torch.zeros_like(s64))
    worst = _ratio((out["per_ray"][ix].cpu().double() - ref_pr).abs(), 1e-4 * ref_pr.abs() + slack)
    for name, rr in grads.items():
        rr = rr.reshape(n, -1)
        a = out[name][ix].cpu().double().reshape(n, -1)
        floor = 1e-6 * float(rr.pow(2).mean().sqrt())
        per = rr.abs().max(1).values.clamp(min=floor)
        worst = max(worst, _ratio((a - rr).abs(), 1e-4 * per[:, None].expand_as(rr)))
    _report(f"pnr_losses {term} R={R} boundary rays ({n})", worst)


# ------------------------------------------------------------------------------------------------ labels and fusion
def _labels_call(t, R, Cn, Kn, out):
    _capi.check(_capi.lib().pnr_label_tiles(_capi.ptr(t["rgb"]), _capi.ptr(t["depth"]), _capi.ptr(t["sem"]),
                                            _capi.ptr(t["inst"]), R, Cn, Kn, _capi.ptr(out["rgb8"]),
                                            _capi.ptr(out["depth_out"]), _capi.ptr(out["sem_label"]),
                                            _capi.ptr(out["inst_label"]), _capi.stream_ptr()), "pnr_label_tiles")


def _fuse_call(t, R, Cn, Kn, tab, out):
    _capi.check(_capi.lib().pnr_panoptic_fuse(_capi.ptr(t["sem"]), _capi.ptr(t["inst"]), R, Cn, Kn,
                                              *(_capi.ptr(tab[k]) for k in ("is_thing", "inst_class", "inst_id",
                                                                            "class_id", "palette")),
                                              _capi.ptr(out["panoptic"]), _capi.ptr(out["f_sem"]),
                                              _capi.ptr(out["f_slot"]), _capi.ptr(out["color"]), _capi.stream_ptr()),
                "pnr_panoptic_fuse")


def test_label_tiles_and_panoptic_fuse_past_2_31():
    """pnr_label_tiles and pnr_panoptic_fuse at C = K = 32767, R = 65 600: both maps hold 2.15e9 elements.  The maps
    repeat a block of 61 rows with ties (rounded rows), NaN rows and a maximum in the last channel; two rays of three
    also carry a per-ray maximum at channel 5r mod C, so their labels follow the ray.  Boundary rays against the
    bit-exact oracle."""
    R, Cn, Kn = 65600, 32767, 32767
    _need(2 * R * Cn * 4, "pnr_label_tiles at 2.15e9 elements")
    g = torch.Generator().manual_seed(51)
    sb, ib = torch.randn(61, Cn, generator=g), torch.randn(61, Kn, generator=g)
    sb[::5] = sb[::5].round(decimals=0)
    ib[::3] = ib[::3].round(decimals=0)
    sb[3, Cn - 1] = sb[3].max() + 1
    sb[4, :] = float("nan")
    sb[6, : Cn // 2] = float("nan")
    ib[7, Kn - 1] = float("nan")
    sem, inst = _tile(sb, R), _tile(ib, R)
    r = torch.arange(R, device=DEV)
    bump = r[r % 3 != 0]
    sem[bump, (bump * 5) % Cn] = 8.0 + (bump % 7).float()
    inst[bump, (bump * 5) % Kn] = 8.0 + (bump % 11).float()
    gd = _gen(52)
    t = dict(sem=sem, inst=inst, rgb=torch.rand(R, 3, generator=gd, device=DEV) * 1.2 - 0.1,
             depth=torch.rand(R, generator=gd, device=DEV) * 50)
    inst_class = (torch.arange(Kn) * 5) % Cn                           # slot k of class 5k: ray k's class has ray k's slot
    is_thing = (torch.rand(Cn, generator=g) > 0.3).to(torch.uint8)
    tab = dict(is_thing=is_thing, inst_class=inst_class.to(I32), inst_id=(inst_class * 1000 + torch.arange(Kn) + 1).to(I32),
               class_id=(torch.randperm(Cn, generator=g) + 3).to(I32),
               palette=torch.randint(0, 256, (Cn, 3), generator=g, dtype=torch.uint8))
    tab_d = {k: v.to(DEV) for k, v in tab.items()}
    _crossing("pnr_label_tiles / pnr_panoptic_fuse maps", R * Cn)
    shapes = dict(rgb8=((R, 3), torch.uint8), depth_out=((R,), F32), sem_label=((R,), torch.int16),
                  inst_label=((R,), torch.int16), panoptic=((R,), I32), f_sem=((R,), torch.int16),
                  f_slot=((R,), torch.int16), color=((R, 3), torch.uint8))
    out, bufs = {}, {}
    for k, (s, dt) in shapes.items():
        out[k], bufs[k] = _poisoned(s, dt)
    _labels_call(t, R, Cn, Kn, out)
    _fuse_call(t, R, Cn, Kn, tab_d, out)
    for k, (s, _) in shapes.items():
        _tail_intact(bufs[k], R, f"labels {k}")

    def run(r0, r1):
        o = {k: torch.empty((r1 - r0,) + s[1:], dtype=dt, device=DEV) for k, (s, dt) in shapes.items()}
        tt = {k: v[r0:r1] for k, v in t.items()}
        _labels_call(tt, r1 - r0, Cn, Kn, o)
        _fuse_call(tt, r1 - r0, Cn, Kn, tab_d, o)
        return o
    _check_chunks("pnr_label_tiles + pnr_panoptic_fuse", R, Cn, run, out)
    idx = _rows(R, Cn, seed=53)
    ix = idx.to(DEV)
    s_c, i_c = sem[ix].cpu(), inst[ix].cpu()
    assert torch.equal(out["sem_label"][ix].cpu(), OP._argmax_first(s_c).to(torch.int16))
    assert torch.equal(out["inst_label"][ix].cpu(), OP._argmax_first(i_c).to(torch.int16))
    rgb = t["rgb"][ix].cpu()
    assert torch.equal(out["rgb8"][ix].cpu().float(), torch.round(rgb.clamp(0, 1) * 255))
    assert torch.equal(out["depth_out"][ix].cpu(), t["depth"][ix].cpu())
    pan, s, k, col = OP.panoptic_fuse(s_c, i_c, tab["is_thing"], tab["inst_class"], tab["inst_id"].long(),
                                      tab["class_id"].long(), tab["palette"])
    assert torch.equal(out["panoptic"][ix].cpu(), pan) and torch.equal(out["f_sem"][ix].cpu(), s)
    assert torch.equal(out["f_slot"][ix].cpu(), k) and torch.equal(out["color"][ix].cpu(), col)
    assert int((k >= 0).sum()) > idx.numel() // 4                      # thing rays with a slot: the slot search runs
    print(f"labels / fusion: {idx.numel()} boundary rays equal the oracle")


# ------------------------------------------------------------------------------------------------ sample_pdf and tags
def test_sample_pdf_and_tags_past_2_31():
    """pnr_sample_pdf at N = Ni = 256, R = 2^22 + 3: z_all [R, 512] holds 2^31 + 1536 elements; then pnr_tag_samples
    on that z_all (sample_box [R, 512] i32).  Coarse depths repeat a block of 509 rays with runs of equal depths, each
    ray shifted by a multiple of 1/4 (exact), weights a block of 503 rays with zero runs, jitter a block of 499 rays;
    the hit intervals are per ray.  Boundary rays against the oracle, bit for bit."""
    R, N, Ni, M = (1 << 22) + 3, 256, 256, 8
    _need(R * (4 * N + (N + Ni)) * 4 + _small(2), "pnr_sample_pdf at 2^31 z_all elements")
    g = torch.Generator().manual_seed(61)
    zb = torch.sort(torch.randint(0, 85, (509, N), generator=g).float() * 0.25 + 1.0, -1).values
    wb = torch.rand(503, N, generator=g) ** 3
    wb[:100] *= (torch.rand(100, N, generator=g) > 0.7)
    wb[100:110] = 0.0
    wb = wb / (wb.sum(-1, keepdim=True) + 1e-3)
    z = _tile(zb, R)
    z += 0.25 * ((torch.arange(R, device=DEV) // 509) % 64).float()[:, None]
    w, u = _tile(wb, R), _tile(torch.rand(499, Ni, generator=g), R)
    z_f, zfb = _poisoned((R, Ni))
    z_all, zab = _poisoned((R, N + Ni))
    _capi.check(_capi.lib().pnr_sample_pdf(z.data_ptr(), w.data_ptr(), R, N, Ni, u.data_ptr(), z_f.data_ptr(), None,
                                           z_all.data_ptr(), _capi.stream_ptr()), "pnr_sample_pdf")
    _tail_intact(zfb, R, "pnr_sample_pdf z_fine")
    _tail_intact(zab, R, "pnr_sample_pdf z_all")
    _crossing("pnr_sample_pdf z_all", R * (N + Ni))

    def run(r0, r1):
        zf, za = P.sample_pdf(z[r0:r1], w[r0:r1], Ni, det=False, u=u[r0:r1])
        return {"z_fine": zf, "z_all": za}
    _check_chunks("pnr_sample_pdf", R, N + Ni, run, {"z_fine": z_f, "z_all": z_all})
    idx = _rows(R, N + Ni, seed=62)
    ix = idx.to(DEV)
    zs, ws, us = z[ix].cpu(), w[ix].cpu(), u[ix].cpu()
    zf_ref, _ = O.sample_pdf(0.5 * (zs[:, 1:] + zs[:, :-1]), ws[:, 1:-1], Ni, det=False, u=us)
    _same_bits(z_f[ix].cpu(), zf_ref, "pnr_sample_pdf z_fine boundary rays")
    _same_bits(z_all[ix].cpu(), O.merge_sorted(zs, zf_ref), "pnr_sample_pdf z_all boundary rays")
    del w, u, z_f, zfb
    torch.cuda.empty_cache()
    # tags on the merged depths
    gd = _gen(63)
    t_in = 1.0 + torch.rand(R, M, generator=gd, device=DEV) * 36
    t_out = t_in + torch.rand(R, M, generator=gd, device=DEV) * 4 * (torch.rand(R, M, generator=gd, device=DEV) > 0.15)
    box_id = torch.randint(0, 50, (R, M), generator=gd, device=DEV, dtype=I32)
    box_id = torch.where(torch.rand(R, M, generator=gd, device=DEV) < 0.2, torch.full_like(box_id, -1), box_id)
    sbox, sbb = _poisoned((R, N + Ni), I32)
    _capi.check(_capi.lib().pnr_tag_samples(z_all.data_ptr(), R, N + Ni, box_id.data_ptr(), t_in.data_ptr(),
                                            t_out.data_ptr(), M, sbox.data_ptr(), _capi.stream_ptr()), "pnr_tag_samples")
    _tail_intact(sbb, R, "pnr_tag_samples sample_box")
    _crossing("pnr_tag_samples sample_box", R * (N + Ni))
    _check_chunks("pnr_tag_samples", R, N + Ni,
                  lambda r0, r1: {"sample_box": P.tag_samples(z_all[r0:r1], box_id[r0:r1], t_in[r0:r1], t_out[r0:r1])},
                  {"sample_box": sbox})
    ref = O.tag_samples(z_all[ix].cpu(), box_id[ix].cpu(), t_in[ix].cpu(), t_out[ix].cpu())
    _same_bits(sbox[ix].cpu(), ref, "pnr_tag_samples boundary rays")
    assert int((ref >= 0).sum()) > idx.numel() * 8                     # samples inside intervals: the tags are exercised


# ------------------------------------------------------------------------------------------------ hash grid
HG = dict(L=32, F=8, T_log2=12, base=2.0, scale=1.25)                  # res 2 .. 2019: dense levels, then hashed


def _hash_call(fn, x, aabb, src, dst):
    _capi.check(getattr(_capi.lib(), fn)(x.data_ptr(), x.shape[0], aabb.data_ptr(), src.data_ptr(), HG["L"], HG["F"],
                                         HG["T_log2"], HG["base"], HG["scale"], dst.data_ptr(), _capi.stream_ptr()), fn)


def test_hashgrid_encode_and_backward_past_2_31():
    """pnr_hashgrid_encode at L = 32, F = 8 (256 outputs per point), n = 2^23 + 5: out holds 2^31 + 1280 elements;
    distinct random points, boundary rows against the oracle bit for bit.  pnr_hashgrid_backward (fp32 atomics: not
    bit for bit) on a grad_out of the same size, against float64 within the bound of
    test_hashgrid_edges_forward_bit_exact_and_backward_against_float64: the first 4096 points are distinct, every
    later point sits on one of 16 known points, so the float64 scatter needs 4096 + 16 points (the later rows of
    grad_out summed per known point in float64, on the device).  The rows of grad_out from 2^23 - 64 on, those around
    and past 2^31, are 2^10 times larger: each is ~0.2% of its known point's sum of |grad_out|, so a kernel that reads
    them from a wrong offset moves the table gradient by far more than the bound."""
    L, F, T = HG["L"], HG["F"], HG["T_log2"]
    n = (1 << 23) + 5
    E = L * F
    _need(2 * n * E * 4 + SMALL * 4 + (1 << 30), "pnr_hashgrid_encode at 2^31 output elements")
    aabb = torch.tensor([[-1.0, -1.0, -1.0], [1.0, 1.0, 1.0]])
    g = torch.Generator().manual_seed(71)
    table = ((torch.rand(L, 1 << T, F, generator=g) * 2 - 1) * 1e4).to(DEV)
    aabb_d = aabb.to(DEV)
    gd = _gen(72)
    x = torch.rand(n, 3, generator=gd, device=DEV) * 2.4 - 1.2
    out, ob = _poisoned((n, E))
    _hash_call("pnr_hashgrid_encode", x, aabb_d, table, out)
    _tail_intact(ob, n, "pnr_hashgrid_encode out")
    _crossing("pnr_hashgrid_encode out", n * E)

    def run(r0, r1):
        o = torch.empty(r1 - r0, E, device=DEV)
        _hash_call("pnr_hashgrid_encode", x[r0:r1], aabb_d, table, o)
        return {"out": o}
    _check_chunks("pnr_hashgrid_encode", n, E, run, {"out": out})
    idx = _rows(n, E, seed=73)
    ref = OP.hashgrid_encode(x[idx.to(DEV)].cpu(), aabb, table.cpu(), HG["base"], HG["scale"])
    _same_bits(out[idx.to(DEV)].cpu(), ref, "pnr_hashgrid_encode boundary rows")
    del out, ob
    torch.cuda.empty_cache()
    # backward
    U = 4096
    known = torch.rand(16, 3, generator=g) * 2 - 1
    xb = torch.empty(n, 3, device=DEV)
    xb[:U] = x[:U]
    xb[U:] = known.to(DEV)[torch.arange(U, n, device=DEV) % 16]
    del x
    grad_out = torch.randn(n, E, generator=gd, device=DEV)
    grad_out[(1 << 23) - 64:] *= 2.0 ** 10
    gt_flat, gtb = _poisoned((L * (1 << T) * F,), tail=F)
    gt_flat.zero_()
    _hash_call("pnr_hashgrid_backward", xb, aabb_d, grad_out, gt_flat)
    _tail_intact(gtb, gt_flat.numel(), "pnr_hashgrid_backward grad_table")
    _crossing("pnr_hashgrid_backward grad_out", n * E)
    # float64: the distinct points as they are, the known points with their rows of grad_out summed
    Gs = torch.zeros(16, E, dtype=F64, device=DEV)
    As = torch.zeros(16, E, dtype=F64, device=DEV)
    for c0 in range(U, n, 1 << 20):
        c1 = min(n, c0 + (1 << 20))
        gg = grad_out[c0:c1].double()
        j = torch.arange(c0, c1, device=DEV) % 16
        Gs.index_add_(0, j, gg)
        As.index_add_(0, j, gg.abs())
        del gg
    pts = torch.cat([xb[:U].cpu(), known])
    up = torch.cat([grad_out[:U].cpu().double(), Gs.cpu()])
    up_abs = torch.cat([grad_out[:U].cpu().double().abs(), As.cpu()])
    t64 = table.cpu().double().requires_grad_(True)
    (OP.hashgrid_encode(pts, aabb, t64, HG["base"], HG["scale"]) * up).sum().backward()
    t64a = table.cpu().double().requires_grad_(True)
    (OP.hashgrid_encode(pts, aabb, t64a, HG["base"], HG["scale"]) * up_abs).sum().backward()
    got = gt_flat.view(L, 1 << T, F).cpu().double()
    assert torch.equal(got == 0, t64a.grad == 0)
    _report(f"pnr_hashgrid_backward n={n}", _ratio((got - t64.grad).abs(), 1e-4 * t64a.grad))


# ------------------------------------------------------------------------------------------------ fused MLP
def _net(precision="fp16x3", **over):
    cfg = make_cfg("cfg2", precision=precision, **over)
    net = SY.init_network_weights(make_network(cfg), seed=81).to(DEV)
    return cfg, net


def _points(S, seed):
    g = _gen(seed)
    pts = (torch.rand(S, 3, generator=g, device=DEV) * 2 - 1) * 4
    vd = torch.randn(S, 3, generator=g, device=DEV)
    vd /= torch.linalg.vector_norm(vd, dim=-1, keepdim=True)
    return pts, vd


def _dyadic(R, N, seed):
    """Rays whose sample points o + d z are exact in fp32 (o on a 1/16 grid, d on a 1/8 grid, z ascending on a 1/16
    grid), so float64 sees the points the kernel forms."""
    g = _gen(seed)
    o = torch.round((torch.rand(R, 3, generator=g, device=DEV) * 4 - 2) * 16) / 16
    d = torch.round(torch.nn.functional.normalize(torch.randn(R, 3, generator=g, device=DEV), dim=-1) * 8) / 8
    d[(d == 0).all(-1), 0] = 1.0
    z = torch.sort(torch.randint(1, 257, (R, N), generator=g, device=DEV).float() / 16, -1).values
    return torch.cat([o, d], -1).contiguous(), z.contiguous()


def _mlp_forward(ctx, pts, vd, rays, z, raw):
    R, N = (pts.shape[0], 1) if pts is not None else z.shape
    _capi.check(_capi.lib().pnr_mlp_forward(ctx, _capi.ptr(pts), _capi.ptr(vd), _capi.ptr(rays), _capi.ptr(z), R, N,
                                            raw.data_ptr(), _capi.stream_ptr()), "pnr_mlp_forward")


def _trunk_forward(ctx, pts, h):
    _capi.check(_capi.lib().pnr_mlp_trunk_forward(ctx, pts.data_ptr(), None, None, pts.shape[0], 1, h.data_ptr(),
                                                  _capi.stream_ptr()), "pnr_mlp_trunk_forward")


def _bound_report(what, got, ref, B, groups):
    r = ratio(got.double(), ref, B)
    worst = {k: float(r[:, sl].max()) for k, sl in groups.items()}
    print(f"{what}: largest error / bound " + " ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    assert max(worst.values()) <= 1.0, f"{what}: an element outside the bound {worst}"


def test_mlp_forward_and_composite_with_heads_past_2_31():
    """pnr_mlp_forward with C = K = 128 heads (D = 8, W = 256, 260 channels; the 64-row kernel) at S = 8 300 017
    points: raw holds 2.16e9 elements; then rays mode at 43 241 rays x 192 samples (raw 2.16e9 elements), and
    pnr_mlp_composite on those rays, whose per-ray maps and weights must equal small launches and, on the boundary
    rays, pnr_composite of the rays-mode raw (weights and fixed maps bit for bit, the maps within test_gpu_render_limits'
    float64 model).  Boundary rows of raw against oracle_bound.forward_bound, as test_gpu_forward_bound holds them."""
    Cn = Kn = 128
    CH = 4 + Cn + Kn
    S = 8_300_017
    Rr, Nr = 43_241, 192
    _need(S * CH * 4 + _small() + S * 24, "pnr_mlp_forward at 2.16e9 raw elements")
    cfg, net = _net(num_classes=Cn, num_instances=Kn)
    ctx = net.pack(torch.device(DEV))
    net.range_status()
    groups = {"rgb": slice(0, 3), "sigma": slice(3, 4), "sem": slice(4, 4 + Cn), "inst": slice(4 + Cn, CH)}
    # points mode
    pts, vd = _points(S, 82)
    raw, rb = _poisoned((S, CH))
    _mlp_forward(ctx, pts, vd, None, None, raw)
    _tail_intact(rb, S, "pnr_mlp_forward raw")
    _crossing("pnr_mlp_forward (points) raw", S * CH)

    def run(r0, r1):
        o = torch.empty(r1 - r0, CH, device=DEV)
        _mlp_forward(ctx, pts[r0:r1], vd[r0:r1], None, None, o)
        return {"raw": o}
    _check_chunks("pnr_mlp_forward (points)", S, CH, run, {"raw": raw})
    idx = _rows(S, CH, seed=83)
    ix = idx.to(DEV)
    ex, e_ex = trunk_input(cfg, net, pts[ix].cpu())
    ed, e_ed = view_encoding(vd[ix].cpu(), cfg.view_res)
    ref, B, _, _ = forward_bound(net, cfg.precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV), chunk=256)
    _bound_report(f"pnr_mlp_forward (points) S={S} boundary rows ({idx.numel()})", raw[ix], ref, B, groups)
    assert net.range_status() == 0
    del raw, rb, pts, vd
    torch.cuda.empty_cache()
    # rays mode
    rays, z = _dyadic(Rr, Nr, 84)
    raw, rb = _poisoned((Rr, Nr, CH))
    _mlp_forward(ctx, None, None, rays, z, raw)
    _tail_intact(rb, Rr, "pnr_mlp_forward rays raw")
    _crossing("pnr_mlp_forward (rays) raw", Rr * Nr * CH)

    def run_r(r0, r1):
        o = torch.empty(r1 - r0, Nr, CH, device=DEV)
        _mlp_forward(ctx, None, None, rays[r0:r1], z[r0:r1], o)
        return {"raw": o}
    _check_chunks("pnr_mlp_forward (rays)", Rr, Nr * CH, run_r, {"raw": raw})
    # 40 random rays: each is 192 samples through the float64 bound of a network with two 128-wide heads, so the
    # boundary rays and these give ~8 000 samples, more than the points mode's 1000 rows
    idx = _rows(Rr, Nr * CH, n_random=40, seed=85)
    ix = idx.to(DEV)
    rs, zs = rays[ix].cpu().double(), z[ix].cpu().double()
    p3 = (rs[:, None, :3] + rs[:, None, 3:] * zs[..., None]).reshape(-1, 3)
    d3 = (rs[:, 3:] / rs[:, 3:].norm(dim=-1, keepdim=True))[:, None].expand(-1, Nr, -1).reshape(-1, 3)
    ex, e_ex = trunk_input(cfg, net, p3.float())
    ed, e_ed = view_encoding(d3, cfg.view_res, rel=VIEWDIR_REL)
    ref, B, _, _ = forward_bound(net, cfg.precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV), chunk=256)
    _bound_report(f"pnr_mlp_forward (rays) R={Rr} boundary rays ({idx.numel()})", raw[ix].reshape(-1, CH), ref, B, groups)
    assert net.range_status() == 0
    # the same rays through pnr_mlp_composite
    g = _gen(86)
    sb = torch.randint(-3, 23, (Rr, Nr), generator=g, device=DEV, dtype=I32)
    bs = torch.randint(-2, Cn + 3, (20,), generator=g, device=DEV, dtype=I32)
    bi = torch.randint(-2, Kn + 3, (20,), generator=g, device=DEV, dtype=I32)

    def composite(r0, r1, poison=False):
        o, bufs = {}, {}
        for k in COMP_MAPS:
            if poison:
                o[k], bufs[k] = _poisoned(_map_shape(k, r1 - r0, Nr, Cn, Kn))
            else:
                o[k] = torch.empty(_map_shape(k, r1 - r0, Nr, Cn, Kn), device=DEV)
        co = _capi.ptr_struct(_capi.PnrCompositeOut, o)
        _capi.check(_capi.lib().pnr_mlp_composite(ctx, rays[r0:r1].data_ptr(), z[r0:r1].data_ptr(), r1 - r0, Nr, 0, 1,
                                                  sb[r0:r1].data_ptr(), bs.data_ptr(), bi.data_ptr(), 20, C.byref(co),
                                                  _capi.stream_ptr()), "pnr_mlp_composite")
        for k, b in bufs.items():
            _tail_intact(b, r1 - r0, f"pnr_mlp_composite {k}")
        return o
    full = composite(0, Rr, poison=True)
    _check_chunks("pnr_mlp_composite", Rr, Nr * CH, composite, full)
    two = P.raw2outputs(raw[ix], z[ix], rays[ix], mask_outside=True, num_classes=Cn, num_instances=Kn,
                        sample_box=sb[ix], box_sem=bs, box_inst=bi)
    got = {k: v[ix] for k, v in full.items()}
    for k in ("weights", "fixed_semantic_map", "fixed_instance_map"):
        _same_bits(got[k], two[k], f"pnr_mlp_composite {k} against pnr_composite")
    worst, where = _per_ray_ratio(got, raw[ix], z[ix], rays[ix], Cn, Kn, sb[ix], bs, bi, False, True, softmax=False)
    _report(f"pnr_mlp_composite R={Rr} boundary rays ({idx.numel()}) [{where}]", worst)
    assert net.range_status() == 0


def test_mlp_trunk_forward_past_2_31():
    """pnr_mlp_trunk_forward of the default network without heads (D = 8, W = 256; the 64-row kernel, which every
    trunk-forward launch runs) at S = 2^23 + 17: h_out holds 2^31 + 4352 elements; boundary rows against
    forward_bound's trunk output."""
    S = (1 << 23) + 17
    Wd = 256
    _need(S * Wd * 4 + _small() + S * 24, "pnr_mlp_trunk_forward at 2^31 h elements")
    cfg, net = _net()
    ctx = net.pack(torch.device(DEV))
    net.range_status()
    pts, vd = _points(S, 91)
    h, hb = _poisoned((S, Wd))
    _trunk_forward(ctx, pts, h)
    _tail_intact(hb, S, "pnr_mlp_trunk_forward h")
    _crossing("pnr_mlp_trunk_forward h", S * Wd)

    def run(r0, r1):
        o = torch.empty(r1 - r0, Wd, device=DEV)
        _trunk_forward(ctx, pts[r0:r1], o)
        return {"h": o}
    _check_chunks("pnr_mlp_trunk_forward", S, Wd, run, {"h": h})
    idx = _rows(S, Wd, seed=92)
    ix = idx.to(DEV)
    ex, e_ex = trunk_input(cfg, net, pts[ix].cpu())
    ed, e_ed = view_encoding(vd[ix].cpu(), cfg.view_res)
    _, _, h_ref, h_B = forward_bound(net, cfg.precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV), chunk=256)
    _bound_report(f"pnr_mlp_trunk_forward S={S} boundary rows ({idx.numel()})", h[ix], h_ref, h_B, {"h": slice(0, Wd)})
    assert net.range_status() == 0


def test_mlp_forward_128_row_kernel_past_2_31():
    """pnr_mlp_forward of the default network without heads (D = 8, W = 256) on the 128-row kernel, its default for
    that network, at S = 2^29 + 17 points: raw [S, 4] holds 2^31 + 68 elements, pts and viewdirs 1.6e9 each.  That
    kernel keeps the trunk's activations in shared memory, so these three are its only global buffers.  raw against
    small launches of the 128-row kernel and against the 64-row kernel at the same S, bit for bit; boundary rows
    against forward_bound."""
    S = (1 << 29) + 17
    _need(S * (3 + 3 + 4 + 4) * 4 + _small(), "pnr_mlp_forward (128 rows) at 2^31 raw elements")
    cfg, net = _net()
    ctx = net.pack(torch.device(DEV))
    net.range_status()
    pts, vd = _points(S, 93)
    raw, rb = _poisoned((S, 4))
    _capi.set_mlp_rows(ctx, 128)                  # PNR_ERR_UNSUPPORTED if this network could not run 128-row tiles
    try:
        _mlp_forward(ctx, pts, vd, None, None, raw)
        _tail_intact(rb, S, "pnr_mlp_forward (128 rows) raw")
        _crossing("pnr_mlp_forward (128 rows) raw", S * 4)

        def run(r0, r1):
            o = torch.empty(r1 - r0, 4, device=DEV)
            _mlp_forward(ctx, pts[r0:r1], vd[r0:r1], None, None, o)
            return {"raw": o}
        _check_chunks("pnr_mlp_forward (128 rows)", S, 4, run, {"raw": raw})
        _capi.set_mlp_rows(ctx, 64)
        raw64, rb64 = _poisoned((S, 4))
        _mlp_forward(ctx, pts, vd, None, None, raw64)
        _tail_intact(rb64, S, "pnr_mlp_forward (64 rows) raw")
    finally:
        _capi.set_mlp_rows(ctx, 0)
    _same_bits(raw64, raw, "pnr_mlp_forward: the 64-row kernel against the 128-row kernel")
    del raw64, rb64
    idx = _rows(S, 4, seed=94)
    ix = idx.to(DEV)
    ex, e_ex = trunk_input(cfg, net, pts[ix].cpu())
    ed, e_ed = view_encoding(vd[ix].cpu(), cfg.view_res)
    ref, B, _, _ = forward_bound(net, cfg.precision, ex.to(DEV), e_ex.to(DEV), ed.to(DEV), e_ed.to(DEV), chunk=256)
    _bound_report(f"pnr_mlp_forward (128 rows) S={S} boundary rows ({idx.numel()})", raw[ix], ref, B,
                  {"rgb": slice(0, 3), "sigma": slice(3, 4)})
    assert net.range_status() == 0


def _backward_call(ctx, pts, grad_h, gs, emb, ld, st, am):
    _capi.check(_capi.lib().pnr_mlp_backward_trunk(ctx, pts.data_ptr(), None, None, pts.shape[0], 1, grad_h.data_ptr(),
                                                   float(gs), emb.data_ptr(), ld, st.data_ptr(), _capi.ptr(am),
                                                   _capi.stream_ptr()), "pnr_mlp_backward_trunk")


def test_mlp_backward_trunk_stash_past_2_32():
    """pnr_mlp_backward_trunk with its stash and stash_absmax, D = 8, W = 256, S = 2^20 + 17: the stash [15, S, W]
    holds 4.03e9 elements, slots >= 8 start past 2^31 and slot 15's last rows pass 2^32.  Stash and d(trunk input)
    against small launches; the samples whose stash rows hold 2^31 - 1 .. 2^32 (and the first, last and random ones)
    through every link of test_gpu_backward_bound (the forward bound of each H slot, the masks, the last slot bit for
    bit, every dZ slot and d(trunk input) within backward_bound); stash_absmax against the maxima of the stash read
    back, bit for bit."""
    S = (1 << 20) + 17
    cfg, net = _net()
    D, Wd = cfg.D, cfg.W
    slots = 2 * D - 1
    _need(slots * S * Wd * 4 + S * (Wd + 64) * 4 + _small(), "pnr_mlp_backward_trunk at 4e9 stash elements")
    ctx = net.pack(torch.device(DEV))
    net.range_status()
    pts, _ = _points(S, 101)
    grad_h = torch.randn(S, Wd, generator=_gen(102), device=DEV)
    gs = default_grad_scale(grad_h)
    Ex = net.in_dim
    ld = (Ex + 15) // 16 * 16
    emb, eb = _poisoned((S, ld))
    sflat, sfb = _poisoned((slots * S * Wd,), tail=Wd)
    st = sflat.view(slots, S, Wd)
    am, ab = _poisoned((slots,), I32)
    _backward_call(ctx, pts, grad_h, gs, emb, ld, st, am)
    assert net.range_status() == 0
    _tail_intact(eb, S, "grad_emb")
    _tail_intact(sfb, slots * S * Wd, "stash")
    _tail_intact(ab, slots, "stash_absmax")
    _crossing("pnr_mlp_backward_trunk stash", slots * S * Wd)

    def run(r0, r1):
        e = torch.empty(r1 - r0, ld, device=DEV)
        s = torch.empty(slots, r1 - r0, Wd, device=DEV)
        _backward_call(ctx, pts[r0:r1], grad_h[r0:r1], gs, e, ld, s, None)
        return {"grad_emb": e, **{f"stash slot {k}": s[k] for k in range(slots)}}
    _check_chunks("pnr_mlp_backward_trunk", S, slots * Wd, run,
                  {"grad_emb": emb, **{f"stash slot {k}": st[k] for k in range(slots)}})
    # stash_absmax: the hi part of each slot's largest magnitude, the gradient slots seen scaled
    half = torch.float16 if cfg.precision.startswith("fp16") else torch.bfloat16
    scale = torch.ones(slots, device=DEV)
    scale[D - 1:] = gs
    want = (torch.stack([torch.linalg.vector_norm(st[k], ord=float("inf")) for k in range(slots)]) * scale).to(half)
    assert torch.equal(am.to(torch.int16).view(half), want), (am, want)
    # float64 on the samples whose stash rows hold the boundaries, in any slot
    s = {0, S - 1}
    for b in (B31 - 1, B31, B32 - 1, B32):
        if b < slots * S * Wd:
            s.add((b // Wd) % S)
    s.update(torch.randint(0, S, (1000,), generator=torch.Generator().manual_seed(103)).tolist())
    idx = torch.tensor(sorted(s))
    ix = idx.to(DEV)
    p_sel = pts[ix].contiguous()
    ex, e_ex = trunk_input(cfg, net, p_sel.cpu())
    st_sel = st[:, ix]
    with torch.no_grad():
        h_fwd = net.trunk_forward(pts=p_sel)
    name = f"pnr_mlp_backward_trunk S={S} boundary samples ({idx.numel()})"
    b = pinned_bound(name, net, cfg.precision, ex, e_ex, grad_h[ix], gs, st_sel, h_fwd)
    check_within(name, b, emb[ix, :Ex], st_sel)


# ------------------------------------------------------------------------------------------------ pnr_wgrad, pnr_linear
def test_wgrad_past_2_31():
    """pnr_wgrad at No = Ni = 256, S = 2^23 + 65: dZ and X hold 2^31 + 16640 elements each.  Split-K order depends on
    S, so every element of dW and db is held to float64 over all rows (on the device) within oracle_bound.wgrad_bound,
    in both precisions.  The rows of dZ from 2^23 - 64 on, around and past 2^31, are 2^20 times larger: dW is
    dominated by them, so a kernel reading them from a wrong offset fails the bound."""
    S, No, Ni = (1 << 23) + 65, 256, 256
    _need(2 * S * No * 4 + (3 << 30), "pnr_wgrad at 2^31 operand elements")
    g = _gen(111)
    x = torch.randn(S, Ni, generator=g, device=DEV)
    x[:, ::3].relu_()
    dz = torch.randn(S, No, generator=g, device=DEV).mul_(1e-6)
    dz[(1 << 23) - 64:] *= 2.0 ** 20
    _crossing("pnr_wgrad dZ and X", S * No)
    ref = _ref_wgrad(dz, x)
    for prec in ("fp16x3", "bf16x3"):
        sc = _pow2_scale(dz) if prec == "fp16x3" else None
        Wv, Wb = _poisoned((No, Ni))
        bv, bb = _poisoned((No,))
        W, b = _wgrad(dz, x, prec, sc, W=Wv, b=bv)
        _tail_intact(Wb, No, "pnr_wgrad dW")
        _tail_intact(bb, No, "pnr_wgrad db")
        _check_wgrad(W, b, ref, S, prec, float(sc) if sc is not None else 1.0, f"pnr_wgrad {prec} S={S}", contract=False)


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_linear_past_2_31(prec):
    """pnr_linear at K = N = 256, S = 2^23 + 65 (bias, ReLU): x and y hold 2^31 + 16640 elements; y against small
    launches bit for bit and its boundary rows against float64 within test_gpu_train_limits' per-element bound."""
    S, K, N = (1 << 23) + 65, 256, 256
    _need(2 * S * K * 4 + _small(), "pnr_linear at 2^31 elements")
    g = _gen(121)
    x = torch.randn(S, K, generator=g, device=DEV)
    x[:, ::3].relu_()
    Wt = torch.randn(N, K, generator=g, device=DEV) / 16
    bias = torch.randn(N, generator=g, device=DEV) * 0.1
    y, yb = _poisoned((S, N))
    _linear(x, Wt, N, prec, bias=bias, relu=True, y=y)
    _tail_intact(yb, S, "pnr_linear y")
    _crossing("pnr_linear x and y", S * K)
    _check_chunks(f"pnr_linear {prec}", S, max(K, N),
                  lambda r0, r1: {"y": _linear(x[r0:r1], Wt, N, prec, bias=bias, relu=True)}, {"y": y})
    idx = _rows(S, N, seed=122).to(DEV)
    _check_linear(y[idx], x[idx], Wt, prec, bias, True, False, 1.0, f"pnr_linear {prec} S={S} boundary rows ({idx.numel()})")
