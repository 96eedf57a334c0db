"""The training path's GEMM kernels at the shapes and sample counts they accept, element by element against float64:
pnr_wgrad (csrc/wgrad_wgmma.cu: every weight and bias gradient) and pnr_linear (csrc/linear_wgmma.cu: the layers after
the trunk, forward and input gradient), through the C ABI; and network_backward at a training step's batch.

The reference is float64 on the device (torch float64 matmuls, in sample chunks of at most 2^18 rows), pinned once
against the CPU.  Every element is held to its own bound, |got - ref| <= tau * A + floor, where A is the same sum
over absolute values (|dZ|^T |X|, or |x| |W|^T + |b|): an entry that is small because its column is small, or
because its terms cancel, is held to what its own terms allow, not to the RMS of the whole tensor.
  tau   = 3 u^2 (the operand split: hi / lo 16-bit parts with unit roundoff u, the lo.lo product dropped)
        + (accumulating wgmmas in one run) * 2^-23 (the tensor cores' fp32 accumulation truncates: at most about one
          ulp of the running sum per instruction; pnr_wgrad restarts its register accumulators every RUN_SLABS slabs
          and adds the run to the CTA's partial, so a run is at most 12 * RUN_SLABS wgmmas whatever S is)
        + round-to-nearest adds of the runs and of the CTAs' partials.
The path's contract, dW within 2e-5 (fp16x3) / 1e-4 (bf16x3) of the RMS and db within 1e-4, is asserted at every S,
except on the column-spread data: there the largest entries are several times the RMS, so a share of the RMS asks
more than 2e-5 of those entries; the per-element bound is what holds them.
  floor = 2^-24 * (sum |x| / scale + sum |dz|) in fp16x3, where a 16-bit part can be subnormal.
Each check prints the largest error it measured as a share of its bound (1 is the bound)."""
import math

import pytest
import torch

from oracle_bound import WGRAD_RUN_SLABS, WGRAD_U, wgrad_bound
from panopticnerf_b200 import _capi
from panopticnerf_b200.lib.train.mlp_backward import _pow2_scale

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64
CHUNK = 1 << 18
U = WGRAD_U                                            # unit roundoff of one 16-bit operand part
RUN_SLABS = WGRAD_RUN_SLABS                           # pnr_wgrad: slabs of 64 samples per run of the register accumulators
CONTRACT = {"fp16x3": 2e-5, "bf16x3": 1e-4}           # pnr_wgrad's dW: max error / RMS of the result


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _report(what, ratio):
    print(f"{what}: largest error / bound = {ratio:.3e}")
    assert ratio <= 1.0, f"{what}: error {ratio:.3e} x its bound"


def _ratio(err, bound):
    """max of err / bound, where a zero bound demands an exact zero error (and NaN errors fail)."""
    assert not bool(torch.isnan(err).any()), "NaN in the result"
    assert bool((err[bound == 0] == 0).all()), "nonzero error where every term is exactly 0"
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


def _ptr(t):
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------ pnr_wgrad
_WS = {}


def _workspace():
    if "wgrad" not in _WS:
        _WS["wgrad"] = torch.empty(int(_capi.lib().pnr_wgrad_workspace_bytes(256, 256)), dtype=torch.uint8, device=DEV)
    return _WS["wgrad"]


def _wgrad(dz, x, prec, scale=None, W=None, b=True, accumulate=0, S=None, ws=True):
    """pnr_wgrad on dz [S, No] and x [S, Ni] (row-strided views as they are).  W: [No, ld_w] output (new: ld_w = Ni);
    b: a [No] output, True for a new one, None for NULL.  Returns (W, b)."""
    S_ = dz.shape[0] if S is None else S
    No, Ni = dz.shape[1], x.shape[1]
    W = torch.empty(No, Ni, device=DEV) if W is None else W
    b = torch.empty(No, device=DEV) if b is True else b
    w = _workspace() if ws else None
    rc = _capi.lib().pnr_wgrad(dz.data_ptr(), max(dz.stride(0), No), No, x.data_ptr(), max(x.stride(0), Ni), Ni, S_,
                               _capi.PREC[prec], _ptr(scale), W.data_ptr(), W.stride(0), _ptr(b), accumulate,
                               _ptr(w), 0 if w is None else w.numel(), _capi.stream_ptr())
    _capi.check(rc, "pnr_wgrad")
    return W, b


def _ref_wgrad(dz, x):
    """float64 on the device: dZ^T X, |dZ|^T |X|, column sums of dZ and |dZ|, column sums of |X|."""
    No, Ni = dz.shape[1], x.shape[1]
    R, A = torch.zeros(No, Ni, dtype=F64, device=DEV), torch.zeros(No, Ni, dtype=F64, device=DEV)
    rb, ab, cx = torch.zeros(No, dtype=F64, device=DEV), torch.zeros(No, dtype=F64, device=DEV), torch.zeros(Ni, dtype=F64, device=DEV)
    for c in range(0, dz.shape[0], CHUNK):
        a, v = dz[c:c + CHUNK].double(), x[c:c + CHUNK].double()
        R.addmm_(a.t(), v)
        rb += a.sum(0)
        a.abs_(), v.abs_()
        A.addmm_(a.t(), v)
        ab += a.sum(0)
        cx += v.sum(0)
        del a, v
    return R, A, rb, ab, cx


def _check_wgrad(W, b, ref, S, prec, sc, what, contract=True):
    """Every element of dW and db within its bound (oracle_bound.wgrad_bound); dW within the path's contract of the
    RMS, db within 1e-4."""
    R, A, rb, ab, cx = ref
    bW, bb = wgrad_bound(A, ab, cx, S, R.shape[0], prec, sc, _sms())
    r = _ratio((W.double() - R).abs(), bW)
    rbias = _ratio((b.double() - rb).abs(), bb) if b is not None else 0.0
    _report(f"{what} dW", r)
    _report(f"{what} db", rbias)
    if contract:
        e_rms = float((W.double() - R).abs().max()) / max(float(R.pow(2).mean().sqrt()), 1e-300)
        e_b = float((b.double() - rb).abs().max()) / max(float(rb.pow(2).mean().sqrt()), 1e-300) if b is not None else 0.0
        print(f"{what}: max err / rms  dW {e_rms:.2e}  db {e_b:.2e}")
        assert e_rms <= CONTRACT[prec] and e_b <= 1e-4, (e_rms, e_b)
    return r


def _data(S, No, Ni, regime, seed):
    """dZ [S, No], X [S, Ni] on the device.
    random: random signs.  adversarial: X >= 0 (ReLU'd), dZ with a same-sign mean on half of its columns, so the
    running sums grow linearly.  spread: both operands' columns scaled over 1e-4 .. 1.  gated: ReLU-gated exact zeros
    in both (and whole zero columns)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(S, Ni, device=DEV, generator=g)
    dz = torch.randn(S, No, device=DEV, generator=g)
    if regime == "random":
        pass
    elif regime == "adversarial":
        x.abs_()
        dz[:, ::2] = dz[:, ::2].abs_() + 0.5
    elif regime == "spread":
        x.relu_()
        dz += 0.3
        x *= torch.logspace(-4, 0, Ni, device=DEV)[torch.randperm(Ni, device=DEV, generator=g)]
        dz *= torch.logspace(-4, 0, No, device=DEV)[torch.randperm(No, device=DEV, generator=g)]
    elif regime == "gated":
        x.relu_()
        dz *= (torch.rand(S, No, device=DEV, generator=g) < 0.4)
        dz[:, No // 3] = 0
        x[:, Ni // 2] = 0
    return dz.mul_(1e-6), x                             # gradients of a mean-reduced loss are ~1e-6


def _scale(dz, prec):
    return _pow2_scale(dz) if prec == "fp16x3" else None


def _run_wgrad(dz, x, prec, what, scale="pow2", contract=True):
    sc = _pow2_scale(dz) if (prec == "fp16x3" and scale == "pow2") else scale if not isinstance(scale, str) else None
    W, b = _wgrad(dz, x, prec, sc)
    return _check_wgrad(W, b, _ref_wgrad(dz, x), dz.shape[0], prec, float(sc) if sc is not None else 1.0, what, contract), W, b


def test_float64_reference_on_device_equals_cpu():
    """The device reference is float64 throughout (TF32 settings do not reach it): it matches the CPU's to rounding."""
    dz, x = _data(3001, 37, 129, "spread", seed=1)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        R, A, rb, ab, cx = _ref_wgrad(dz, x)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    Rc = dz.cpu().double().t() @ x.cpu().double()
    Ac = dz.cpu().double().abs().t() @ x.cpu().double().abs()
    assert float(((R.cpu() - Rc).abs() / Ac.clamp(min=1e-300)).max()) < 1e-13
    assert float(((A.cpu() - Ac).abs() / Ac.clamp(min=1e-300)).max()) < 1e-13
    assert torch.allclose(rb.cpu(), dz.cpu().double().sum(0), rtol=1e-13, atol=0)


WGRAD_SHAPES = [(1, 1), (15, 3), (16, 4), (17, 5), (127, 15), (128, 16), (129, 17), (255, 127), (256, 128), (1, 129),
                (17, 241), (129, 255), (256, 256), (255, 3), (128, 255), (16, 127)]


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("No,Ni", WGRAD_SHAPES)
def test_wgrad_shapes_and_short_sample_counts(No, Ni, prec):
    worst = 0.0
    for S in (1, 7, 8, 9, 63, 64, 65, 1000):
        dz, x = _data(S, No, Ni, "gated" if S % 2 else "adversarial", seed=S + No + Ni)
        worst = max(worst, _run_wgrad(dz, x, prec, f"wgrad {prec} No={No} Ni={Ni} S={S}", contract=S >= 64)[0])
    print(f"wgrad {prec} No={No} Ni={Ni}: worst over S = {worst:.3e}")


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("No", [128, 256])
def test_wgrad_around_the_grid_boundaries(No, prec):
    """S where the grid stops growing (one slab per CTA), and where the CTAs' runs fill up: 64 (CTAs per block +- 1)
    + {0, 1, 63}, and around a run's end: 64 * CTAs * RUN_SLABS + {0, 1, 64}."""
    per = _sms() // (2 if No > 128 else 1)
    Ss = [64 * (per + d) + r for d in (-1, 0, 1) for r in (0, 1, 63)] + [64 * per * RUN_SLABS + r for r in (0, 1, 64)]
    for S in Ss:
        dz, x = _data(S, No, 129, "adversarial", seed=S)
        _run_wgrad(dz, x, prec, f"wgrad {prec} No={No} S={S}")


@pytest.mark.parametrize("regime", ["random", "adversarial", "spread", "gated"])
def test_wgrad_at_a_training_steps_sample_count(regime):
    """S = 393 216 (2048 rays x 192 samples), No = Ni = 256, both precisions; two runs give the same bits."""
    dz, x = _data(393216, 256, 256, regime, seed=7)
    for prec in ("fp16x3", "bf16x3"):
        _, W, b = _run_wgrad(dz, x, prec, f"wgrad {prec} S=393216 {regime}", contract=regime != "spread")
        W2, b2 = _wgrad(dz, x, prec, _scale(dz, prec))
        assert torch.equal(W, W2) and torch.equal(b, b2)


@pytest.mark.parametrize("regime", ["random", "adversarial", "spread", "gated"])
@pytest.mark.parametrize("S,No,Ni", [(1 << 21, 256, 256), (1 << 23, 256, 32)])
def test_wgrad_long_accumulations(S, No, Ni, regime):
    """The longest per-CTA shares of the samples: S = 2^21 at 256 x 256, and S = 2^23 at No = 256 (~9.7 GB of
    operands); the adversarial data's sums grow linearly with S."""
    dz, x = _data(S, No, Ni, regime, seed=3)
    for prec in ("fp16x3", "bf16x3"):
        _run_wgrad(dz, x, prec, f"wgrad {prec} S={S} No={No} Ni={Ni} {regime}", contract=regime != "spread")
    del dz, x
    torch.cuda.empty_cache()


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_wgrad_contract_over_long_runs(prec):
    """All-positive data at a training step's S: before the runs were bounded, the truncating accumulation drifted to
    5e-5 of the RMS here."""
    dz, x = _data(393216, 256, 256, "adversarial", seed=7)
    W, _ = _wgrad(dz, x, prec, _scale(dz, prec))
    R = _ref_wgrad(dz, x)[0]
    e_rms = float((W.double() - R).abs().max() / R.pow(2).mean().sqrt())
    print(f"wgrad {prec} S=393216 adversarial: max err / rms {e_rms:.2e}")
    assert e_rms <= CONTRACT[prec]


def test_wgrad_fp16_and_bf16_ranges():
    g = torch.Generator(device=DEV).manual_seed(5)
    S, No, Ni = 20000, 129, 65
    # fp16x3 without dz_scale on O(1) data
    dz, x = torch.randn(S, No, device=DEV, generator=g), torch.rand(S, Ni, device=DEV, generator=g)
    _run_wgrad(dz, x, "fp16x3", "wgrad fp16x3 O(1) dz_scale=NULL", scale=None)
    # fp16x3 with |X| and |dZ * scale| just below 65504
    dz = torch.rand(S, No, device=DEV, generator=g) * 1.99
    x = torch.rand(S, Ni, device=DEV, generator=g) * 65000.0
    sc = torch.tensor([2.0 ** 15], device=DEV)
    assert float(dz.abs().max() * 2 ** 15) < 65504 and float(x.max()) < 65504
    _run_wgrad(dz, x, "fp16x3", "wgrad fp16x3 near 65504", scale=sc)
    # bf16x3 at 1e+-30: fp32's exponent range
    dz = torch.randn(S, No, device=DEV, generator=g) * 1e30
    x = torch.rand(S, Ni, device=DEV, generator=g) * 1e-30
    _run_wgrad(dz, x, "bf16x3", "wgrad bf16x3 dz 1e30 x 1e-30")
    dz = torch.randn(S, No, device=DEV, generator=g) * 1e-30
    x = torch.rand(S, Ni, device=DEV, generator=g) * 1e30
    _run_wgrad(dz, x, "bf16x3", "wgrad bf16x3 dz 1e-30 x 1e30")


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_wgrad_accumulate_row_stride_and_no_bias(prec):
    S, No, Ni = 5000, 200, 37
    dz, x = _data(S, No, Ni, "spread", seed=9)
    sc = _scale(dz, prec)
    fresh_W, fresh_b = _wgrad(dz, x, prec, sc)
    # ld_w > Ni: the columns past Ni are never written
    Wbuf = torch.full((No, Ni + 7), float("nan"), device=DEV)
    W, b = _wgrad(dz, x, prec, sc, W=Wbuf[:, :Ni])
    assert torch.equal(W, fresh_W) and torch.equal(b, fresh_b) and bool(Wbuf[:, Ni:].isnan().all())
    # accumulate = 1: prev + fresh, bit for bit, for dW and db
    prev_W, prev_b = torch.randn(No, Ni, device=DEV) * 1e-3, torch.randn(No, device=DEV) * 1e-3
    acc_W, acc_b = prev_W.clone(), prev_b.clone()
    _wgrad(dz, x, prec, sc, W=acc_W, b=acc_b, accumulate=1)
    assert torch.equal(acc_W, prev_W + fresh_W) and torch.equal(acc_b, prev_b + fresh_b)
    # db = NULL: dW is the same
    W, b = _wgrad(dz, x, prec, sc, b=None)
    assert b is None and torch.equal(W, fresh_W)


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_wgrad_four_byte_loads_equal_sixteen_byte_loads(prec):
    """Contiguous operands with widths of multiples of 4 take the 16-byte load path; a base one float off 16-byte
    alignment and an odd row stride take the 4-byte path: same bits."""
    S, No, Ni = 3001, 128, 64
    dz, x = _data(S, No, Ni, "gated", seed=4)
    for t in (dz, x):                                      # the 16-byte path's conditions (pnr_wgrad: vec_a / vec_b)
        assert t.data_ptr() % 16 == 0 and t.stride(0) % 4 == 0
    sc = _scale(dz, prec)
    W, b = _wgrad(dz, x, prec, sc)
    dzb = torch.zeros(S, No + 5, device=DEV)
    dzb[:, 1:No + 1] = dz                                  # base + 4 bytes, row stride No + 5 = 133
    xb = torch.zeros(S * (Ni + 1) + 1, device=DEV)
    xv = xb[1:].view(S, Ni + 1)[:, :Ni]                    # base + 4 bytes, row stride Ni + 1 = 65
    xv.copy_(x)
    for t in (dzb[:, 1:No + 1], xv):
        assert t.data_ptr() % 16 != 0 and t.stride(0) % 4 != 0
    W1, b1 = _wgrad(dzb[:, 1:No + 1], xv, prec, sc)
    assert torch.equal(W1, W) and torch.equal(b1, b)
    W2, b2 = _wgrad(dzb[:, 1:No + 1], x, prec, sc)
    assert torch.equal(W2, W) and torch.equal(b2, b)


def test_wgrad_with_no_samples():
    """S = 0: dW and db are zeroed, with or without a workspace; under accumulate they are left as they were."""
    dz, x = torch.zeros(1, 40, device=DEV), torch.zeros(1, 20, device=DEV)
    for ws in (True, False):
        for prec in ("fp16x3", "bf16x3"):
            W, b = torch.full((40, 20), float("nan"), device=DEV), torch.full((40,), float("nan"), device=DEV)
            _wgrad(dz, x, prec, W=W, b=b, S=0, ws=ws)
            assert bool((W == 0).all()) and bool((b == 0).all()), (ws, prec)
            W, b = torch.randn(40, 20, device=DEV), torch.randn(40, device=DEV)
            W0, b0 = W.clone(), b.clone()
            _wgrad(dz, x, prec, W=W, b=b, S=0, ws=ws, accumulate=1)
            assert torch.equal(W, W0) and torch.equal(b, b0)


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_wgrad_non_finite_values_stay_in_their_row_and_column(prec):
    S, No, Ni = 9000, 160, 33
    dz, x = _data(S, No, Ni, "random", seed=2)
    sc = _scale(dz, prec)
    W, b = _wgrad(dz, x, prec, sc)
    o, i, s = 131, 17, 6001
    dzn = dz.clone()
    dzn[s, o] = float("nan")
    Wn, bn = _wgrad(dzn, x, prec, sc)
    rows = torch.arange(No, device=DEV) != o
    assert bool(Wn[o].isnan().all()) and bool(bn[o].isnan())
    assert torch.equal(Wn[rows], W[rows]) and torch.equal(bn[rows], b[rows])
    xn = x.clone()
    xn[s, i] = float("inf")
    Wn, bn = _wgrad(dz, xn, prec, sc)
    cols = torch.arange(Ni, device=DEV) != i
    assert not bool(torch.isfinite(Wn[:, i]).any())
    assert torch.equal(Wn[:, cols], W[:, cols]) and torch.equal(bn, b)


# ------------------------------------------------------------------------------------------------ pnr_linear
def _linear(x, Wt, N, prec, bias=None, relu=False, transposed=False, scale=None, y=None, S=None):
    """pnr_linear on x [S, K] (a row-strided view as it is) and Wt ([N, K], or [K, N] with transposed); y: output view
    [S, N] (new if None)."""
    S_ = x.shape[0] if S is None else S
    K = x.shape[1]
    y = torch.empty(S_, N, device=DEV) if y is None else y
    L = _capi.lib()
    if "linear" not in _WS:
        _WS["linear"] = torch.empty(int(L.pnr_linear_workspace_bytes(256, 512)), dtype=torch.uint8, device=DEV)
    ws = _WS["linear"]
    rc = L.pnr_linear(x.data_ptr(), max(x.stride(0), K), K, Wt.data_ptr(), max(Wt.stride(0), Wt.shape[1]), int(transposed),
                      _ptr(bias), N, S_, int(relu), _capi.PREC[prec], _ptr(scale), y.data_ptr(), max(y.stride(0), N),
                      ws.data_ptr(), ws.numel(), _capi.stream_ptr())
    _capi.check(rc, "pnr_linear")
    return y


def _ref_linear(x, Wt, transposed, bias):
    W = (Wt.t() if transposed else Wt).double()           # [N, K]
    ref, A, rx = [], [], []
    for c in range(0, x.shape[0], CHUNK):
        a = x[c:c + CHUNK].double()
        r = a @ W.t()
        aa = a.abs()
        m = aa @ W.abs().t()
        if bias is not None:
            r += bias.double()
            m += bias.double().abs()
        ref.append(r), A.append(m), rx.append(aa.sum(1))
    return torch.cat(ref), torch.cat(A), torch.cat(rx), W.abs().sum(1)


def _check_linear(y, x, Wt, prec, bias, relu, transposed, sc, what):
    ref, A, rx, rw = _ref_linear(x, Wt, transposed, bias)
    if relu:
        ref = ref.clamp(min=0)
    K = x.shape[1]
    tau = 3 * U[prec] ** 2 + (3 * -(-K // 16) + 2) * 2.0 ** -23
    floor = 2.0 ** -24 * (rx[:, None] + rw[None, :] / sc) if prec == "fp16x3" else 0.0
    r = _ratio((y.double() - ref).abs(), tau * A + floor)
    _report(what, r)
    return r


LINEAR_SHAPES = [(1, 1), (3, 3), (15, 4), (16, 5), (17, 16), (127, 17), (128, 63), (129, 64), (144, 65), (255, 255),
                 (256, 256), (1, 257), (17, 283), (129, 319), (256, 511), (255, 512), (144, 17), (3, 65)]


def _linear_case(S, K, N, transposed, seed, gscale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(S, K, device=DEV, generator=g) * gscale
    x[:, ::3] = x[:, ::3].relu()                        # mixed signs and exact zeros
    W = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    b = torch.randn(N, device=DEV, generator=g) * 0.1
    return x, (W.t().contiguous() if transposed else W), b


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("N,K", LINEAR_SHAPES)
def test_linear_shapes_and_short_sample_counts(N, K, transposed, prec):
    """Bias or NULL and relu or not alternate over S; the output sits in a NaN-filled buffer whose columns past N and
    rows past S must stay untouched."""
    for j, S in enumerate((1, 63, 64, 65, 127, 128, 129)):
        x, Wt, b = _linear_case(S, K, N, transposed, seed=S + 7 * N + K)
        bias, relu = (b if j % 2 == 0 else None), j % 3 == 1
        buf = torch.full((S + 2, N + 3), float("nan"), device=DEV)
        y = _linear(x, Wt, N, prec, bias=bias, relu=relu, transposed=transposed, y=buf[:S, :N])
        assert bool(buf[:, N:].isnan().all()) and bool(buf[S:].isnan().all()), "written outside y"
        _check_linear(y, x, Wt, prec, bias, relu, transposed, 1.0,
                      f"linear {prec} N={N} K={K} t={transposed} S={S} bias={bias is not None} relu={relu}")


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("N,K", [(256, 256), (144, 283), (17, 65)])
def test_linear_around_the_grid_boundary_and_at_a_training_steps_sample_count(N, K, prec):
    for S in (128 * _sms() - 1, 128 * _sms() + 1, 393216):
        x, Wt, b = _linear_case(S, K, N, 0, seed=S + N)
        y = _linear(x, Wt, N, prec, bias=b, relu=True)
        _check_linear(y, x, Wt, prec, b, True, False, 1.0, f"linear {prec} N={N} K={K} S={S}")


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("N,K", [(128, 283), (256, 17), (45, 65)])
def test_linear_scaled_gradients(N, K, prec):
    """~1e-7 gradients with the power-of-two in_scale, with and without a bias (added after the division by it)."""
    S = 5000
    x, Wt, b = _linear_case(S, K, N, 1, seed=N + K, gscale=3e-7)
    sc = _pow2_scale(x)
    for bias in (None, b * 1e-7):
        y = _linear(x, Wt, N, prec, bias=bias, transposed=True, scale=sc)
        _check_linear(y, x, Wt, prec, bias, False, True, float(sc),
                      f"linear {prec} scaled N={N} K={K} bias={bias is not None}")


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
@pytest.mark.parametrize("K", [256, 283])
def test_linear_misaligned_input_equals_aligned(K, prec):
    """x on the 16-byte load path (aligned base, row stride a multiple of 4 floats and >= K rounded up to 4) and on
    the 4-byte path (base + 4 bytes, row stride K + 2): same bits."""
    S, N = 1000, 129
    x, Wt, b = _linear_case(S, K, N, 0, seed=1)
    xa = torch.zeros(S, (K + 3) // 4 * 4, device=DEV)[:, :K]
    xa.copy_(x)
    assert xa.data_ptr() % 16 == 0 and xa.stride(0) % 4 == 0           # pnr_linear's vec_in conditions
    y = _linear(xa, Wt, N, prec, bias=b)
    buf = torch.zeros(S, K + 2, device=DEV)
    xm = buf[:, 1:K + 1]
    xm.copy_(x)
    assert xm.data_ptr() % 16 != 0 and xm.stride(0) % 4 != 0
    assert torch.equal(_linear(xm, Wt, N, prec, bias=b), y)


def test_linear_with_no_samples_writes_nothing():
    x, Wt, b = _linear_case(4, 64, 32, 0, seed=0)
    y = torch.full((4, 32), float("nan"), device=DEV)
    _linear(x, Wt, 32, "fp16x3", bias=b, y=y, S=0)
    torch.cuda.synchronize()
    assert bool(y.isnan().all())


@pytest.mark.parametrize("prec", ["fp16x3", "bf16x3"])
def test_linear_non_finite_values_stay_in_their_row_and_column(prec):
    S, K, N = 700, 100, 70
    x, Wt, b = _linear_case(S, K, N, 0, seed=3)
    for relu in (False, True):
        y = _linear(x, Wt, N, prec, bias=b, relu=relu)
        xn = x.clone()
        xn[333, 41] = float("nan")
        yn = _linear(xn, Wt, N, prec, bias=b, relu=relu)
        rows = torch.arange(S, device=DEV) != 333
        assert bool(yn[333].isnan().all()), "NaN lost (relu must keep NaN as torch.relu does)"
        assert torch.equal(yn[rows], y[rows])
        Wn = Wt.clone()
        Wn[9, 5] = float("nan")
        yn = _linear(x, Wn, N, prec, bias=b, relu=relu)
        cols = torch.arange(N, device=DEV) != 9
        assert bool(yn[:, 9].isnan().all()) and torch.equal(yn[:, cols], y[:, cols])


# ------------------------------------------------------------------------------------------------ network backward
def _min_preactivation(onet, pts, vd):
    """Smallest |pre-activation| over every ReLU of the float64 oracle network, per sample, on the samples' device
    (test_gpu_backward._min_preactivation, which runs on the CPU)."""
    from oracle import reference_renderer as O
    ex, ed = O.embed(pts, onet.Lx).double(), O.embed(vd, onet.Ld).double()
    m = torch.full((pts.shape[0],), float("inf"), dtype=F64, device=pts.device)
    track = lambda t: torch.minimum(m, t.abs().min(dim=1).values)
    h = ex
    with torch.no_grad():
        for i, lin in enumerate(onet.pts_linears):
            pre = lin(h); m = track(pre); h = torch.relu(pre)
            if i == onet.skip:
                h = torch.cat([ex, h], -1)
        m = track(onet.views_linears[0](torch.cat([onet.feature_linear(h), ed], -1)))
        if onet.C > 0:
            m = track(onet.semantic_linears[0](h))
        if onet.K > 0:
            m = track(onet.instance_linears[0](h))
    return m


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
def test_network_backward_at_a_training_steps_batch(precision):
    """network_backward of cfg3 at 393 216 points (2048 rays x 192 samples: the stash is ~6 GB) against float64
    autograd through the oracle network on the device, every parameter, on samples clear of the ReLU kinks (as
    test_gpu_backward.test_network_backward_every_parameter selects them, at its tolerances)."""
    from panopticnerf_b200 import make_cfg, make_network, synthetic as SY
    from panopticnerf_b200.lib.train import network_backward
    from test_gpu_backward import _oracle_net
    from util import assert_close, rms
    cfg = make_cfg("cfg3", precision=precision)
    net = SY.init_network_weights(make_network(cfg), seed=11)
    onet = _oracle_net(cfg, net).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(1)
    n = 393216
    kink = 1e-4 if precision == "bf16x3" else 3e-5
    pts, vd = [], []
    have = 0
    while have < n:
        p = (torch.rand(n, 3, device=DEV, generator=g) * 2 - 1) * 4
        d = torch.nn.functional.normalize(torch.randn(n, 3, device=DEV, generator=g), dim=-1)
        keep = torch.cat([_min_preactivation(onet, p[c:c + 65536].double(), d[c:c + 65536].double()) >= kink
                          for c in range(0, n, 65536)])
        pts.append(p[keep]), vd.append(d[keep])
        have += int(keep.sum())
    pts, vd = torch.cat(pts)[:n].contiguous(), torch.cat(vd)[:n].contiguous()
    d_raw = torch.randn(n, 4 + cfg.num_classes + cfg.num_instances, device=DEV, generator=g)
    net = net.to(DEV)
    got = network_backward(net, d_raw, pts=pts, viewdirs=vd)
    assert net.range_status() == 0
    for c in range(0, n, 65536):                          # float64 autograd in chunks; .grad accumulates
        onet(pts[c:c + 65536].double(), vd[c:c + 65536].double()).backward(d_raw[c:c + 65536].double())
    tol = 2e-4 if precision == "bf16x3" else 1e-4
    for name, p in onet.named_parameters():
        e = assert_close(got[name].double(), p.grad, rms(p.grad), f"cfg3 {precision} S={n} d/d{name}", rel=tol)
        print(f"cfg3 {precision} S={n} d/d{name}: largest error / bound = {e / tol:.3e}")
    del got, onet
    torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
def test_stash_maxima_at_a_training_steps_batch(precision):
    """The maxima pnr_mlp_backward_trunk reports for each stash slot of cfg3 at 393 216 points (the ~6 GB stash the
    weight gradients are computed on), bit for bit against the stash they describe."""
    from panopticnerf_b200 import make_cfg, make_network, synthetic as SY
    cfg = make_cfg("cfg3", precision=precision)
    net = SY.init_network_weights(make_network(cfg), seed=11).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(2)
    n = 393216
    pts = (torch.rand(n, 3, device=DEV, generator=g) * 2 - 1) * 4
    grad_h = torch.randn(n, cfg.W, device=DEV, generator=g) * 1e-6
    gs = 2.0 ** 20
    _, stash, mx = net.backward_trunk(grad_h, pts=pts, stash=True, absmax=True, grad_scale=gs)
    assert net.range_status() == 0
    half = torch.float16 if precision.startswith("fp16") else torch.bfloat16
    scale = torch.ones(2 * cfg.D - 1, device=DEV)
    scale[cfg.D - 1:] = gs
    want = (torch.linalg.vector_norm(stash, ord=float("inf"), dim=(1, 2)) * scale).to(half).float() / scale
    assert mx.shape == want.shape and torch.equal(mx, want), (mx, want)
    del stash
    torch.cuda.empty_cache()
