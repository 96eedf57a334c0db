"""CPU tier of the fixed-point hash-grid table gradient (pnr_hashgrid_backward_fixed, rule in include/pnr.h): the oracle
(tests/oracle_hashgrid_fixed.py) on known answers, the overflow bound at its worst case and the NaN confinement rule;
the entry point's argument checks, which run before any CUDA call (the pointers passed are placeholders that are
never dereferenced); the workspace size against its documented layout; cfg.hash_grad."""
import numpy as np
import pytest
import torch

from oracle import reference_panoptic as OP
from oracle_hashgrid_fixed import (F32, ceil_log2, corners, forward_from_corners, frexp_exponent, level_scale,
                                   table_grad_fixed)
from panopticnerf_b200 import _capi

X = 64          # a non-null, 16-byte aligned placeholder pointer (never dereferenced: the argument checks refuse first)
ERR_ARG = -1


# ------------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("L,F,T_log2,base,scale", [(8, 2, 12, 4.0, 2.0), (6, 4, 10, 3.0, 1.9), (3, 1, 4, 2.0, 1.5)])
def test_corners_recompose_the_reference_encoder(L, F, T_log2, base, scale):
    """The oracle's corner weights and rows are the encoder's: summed against a table in the forward's order they give
    oracle/reference_panoptic.hashgrid_encode bit for bit (dense and hashed levels, points outside the box)."""
    g = torch.Generator().manual_seed(L * 10 + F)
    aabb = torch.tensor([[-1.0, -2.0, -1.0], [1.0, 2.0, 3.0]])
    x = torch.rand(700, 3, generator=g) * torch.tensor([2.4, 4.8, 4.8]) + torch.tensor([-1.2, -2.4, -1.4])
    table = torch.randn(L, 1 << T_log2, F, generator=g)
    cs = corners(x, aabb, L, 1 << T_log2, base, scale)
    assert torch.equal(forward_from_corners(cs, table), OP.hashgrid_encode(x, aabb, table, base, scale))


def test_corner_weights_sum_to_at_most_one_plus_2_pow_minus_20():
    g = torch.Generator().manual_seed(3)
    x = torch.rand(100_000, 3, generator=g)
    for w, _ in corners(x, None, 16, 1 << 19, 16.0, 1.3819):
        assert float(w.astype(np.float64).sum(1).max()) <= 1 + 2.0 ** -20


@pytest.mark.parametrize("n,clog", [(1, 0), (2, 1), (3, 2), (4, 2), (255, 8), (256, 8), (257, 9), (2 ** 19 - 1, 19),
                                    (2 ** 19, 19), (2 ** 19 + 1, 20), (2 ** 40 + 1, 41)])
def test_scale_follows_ceil_log2_n(n, clog):
    assert ceil_log2(n) == clog
    assert level_scale(1.0, n) == 60 - clog                      # 1.0 = 0.5 * 2^1
    assert level_scale(0.0, n) is None


@pytest.mark.parametrize("m,e", [(1.0, 1), (0.5, 0), (2.0 ** -10, -9), (2.0 ** 100, 101), (float(np.nextafter(F32(1), F32(0))), 0),
                                 (2.0 ** -149, -148), (2.0 ** -126, -125), (float(np.finfo(F32).max), 128)])
def test_frexp_exponent_at_powers_of_two_and_the_ends_of_fp32(m, e):
    assert frexp_exponent(m) == e
    assert level_scale(m, 1) == 61 - e


def _dense_index(c, res):
    r1 = res + 1
    return c[0] + c[1] * r1 + c[2] * r1 * r1


def test_cell_centre_points_give_exact_eighths():
    """L = 1, res = 4 (dense in a table of 128 rows): points at the centre of cell (1, 1, 1) have w_k = 1/8 at all 8
    corners, so every q is exact and each corner entry receives exactly fp32(sum(g) / 8)."""
    x = np.full((3, 3), 1.5 / 4, F32)
    g = np.array([[1.0], [-0.75], [0.3]], F32)
    stats = {}
    got = table_grad_fixed(x, None, g, 1, 1, 7, 4.0, 2.0, stats=stats)
    w, _ = corners(x, None, 1, 128, 4.0, 2.0)[0]
    assert (w == F32(0.125)).all()
    assert stats[0]["m"] == 1.0 and stats[0]["s"] == 61 - 2 - 1
    want = F32((1.0 - 0.75 + float(F32(0.3))) / 8)                 # the exact sum, rounded once
    rows = [_dense_index((1 + (k & 1), 1 + (k >> 1 & 1), 1 + (k >> 2)), 4) for k in range(8)]
    assert (got[0, rows, 0] == want).all()
    assert np.count_nonzero(got) == 8
    # accumulation: one fp32 add onto what grad_table held
    base = np.arange(128, dtype=F32).reshape(1, 128, 1) * F32(0.1)
    acc = table_grad_fixed(x, None, g, 1, 1, 7, 4.0, 2.0, grad_table=base)
    assert np.array_equal(acc, (base + got).astype(F32))


@pytest.mark.parametrize("k", [0, 1, 12])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_overflow_bound_at_its_worst_case(k, sign):
    """n = 2^k points on one grid vertex (w = 1 on one corner) with g = +-m_l, m_l just below a power of two: the worst
    case of the bound, sum |q| = n * round(m_l 2^s_l) -> 2^61.  It stays below 2^61 (1 + 2^-20) + 4n < 2^63.  The
    rule keeps two spare bits: two more units of scale still fit, three overflow."""
    n = 2 ** k
    m = np.nextafter(F32(1), F32(0))
    stats = {}
    x = np.zeros((n, 3), F32)
    table_grad_fixed(x, None, np.full((n, 1), sign * m, F32), 1, 1, 4, 2.0, 1.5, stats=stats)
    s, total = stats[0]["s"], stats[0]["abs_sum"]
    assert s == 61 - k
    q = int(np.rint(float(m) * 2.0 ** s))
    assert total == n * q == 2 ** 61 - 2 ** 37
    assert int(stats[0]["acc"][0, 0]) == int(sign) * total
    assert total < 2 ** 61 * (1 + 2.0 ** -20) + 4 * n < 2 ** 63
    assert 4 * total < 2 ** 63 <= 8 * total


def test_non_finite_gradients_poison_their_corners_only():
    """Two points in cells that share no corner (L = 1, res = 4, F = 2).  Point 0: g = (NaN, 1); point 1: g = (+Inf, -2).
    Feature 0 of both points' 8 corners is NaN; feature 1 is the rule over the finite values (m = 2, left out: NaN /
    Inf); every other entry is 0.  A level whose finite values are all 0 adds nothing but still marks its NaNs."""
    x = np.array([[1.5 / 4] * 3, [3.5 / 4] * 3], F32)
    g = np.array([[np.nan, 1.0], [np.inf, -2.0]], F32)
    stats = {}
    got = table_grad_fixed(x, None, g, 1, 2, 7, 4.0, 2.0, stats=stats)
    assert stats[0]["m"] == 2.0
    r0 = [_dense_index((1 + (k & 1), 1 + (k >> 1 & 1), 1 + (k >> 2)), 4) for k in range(8)]
    r1 = [_dense_index((3 + (k & 1), 3 + (k >> 1 & 1), 3 + (k >> 2)), 4) for k in range(8)]
    assert np.isnan(got[0, r0 + r1, 0]).all() and np.isnan(got).sum() == 16
    assert (got[0, r0, 1] == F32(0.125)).all() and (got[0, r1, 1] == F32(-0.25)).all()
    others = np.ones(got.shape[1], bool)
    others[r0 + r1] = False
    assert (got[0, others] == 0).all()
    # every finite gradient zero: m = 0, nothing is added (grad_table keeps its values), the NaNs are still marked
    base = np.full((1, 128, 2), -0.0, F32)
    z = table_grad_fixed(x, None, np.array([[np.nan, 0.0], [0.0, -0.0]], F32), 1, 2, 7, 4.0, 2.0, grad_table=base)
    assert np.isnan(z[0, r0, 0]).all() and np.isnan(z).sum() == 8
    fin = ~np.isnan(z)
    assert (z[fin] == 0).all() and np.signbit(z[fin]).all()


# ------------------------------------------------------------------------------------------------ the entry points
def _refused(rc, needle):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg, msg


def _layout_bytes(L, F, T_log2):
    entries = L * F << T_log2
    r16 = lambda b: (b + 15) // 16 * 16
    return r16(8 * entries + r16((entries + 31) // 32 * 4) + 8 * L + 8)


def _fixed(n=100, x=X, grad_out=X, grad_table=X, L=16, F=2, T_log2=19, base=16.0, scale=1.3819, ws=X, ws_bytes=None):
    Lib = _capi.lib()
    need = Lib.pnr_hashgrid_fixed_workspace_bytes(max(min(L, 32), 1), F if F in (1, 2, 4, 8) else 2, max(min(T_log2, 28), 4))
    return Lib.pnr_hashgrid_backward_fixed(x, n, None, grad_out, L, F, T_log2, base, scale, grad_table, ws,
                                           need if ws_bytes is None else ws_bytes, None)


@pytest.mark.parametrize("L,F,T_log2", [(16, 2, 19), (1, 1, 4), (32, 8, 4), (3, 4, 10), (32, 8, 28), (5, 1, 7)])
def test_workspace_bytes_follow_the_documented_layout(L, F, T_log2):
    assert _capi.lib().pnr_hashgrid_fixed_workspace_bytes(L, F, T_log2) == _layout_bytes(L, F, T_log2)


@pytest.mark.parametrize("L,F,T_log2", [(0, 2, 19), (33, 2, 19), (16, 3, 19), (16, 0, 19), (16, 2, 3), (16, 2, 29)])
def test_workspace_bytes_are_zero_for_a_refused_shape(L, F, T_log2):
    assert _capi.lib().pnr_hashgrid_fixed_workspace_bytes(L, F, T_log2) == 0


@pytest.mark.parametrize("kw,needle", [
    ({"L": 0}, "L=0"), ({"L": 33}, "L=33"), ({"F": 3}, "F=3"), ({"F": 0}, "F=0"),
    ({"T_log2": 3}, "T_log2=3"), ({"T_log2": 29}, "T_log2=29"),
    ({"base": 0.5}, "base_resolution"), ({"scale": 0.99}, "per_level_scale"),
    ({"L": 17, "base": 16.0, "scale": 2.0}, "finest resolution 1048576"),
    ({"x": None}, "x is null"), ({"grad_out": None}, "grad_out is null"), ({"grad_table": None}, "grad_table is null"),
    ({"n": -1}, "n=-1"),
    ({"ws": None}, "workspace of"), ({"ws": X + 8}, "16-byte aligned")])
def test_fixed_refuses_each_argument_by_name(kw, needle):
    _refused(_fixed(**kw), needle)
    assert b"pnr_hashgrid_backward_fixed" in _capi.lib().pnr_last_error()


@pytest.mark.parametrize("L,F,T_log2", [(16, 2, 19), (1, 1, 4), (32, 8, 10)])
def test_fixed_refuses_a_workspace_one_byte_short(L, F, T_log2):
    need = _capi.lib().pnr_hashgrid_fixed_workspace_bytes(L, F, T_log2)
    _refused(_fixed(L=L, F=F, T_log2=T_log2, base=2.0, scale=1.2, ws_bytes=need - 1), f"{need - 1} bytes, {need} needed")


def test_fixed_with_no_points_returns_before_the_device():
    assert _fixed(n=0, x=None, ws=None) == 0


# ------------------------------------------------------------------------------------------------ cfg.hash_grad
def test_cfg_hash_grad_selects_the_path_and_refuses_other_values():
    import panopticnerf_b200 as PN
    from oracle_hashgrid import hash_cfg
    from panopticnerf_b200.lib.networks.encoding import HashGrid
    assert PN.make_network(hash_cfg("cfg1", hash_log2_size=10)).xyz_encoder.grad == "atomic"
    assert PN.make_network(hash_cfg("cfg1", hash_log2_size=10, hash_grad="fixed")).xyz_encoder.grad == "fixed"
    with pytest.raises(ValueError, match="cfg.hash_grad='deterministic'"):
        PN.make_network(hash_cfg("cfg1", hash_log2_size=10, hash_grad="deterministic"))
    with pytest.raises(ValueError, match="grad='Fixed'"):
        HashGrid(4, 2, 10, grad="Fixed")
