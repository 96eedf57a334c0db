"""The first value outside every range a sampling, compositing, loss, label or encoder entry point accepts is refused
with PNR_ERR_ARG and an error that names it.  The checks run before any CUDA call, so this needs no GPU: the pointers
passed are placeholders that are never dereferenced.  tests/test_gpu_stage_limits.py runs the same entry points at
the last accepted values."""
import ctypes as C

import pytest

from panopticnerf_b200 import _capi

X = 64          # a non-null placeholder pointer (never dereferenced: the argument checks refuse first)
ERR_ARG = -1


def _refused(rc, needle):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg, msg


def _composite(R=4, N=64, C_=3, K=2):
    out = _capi.PnrCompositeOut(rgb_map=X)
    return _capi.lib().pnr_composite(X, X, X, R, N, C_, K, 0, 0, 0, None, None, None, 0, C.byref(out), None)


def _composite_backward(R=4, N=64, C_=3, K=2):
    g = _capi.PnrCompositeGrads(rgb_map=X)
    return _capi.lib().pnr_composite_backward(X, X, X, R, N, C_, K, 0, 0, 0, None, None, None, 0, C.byref(g), X, None)


@pytest.mark.parametrize("fn", [_composite, _composite_backward])
@pytest.mark.parametrize("kw,needle", [({"N": 257}, "N=257"), ({"N": 0}, "N=0"), ({"C_": 129}, "C=129"),
                                       ({"K": 129}, "K=129"), ({"C_": -1}, "C=-1"), ({"R": -1}, "R=-1")])
def test_composite_refuses_out_of_range(fn, kw, needle):
    _refused(fn(**kw), needle)


def test_composite_backward_refuses_softmax():
    g = _capi.PnrCompositeGrads(rgb_map=X)
    rc = _capi.lib().pnr_composite_backward(X, X, X, 4, 64, 3, 0, 0, 1, 0, None, None, None, 0, C.byref(g), X, None)
    assert rc == -4 and b"softmax" in _capi.lib().pnr_last_error()


@pytest.mark.parametrize("N,Ni,needle", [(2, 8, "N=2"), (257, 8, "N=257"), (256, 257, "N+Ni=513"), (3, 510, "N+Ni=513"),
                                         (64, 0, "Ni=0")])
def test_sample_pdf_refuses_out_of_range(N, Ni, needle):
    _refused(_capi.lib().pnr_sample_pdf(X, X, 4, N, Ni, X, X, None, X, None), needle)


@pytest.mark.parametrize("N,M,needle", [(257, 4, "N=257"), (0, 4, "N=0"), (64, 9, "M=9"), (64, 0, "M=0")])
def test_sample_intervals_refuses_out_of_range(N, M, needle):
    _refused(_capi.lib().pnr_sample_intervals(X, X, X, None, 4, N, 0.0, X, X, X, M, X, X, None), needle)


@pytest.mark.parametrize("N,M,needle", [(0, 4, "N < 1"), (64, 9, "M=9"), (64, 0, "M=0")])
def test_sample_stratified_refuses_out_of_range(N, M, needle):
    _refused(_capi.lib().pnr_sample_stratified(X, X, X, None, 4, N, 0.0, X, X, X, M, X, X, None), needle)


@pytest.mark.parametrize("R,N,M,needle", [(4, 0, 4, "N=0"), (4, -3, 4, "N=-3"), (-1, 8, 4, "R=-1"), (4, 8, 9, "M=9"),
                                          (4, 8, 0, "M=0")])
def test_tag_samples_refuses_out_of_range(R, N, M, needle):
    _refused(_capi.lib().pnr_tag_samples(X, R, N, X, X, X, M, X, None), needle)


@pytest.mark.parametrize("B,M,needle", [(4, 9, "M=9"), (4, 0, "M=0"), (-1, 4, "B=-1")])
def test_intersect_refuses_out_of_range(B, M, needle):
    _refused(_capi.lib().pnr_intersect(X, 4, X, X, X, B, M, X, X, X, X, None), needle)


@pytest.mark.parametrize("M", [0, 9])
def test_bound_by_primitives_refuses_out_of_range(M):
    _refused(_capi.lib().pnr_bound_by_primitives(X, X, X, X, 4, M, X, X, None), f"M={M}")


@pytest.mark.parametrize("L", [17, -1])
def test_encode_refuses_out_of_range(L):
    _refused(_capi.lib().pnr_encode(X, 4, L, X, None), f"L={L}")


@pytest.mark.parametrize("name", ["pnr_hashgrid_encode", "pnr_hashgrid_backward"])
@pytest.mark.parametrize("L,F,T,base,scale,needle", [
    (4, 2, 29, 16.0, 1.5, "T_log2=29"), (4, 2, 3, 16.0, 1.5, "T_log2=3"), (33, 2, 19, 16.0, 1.1, "L=33"),
    (0, 2, 19, 16.0, 1.5, "L=0"), (4, 3, 19, 16.0, 1.5, "F=3"), (4, 16, 19, 16.0, 1.5, "F=16"),
    (1, 2, 19, 1048576.0, 1.0, "finest resolution 1048576"), (2, 2, 19, 524288.0, 2.0, "finest resolution 1048576"),
    (4, 2, 19, 0.5, 1.5, "base_resolution")])
def test_hashgrid_refuses_out_of_range(name, L, F, T, base, scale, needle):
    _refused(getattr(_capi.lib(), name)(X, 4, None, X, L, F, T, base, scale, X, None), needle)


def _loss_args(**kw):
    a = _capi.PnrLossArgs()
    a.R, a.C, a.eps = 4, 3, 1e-6
    a.semantic_map, a.label, a.per_ray = X, X, X
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,needle", [({"C": 32768}, "bad sizes"), ({"C": -1}, "bad sizes"), ({"R": -1}, "bad sizes"),
                                       ({"eps": 0.0}, "eps"), ({"C": 0}, "C > 0")])
def test_losses_refuse_out_of_range(kw, needle):
    _refused(_capi.lib().pnr_losses(C.byref(_loss_args(**kw)), None), needle)


@pytest.mark.parametrize("C_,K,R", [(32768, 4, 4), (4, 32768, 4), (-1, 4, 4), (4, 4, -1)])
def test_label_tiles_refuse_out_of_range(C_, K, R):
    _refused(_capi.lib().pnr_label_tiles(X, X, X, X, R, C_, K, X, X, X, X, None), "bad sizes")


@pytest.mark.parametrize("C_,K,R", [(32768, 4, 4), (0, 4, 4), (4, 32768, 4), (4, -1, 4), (4, 4, -1)])
def test_panoptic_fuse_refuses_out_of_range(C_, K, R):
    _refused(_capi.lib().pnr_panoptic_fuse(X, X, R, C_, K, X, X, None, None, None, X, None, None, None, None),
             "bad sizes")
