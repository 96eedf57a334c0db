"""The first value outside every range the training path's GEMMs accept (pnr_linear, pnr_wgrad) is refused with
PNR_ERR_ARG and an error that names it.  These checks run before any CUDA call, so this needs no GPU: the pointers
passed are placeholders that are never dereferenced.  tests/test_gpu_train_limits.py runs both kernels at the last
accepted values."""
import pytest

from panopticnerf_b200 import _capi

X = 64          # a non-null, 16-byte aligned placeholder pointer (never dereferenced: the argument checks refuse first)
ERR_ARG = -1
FP16X3 = _capi.PREC["fp16x3"]


def _refused(rc, needle):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg, msg


def _linear(N=256, K=512, S=10, ld_x=None, ld_w=None, ld_y=None, transposed=0, ws=X, ws_bytes=None):
    L = _capi.lib()
    need = L.pnr_linear_workspace_bytes(max(min(N, 256), 1), max(min(K, 512), 1))
    return L.pnr_linear(X, K if ld_x is None else ld_x, K, X, (N if transposed else K) if ld_w is None else ld_w,
                        transposed, None, N, S, 0, FP16X3, None, X, N if ld_y is None else ld_y, ws,
                        need if ws_bytes is None else ws_bytes, None)


def _wgrad(No=256, Ni=256, S=10, ld_dz=None, ld_x=None, ld_w=None):
    return _capi.lib().pnr_wgrad(X, No if ld_dz is None else ld_dz, No, X, Ni if ld_x is None else ld_x, Ni, S, FP16X3, None,
                                 X, Ni if ld_w is None else ld_w, X, 0, X, 1 << 30, None)


@pytest.mark.parametrize("kw,needle", [({"N": 0}, "N = 0"), ({"N": 257}, "N = 257"), ({"K": 0}, "K = 0"), ({"K": 513}, "K = 513"),
                                       ({"S": -1}, "S = -1"),
                                       ({"ld_x": 511}, "ld_x = 511 < K = 512"), ({"ld_y": 255}, "ld_y = 255 < N = 256"),
                                       ({"ld_w": 511}, "ld_w = 511 < K = 512"),
                                       ({"transposed": 1, "ld_w": 255}, "ld_w = 255 < N = 256")])
def test_linear_refuses_out_of_range(kw, needle):
    _refused(_linear(**kw), needle)


@pytest.mark.parametrize("N,K", [(256, 512), (1, 1), (17, 65)])
def test_linear_refuses_a_short_or_misaligned_workspace(N, K):
    need = _capi.lib().pnr_linear_workspace_bytes(N, K)
    assert need > 0
    _refused(_linear(N=N, K=K, ws_bytes=need - 1), "workspace of")
    _refused(_linear(N=N, K=K, ws=X + 8), "16-byte aligned")
    _refused(_linear(N=N, K=K, ws=None), "workspace of")


def test_linear_accepts_the_last_values_up_to_the_device():
    """The same call at the range's edges passes every argument check; S = 0 returns before touching the device."""
    assert _linear(N=256, K=512, S=0) == 0
    assert _linear(N=1, K=1, S=0) == 0
    assert _linear(N=256, K=512, S=0, transposed=1) == 0


@pytest.mark.parametrize("kw,needle", [({"No": 0}, "No = 0"), ({"No": 257}, "No = 257"), ({"Ni": 0}, "Ni = 0"),
                                       ({"Ni": 257}, "Ni = 257"), ({"S": -1}, "S = -1"),
                                       ({"ld_dz": 255}, "ld_dz = 255 < No = 256"), ({"ld_x": 255}, "ld_x = 255 < Ni = 256"),
                                       ({"ld_w": 255}, "ld_w = 255 < Ni = 256"),
                                       ({"No": 17, "Ni": 3, "ld_x": 2}, "ld_x = 2 < Ni = 3")])
def test_wgrad_refuses_out_of_range(kw, needle):
    _refused(_wgrad(**kw), needle)
