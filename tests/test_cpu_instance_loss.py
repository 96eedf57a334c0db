"""CPU tier of the instance term of `pnr_losses` (DESIGN 3.4): the float64 oracle on rays whose answer is known in
closed form, the argument checks of the new fields (refused with PNR_ERR_ARG before any CUDA call: the pointers are
placeholders that are never dereferenced) and the ctypes layout of pnr_loss_args against the header."""
import ctypes as C
import math
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_instance as OI
from panopticnerf_b200 import _capi

ROOT = Path(__file__).resolve().parent.parent
X = 64          # a non-null placeholder pointer
ERR_ARG = -1


@pytest.mark.parametrize("K", [1, 2, 7, 64, 1000])
def test_uniform_logits_give_log_k(K):
    im = torch.full((3, K), 2.5, dtype=torch.float64)
    fim = torch.zeros(3, K, dtype=torch.float64)
    fim[:, K - 1] = 0.9
    mean, per_ray, label, n = OI.instance_loss(im, fim, 0.5)
    assert n == 3 and label.tolist() == [K - 1] * 3
    assert torch.allclose(per_ray, torch.full((3,), math.log(K), dtype=torch.float64), rtol=0, atol=1e-12)
    assert float(mean) == pytest.approx(math.log(K), abs=1e-12)


def test_a_tie_in_the_fixed_map_picks_the_lowest_slot():
    fim = torch.tensor([[0.0, 0.5, 0.2, 0.5], [0.3, 0.3, 0.3, 0.1], [0.6, 0.0, 0.0, 0.6]], dtype=torch.float64)
    assert OI.instance_labels(fim, 0.25).tolist() == [1, 0, 0]


def test_the_threshold_counts_at_equality_and_not_one_ulp_below():
    thr = np.float32(0.5)
    below = float(np.nextafter(thr, np.float32(0)))
    fim = torch.tensor([[float(thr), 0.1], [0.1, below]], dtype=torch.float32).double()
    assert OI.instance_labels(fim, float(thr)).tolist() == [0, -1]
    im = torch.tensor([[3.0, -1.0], [0.0, 9.0]], dtype=torch.float64, requires_grad=True)
    mean, per_ray, _, n = OI.instance_loss(im, fim, float(thr))
    mean.backward()
    assert n == 1 and float(per_ray.detach()[1]) == 0.0 and float(im.grad[1].abs().sum()) == 0.0
    p = torch.softmax(im.detach()[0], 0)
    assert torch.allclose(im.grad[0], p - torch.tensor([1.0, 0.0], dtype=torch.float64))


def test_rays_without_primitives_and_nan_rows_are_ignored():
    fim = torch.tensor([[0.0, 0.0, 0.0], [0.2, float("nan"), 0.9], [0.0, 0.8, 0.1]], dtype=torch.float64)
    im = torch.randn(3, 3, dtype=torch.float64)
    mean, per_ray, label, n = OI.instance_loss(im, fim, 0.5)
    assert label.tolist() == [-1, -1, 1] and n == 1
    assert float(mean) == pytest.approx(float(torch.logsumexp(im[2], 0) - im[2, 1]), abs=1e-12)
    assert per_ray[:2].tolist() == [0.0, 0.0]


def _refused(rc, needle):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg, msg


def _inst_args(**kw):
    a = _capi.PnrLossArgs()
    a.R, a.C, a.eps = 4, 0, 1e-6
    a.K, a.instance_map, a.fixed_instance_map, a.inst_label, a.n_inst = 3, X, X, X, X
    a.w_inst, a.inst_min_weight = 1.0, 0.5
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,needle", [
    ({"K": 0}, "K=0"), ({"K": 32768}, "K=32768"), ({"K": -1}, "K=-1"),
    ({"fixed_instance_map": None}, "fixed_instance_map"), ({"inst_label": None}, "inst_label"),
    ({"n_inst": None}, "n_inst"), ({"inst_min_weight": 0.0}, "inst_min_weight"),
    ({"inst_min_weight": float(np.nextafter(np.float32(1), np.float32(2)))}, "inst_min_weight"),
    ({"inst_min_weight": -0.5}, "inst_min_weight"), ({"inst_min_weight": float("nan")}, "inst_min_weight")])
def test_losses_refuse_bad_instance_arguments(kw, needle):
    _refused(_capi.lib().pnr_losses(C.byref(_inst_args(**kw)), None), needle)


def test_pnr_loss_args_ctypes_layout_matches_the_header(tmp_path):
    """Offsets of every pnr_loss_args field (the ctypes mirror vs offsetof in a host program built against
    include/pnr.h)."""
    if not shutil.which("g++"):
        pytest.skip("no host compiler")
    fields = [f for f, _ in _capi.PnrLossArgs._fields_]
    src = tmp_path / "offsets.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(pnr_loss_args, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(pnr_loss_args));\n  return 0;\n}\n')
    exe = tmp_path / "offsets"
    subprocess.check_call(["g++", "-x", "c++", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got[:-1] == [getattr(_capi.PnrLossArgs, f).offset for f in fields]
    assert got[-1] == C.sizeof(_capi.PnrLossArgs)
