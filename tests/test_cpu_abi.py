"""CPU: the C-ABI library builds (cross-compiled for sm_90a), loads, and exports every symbol that
include/pnr.h declares; the ctypes table mirrors the header; the product refuses CPU tensors loudly.
No compute call is made (there is no GPU here)."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


def header_functions():
    txt = (ROOT / "include" / "pnr.h").read_text()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(pnr_[a-z_0-9]+)\s*\(", txt)))


def test_build_and_symbols():
    import __graft_entry__ as g
    g.build()
    from panopticnerf_b200 import _capi
    lib = C.CDLL(str(ROOT / "panopticnerf_b200" / "libpnr.so"))
    names = header_functions()
    assert len(names) >= 16
    for n in names:
        assert hasattr(lib, n), f"libpnr.so does not export {n} declared in include/pnr.h"
    assert sorted(_capi.SIGNATURES) == names, "ctypes table and include/pnr.h disagree"
    assert _capi.lib().pnr_version() == 100


def test_ctypes_argument_counts_match_header():
    """Every prototype in include/pnr.h has as many parameters as its ctypes signature (a mismatch would corrupt
    the call stack silently)."""
    from panopticnerf_b200 import _capi
    txt = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "pnr.h").read_text(), flags=re.S)
    protos = dict(re.findall(r"\b(pnr_[a-z_0-9]+)\s*\(([^;{]*?)\)\s*;", txt, flags=re.S))
    assert set(protos) == set(_capi.SIGNATURES)
    for name, args in protos.items():
        args = " ".join(args.split())
        n = 0 if args in ("", "void") else args.count(",") + 1
        assert n == len(_capi.SIGNATURES[name][1]), f"{name}: header has {n} parameters, ctypes {len(_capi.SIGNATURES[name][1])}"


def test_sass_is_hopper_native():
    """cuobjdump evidence: wgmma -> HGMMA (fp16 and bf16 operands), bulk TMA -> UBLKCP, mbarrier waits -> SYNCS;
    and only sm_90a code is embedded."""
    import subprocess
    so = ROOT / "panopticnerf_b200" / "libpnr.so"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert not re.search(r"arch = sm_(?!90a)", sass)
    for mnem in ("HGMMA.64x128x16.F32 ", "HGMMA.64x128x16.F32.BF16", "UBLKCP", "SYNCS"):
        assert mnem in sass, mnem


def test_product_has_no_cpu_path():
    import panopticnerf_b200 as PN
    from panopticnerf_b200 import synthetic as S
    cfg = PN.make_cfg("cfg1")
    net = PN.make_network(cfg)
    ren = PN.make_renderer(cfg, net)
    with pytest.raises(Exception, match="CUDA|GPU|CPU"):
        net(torch.zeros(4, 3), torch.zeros(4, 3))
    with pytest.raises(Exception, match="CUDA|GPU|CPU"):
        ren.render(S.make_batch(cfg, rows=1))


def test_product_does_not_import_oracle():
    for py in (ROOT / "panopticnerf_b200").rglob("*.py"):
        assert "oracle" not in py.read_text().replace("the oracle", "").replace("oracle's", "").replace(
            "oracle restatement", "").replace("oracle/reference_renderer.py", ""), py


def test_state_dict_is_drop_in():
    import panopticnerf_b200 as PN
    from oracle import reference_renderer as O
    for preset in ("cfg1", "cfg2", "cfg3"):
        cfg = PN.make_cfg(preset)
        a, b = PN.make_network(cfg), O.make_network(cfg)
        assert [(k, tuple(v.shape)) for k, v in a.state_dict().items()] == \
               [(k, tuple(v.shape)) for k, v in b.state_dict().items()]
        a.load_state_dict(b.state_dict())
        assert 2 * sum(p.numel() for n, p in a.named_parameters() if n.endswith("weight")) == O.mlp_flops_per_sample(cfg)


def test_network_copies_do_not_share_the_native_handle(tmp_path):
    """The libpnr context is a raw pointer owned by one Network object: deepcopy (EMA weights), pickle / torch.save
    of the module and DataParallel-style replicas must start WITHOUT it, or the copy's release() / __del__ would
    destroy the context the original still uses (ADVICE r1: use-after-free / double free)."""
    import copy
    import pickle
    import panopticnerf_b200 as PN
    net = PN.make_network(PN.make_cfg("cfg1"))
    net._ctx, net._ctx_key = 0xDEAD0000, ("cuda:0", "fp16x3")   # pretend a context exists (never dereferenced here)
    try:
        dup = copy.deepcopy(net)
        assert dup._ctx is None and dup._ctx_key is None and net._ctx == 0xDEAD0000
        assert all(torch.equal(a, b) and a.data_ptr() != b.data_ptr()
                   for a, b in zip(net.state_dict().values(), dup.state_dict().values()))
        back = pickle.loads(pickle.dumps(net))
        assert back._ctx is None and back._ctx_key is None
        torch.save(net, tmp_path / "net.pt")
        loaded = torch.load(tmp_path / "net.pt", weights_only=False)
        assert loaded._ctx is None
        rep = net._replicate_for_data_parallel()
        assert rep._ctx is None and net._ctx == 0xDEAD0000
    finally:
        net._ctx, net._ctx_key = None, None                      # nothing to destroy


def test_renderer_rejects_too_many_samples_up_front():
    import panopticnerf_b200 as PN
    cfg = PN.make_cfg("cfg2", N_samples=192, N_importance=128)
    with pytest.raises(ValueError, match="samples"):
        PN.make_renderer(cfg, PN.make_network(cfg))
