"""CPU tier of the 128-row fused MLP kernel (mlp_rows128_kernel): its shared-memory map (csrc/mlp_program.h, compiled
for the host) and the rule that routes a forward program to it (mlp_rows128_ok, through pnr_program_tile_rows), for the
configuration space pnr_create accepts: a 256-wide network without heads runs 128-sample tiles, in every precision and
with either trunk input; any head, a narrower trunk or a backward program keeps the 64-sample tiles."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest

import test_cpu_hashgrid_network as H
from oracle_hashgrid import hash_cfg
from panopticnerf_b200 import _capi, make_cfg, make_network, synthetic as S
from test_cpu_config_space import FORWARD, GRID_MODES, GRID_SHAPES, GRIDS, _id
from test_cpu_program import PROGRAM_BACKWARD, MlpProgram, build

CSRC = Path(__file__).resolve().parent.parent / "panopticnerf_b200" / "csrc"
SMEM_LIMIT = 232448   # 227 KB of dynamic shared memory per CTA on sm_90


def _tile_rows(prog):
    rows = C.c_int32()
    _capi.check(_capi.lib().pnr_program_tile_rows(C.byref(prog), C.sizeof(MlpProgram), C.byref(rows)),
                "pnr_program_tile_rows")
    return rows.value


def _expect(cfg):
    return 128 if cfg.W == 256 and cfg.num_classes == 0 and cfg.num_instances == 0 else 64


@pytest.mark.parametrize("over", FORWARD, ids=[_id(o) for o in FORWARD])
def test_routing_over_the_accepted_configurations(over):
    cfg = make_cfg("cfg2", **over)
    net = S.init_network_weights(make_network(cfg), seed=0)
    prog, _, _ = build(cfg, net)
    assert _tile_rows(prog) == _expect(cfg), over
    if cfg.precision.endswith("x3") and cfg.D <= 9:
        bprog, _, _ = build(cfg, net, flags=PROGRAM_BACKWARD)
        assert _tile_rows(bprog) == 64, over


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3", "fp16", "bf16"])
@pytest.mark.parametrize("over", [dict(), dict(D=3), dict(D=16), dict(xyz_res=0), dict(view_res=0),
                                  dict(num_classes=1), dict(num_instances=1), dict(W=128), dict(W=64)],
                         ids=lambda o: _id(o) or "cfg2")
def test_cfg2_variants_route_by_heads_and_width(over, precision):
    cfg = make_cfg("cfg2", precision=precision, **over)
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=1))
    assert _tile_rows(prog) == _expect(cfg)


def test_cfg3_stays_on_64_rows():
    cfg = make_cfg("cfg3")
    prog, _, _ = build(cfg, S.init_network_weights(make_network(cfg), seed=2))
    assert _tile_rows(prog) == 64


@pytest.mark.parametrize("k", range(len(GRIDS)), ids=[f"L{L}F{F}" for L, F in GRIDS])
def test_hashgrid_programs_route_like_the_frequency_ones(k):
    L, F = GRIDS[k]
    cfg = hash_cfg("cfg2", hash_levels=L, hash_features=F, hash_log2_size=12, precision=GRID_MODES[k], **GRID_SHAPES[k])
    prog, _, _ = H.build(cfg, S.init_network_weights(make_network(cfg), seed=3))
    assert _tile_rows(prog) == _expect(cfg)
    cfg = hash_cfg("cfg2", hash_levels=L, hash_features=F, hash_log2_size=12, precision=GRID_MODES[k])
    prog, _, _ = H.build(cfg, S.init_network_weights(make_network(cfg), seed=3))
    assert _tile_rows(prog) == 128, "cfg2 with a hash-grid trunk input"


def test_tile_rows_refuses_bad_arguments():
    prog = MlpProgram()
    rows = C.c_int32()
    L = _capi.lib()
    assert L.pnr_program_tile_rows(C.byref(prog), C.sizeof(MlpProgram) - 4, C.byref(rows)) != 0
    assert b"bytes" in L.pnr_last_error()
    assert L.pnr_program_tile_rows(None, C.sizeof(MlpProgram), C.byref(rows)) != 0
    assert L.pnr_program_tile_rows(C.byref(prog), C.sizeof(MlpProgram), C.byref(rows)) == 0 and rows.value == 64
    assert L.pnr_set_mlp_rows(None, 128) != 0


MAP_PROBE = r"""
#include <cstdio>
#include "mlp_program.h"
using namespace pnr;
int main() {
  std::printf("%d %d %d %d %d %d %d %d %d %d %d %d %d %d %d %d\n", kSmem128Ring, kSlots128, kSlot128Bytes, kSmem128Blk,
              kBlk128Op, kBlk128Emb, kBlk128Dir, kBlk128Bytes, kSmem128Sig, kSmem128Bars, kSmem128Total, kRows,
              kOpKCoreBytes, kEmbPartBytes, kDirPartBytes, kColAHi);
}
"""


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs a host C++ compiler")
def test_shared_memory_map(tmp_path):
    src = tmp_path / "probe.cpp"
    src.write_text(MAP_PROBE)
    exe = tmp_path / "probe"
    subprocess.check_call(["g++", "-std=c++17", "-I", str(CSRC), "-o", str(exe), str(src)])
    (ring, slots, slot_bytes, blk, op, emb, dirr, blk_bytes, sig, bars, total, rows, kcore, emb_part, dir_part,
     col_a_hi) = map(int, subprocess.check_output([str(exe)], text=True).split())
    assert rows == 64 and kcore == rows * 16
    # regions, each [start, end): the ring, two blocks of (activations, embedding, view-dir embedding), sigma, barriers
    regions = [("ring", ring, ring + slots * slot_bytes)]
    for g in range(2):
        b = blk + g * blk_bytes
        regions += [(f"act{g}", b + op, b + op + (512 - col_a_hi) // 4 * kcore),     # columns [256, 512), hi + lo
                    (f"emb{g}", b + emb, b + emb + 2 * emb_part),                    # 64 K, hi + lo
                    (f"dir{g}", b + dirr, b + dirr + 2 * dir_part)]                  # 32 K, hi + lo
    regions += [("sig", sig, sig + 2 * rows * 4), ("bars", bars, bars + 2 * slots * 8)]
    regions.sort(key=lambda r: r[1])
    assert regions[0][1] == 0 and regions[-1][2] == total <= SMEM_LIMIT
    for (n0, _, e0), (n1, s1, _) in zip(regions, regions[1:]):
        assert e0 <= s1, f"{n0} overlaps {n1}"
    assert slots == 3 and slot_bytes == 16384
    assert (regions[1][2] - regions[1][1], emb_part, dir_part) == (65536, 8192, 4096)
    for name, s, _ in regions:   # operands and ring slots: 1024-byte aligned bases (16 bytes is what wgmma needs)
        if name != "bars" and name != "sig":
            assert s % 1024 == 0, name
    assert bars % 8 == 0
