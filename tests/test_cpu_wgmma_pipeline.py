"""CPU: the fused MLP kernel keeps several wgmmas in flight.

ptxas serializes every wgmma of a function (each one followed by a wait for it) when it cannot prove the pipeline safe:
a call anywhere in the kernel, a wgmma whose accumulator array or N is chosen at run time, registers of an in-flight
accumulator moved by other instructions, or a join between a wgmma and its commit.  It says so with a "Potential
Performance Loss" note (C7510, C7515, C7520, ...).  Such a kernel runs every MMA at its full latency.  These tests read
the ptxas log of mlp_wgmma.cu and the SASS of the built library."""
import re
import subprocess
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "panopticnerf_b200" / "csrc"


def _nvcc():
    from panopticnerf_b200 import _build
    return _build._nvcc(), _build.NVCC_FLAGS


def test_ptxas_does_not_serialize_wgmma(tmp_path):
    nvcc, flags = _nvcc()
    r = subprocess.run([nvcc, *flags, "-Xptxas", "-v", "-c", str(CSRC / "mlp_wgmma.cu"), "-o", str(tmp_path / "mlp.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    assert "mlp_fused_kernel" in log
    notes = [l for l in log.splitlines() if "wgmma.mma_async instructions are serialized" in l]
    assert not notes, "\n".join(notes[:8])
    for code in ("C7510", "C7515", "C7520"):
        assert code not in log, code
    # no spills: the accumulators stay in registers next to the epilogue state
    for m in re.finditer(r"Compiling entry function '(\w*mlp_fused_kernel\w*)'.*?(\d+) bytes spill stores", log, re.S):
        assert m.group(2) == "0", f"{m.group(1)} spills {m.group(2)} bytes"


def test_sass_keeps_wgmma_groups_in_flight():
    so = ROOT / "panopticnerf_b200" / "libpnr.so"
    assert so.exists(), "build the library first (__graft_entry__.build())"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True).stdout
    hgmma, depbar, fn = Counter(), Counter(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if "mlp_fused_kernel" in m.group(1) else None
        elif fn is not None:
            hgmma[fn] += "HGMMA" in line
            depbar[fn] += "WARPGROUP.DEPBAR" in line
    assert len(hgmma) == 10, sorted(hgmma)   # {x3, 1-pass} x {fp16, bf16} x {raw, compositing} + backward x {fp16, bf16}
    for fn in hgmma:
        # a serialized kernel waits after every HGMMA; a pipelined one only once per issued group
        assert hgmma[fn] > 0 and depbar[fn] * 3 <= hgmma[fn], f"{fn}: {hgmma[fn]} HGMMA, {depbar[fn]} WARPGROUP.DEPBAR"
