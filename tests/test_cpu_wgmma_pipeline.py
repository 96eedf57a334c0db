"""CPU: the fused MLP kernel and the weight-gradient kernel keep several wgmmas in flight.

ptxas serializes every wgmma of a function (each one followed by a wait for it) when it cannot prove the pipeline safe:
a call anywhere in the kernel, a wgmma whose accumulator array or N is chosen at run time, registers of an in-flight
accumulator moved by other instructions, or a join between a wgmma and its commit.  It says so with a "Potential
Performance Loss" note (C7510, C7515, C7520, ...).  Such a kernel runs every MMA at its full latency.  These tests read
the ptxas logs of mlp_wgmma.cu and wgrad_wgmma.cu and the SASS of the built library."""
import re
import subprocess
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "panopticnerf_b200" / "csrc"
PIPELINED = {"mlp_wgmma.cu": "mlp_fused_kernel", "wgrad_wgmma.cu": "wgrad_kernel"}   # source -> kernel


def _nvcc():
    from panopticnerf_b200 import _build
    return _build._nvcc(), _build.NVCC_FLAGS


def test_ptxas_does_not_serialize_wgmma(tmp_path):
    nvcc, flags = _nvcc()
    procs = {src: subprocess.Popen([nvcc, *flags, "-Xptxas", "-v", "-c", str(CSRC / src), "-o", str(tmp_path / (src + ".o"))],
                                   stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for src in PIPELINED}
    logs = {src: p.communicate()[0] for src, p in procs.items()}
    for src, kernel in PIPELINED.items():
        log = logs[src]
        assert procs[src].returncode == 0, log
        assert kernel in log, src
        notes = [l for l in log.splitlines() if "wgmma.mma_async instructions are serialized" in l]
        assert not notes, "\n".join(notes[:8])
        for code in ("C7510", "C7515", "C7520"):
            assert code not in log, f"{src}: {code}"
    # no spills: the accumulators stay in registers next to the epilogue state
    for m in re.finditer(r"Compiling entry function '(\w*mlp_fused_kernel\w*)'.*?(\d+) bytes spill stores",
                         logs["mlp_wgmma.cu"], re.S):
        assert m.group(2) == "0", f"{m.group(1)} spills {m.group(2)} bytes"


def test_sass_keeps_wgmma_groups_in_flight():
    so = ROOT / "panopticnerf_b200" / "libpnr.so"
    assert so.exists(), "build the library first (__graft_entry__.build())"
    sass = subprocess.run(["cuobjdump", "-sass", str(so)], capture_output=True, text=True).stdout
    hgmma, depbar, fn = Counter(), Counter(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if any(k in m.group(1) for k in PIPELINED.values()) else None
        elif fn is not None:
            hgmma[fn] += "HGMMA" in line
            depbar[fn] += "WARPGROUP.DEPBAR" in line
    fused = [fn for fn in hgmma if "mlp_fused_kernel" in fn]
    assert len(fused) == 10, sorted(fused)   # {x3, 1-pass} x {fp16, bf16} x {raw, compositing} + backward x {fp16, bf16}
    assert len(hgmma) - len(fused) == 2, sorted(hgmma)   # wgrad_kernel x {fp16, bf16}
    for fn in hgmma:
        # a serialized kernel waits after every HGMMA; a pipelined one only once per issued group
        assert hgmma[fn] > 0 and depbar[fn] * 3 <= hgmma[fn], f"{fn}: {hgmma[fn]} HGMMA, {depbar[fn]} WARPGROUP.DEPBAR"
