"""CPU tier: the driver-facing contract of bench.py that can be exercised without a GPU - the reference arm
(`--impl reference`, the in-repo oracle on the host cores): exactly one JSON line on stdout with the agreed keys,
alone and under torchrun (rank 0 prints, the other ranks exit 0 silently); --dump-outputs stays within its 64 MB
whatever the configuration's bytes per ray."""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
KEYS = {"impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
        "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"}


def _run(cmd):
    p = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, f"stdout must be one JSON line, got {len(lines)}: {p.stdout[:500]}"
    return json.loads(lines[0])


def _check(d, n_gpus):
    assert KEYS <= set(d), KEYS - set(d)
    assert d["impl"] == "reference" and d["n_gpus"] == n_gpus and d["unit"] == "rays/s"
    assert d["value"] > 0 and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"]


def test_reference_arm_prints_one_json_line():
    _check(_run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "1", "--ref-rows", "1"]), 1)


def _free_port() -> int:
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_reference_arm_under_torchrun_only_rank0_reports():
    d = _run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
              "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), "bench.py", "--impl", "reference",
              "--gpus", "2", "--steps", "1", "--warmup", "1", "--ref-rows", "1"])
    _check(d, 2)


def test_reference_arm_dumps_outputs(tmp_path):
    _check(_run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "1", "--ref-rows", "1",
                 "--dump-outputs", str(tmp_path)]), 1)
    import numpy as np
    rgb, rows = np.load(tmp_path / "rgb_map.npy"), np.load(tmp_path / "sample_rays.npy")
    assert rgb.dtype == np.float32 and rgb.shape == (len(rows), 3) and rows.dtype == np.float64


# The outputs of a config-3 frame (pnr_render_fused with heads and a fine pass; panopticnerf_renderer.py): final and
# coarse maps, per-sample weights / depths / primitive ids of both passes.  ~4.5 KB per ray as dumped.
_CFG3_SHAPES = {"rgb_map": (3,), "depth_map": (), "acc_map": (), "disp_map": (), "semantic_map": (45,),
                "instance_map": (64,), "fixed_semantic_map": (45,), "fixed_instance_map": (64,), "weights": (192,),
                "z_vals": (192,), "rgb_map_0": (3,), "depth_map_0": (), "acc_map_0": (), "disp_map_0": (),
                "semantic_map_0": (45,), "instance_map_0": (64,), "weights_0": (64,), "z_vals_0": (64,),
                "near": (), "far": (), "t_in": (4,), "t_out": (4,)}
_CFG3_INT = {"sample_box": (192,), "box_id": (4,), "hit_mask": ()}


def test_dump_outputs_fits_config3_frame(tmp_path):
    """A cfg3-sized output dict (529 408 rays; expanded tensors, so nothing large is allocated) goes through
    bench.dump_outputs in a subprocess (importing bench rebinds this process's stdout): the files stay under 64 MB and
    two dumps write the same sample."""
    code = f"""
import sys, torch
sys.path.insert(0, {str(ROOT)!r})
import bench
R = 529408
out = {{k: torch.ones(1, *s).expand(R, *s) for k, s in {_CFG3_SHAPES!r}.items()}}
out.update({{k: torch.ones(1, *s, dtype=torch.int32).expand(R, *s) for k, s in {_CFG3_INT!r}.items()}})
for d in sys.argv[1:]:
    bench.dump_outputs(out, __import__("pathlib").Path(d))
"""
    dirs = [tmp_path / "a", tmp_path / "b"]
    p = subprocess.run([sys.executable, "-c", code, *map(str, dirs)], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    import numpy as np
    for d in dirs:
        total = sum(f.stat().st_size for f in d.glob("*.npy"))
        assert 0 < total <= 64 << 20, total
    rows = np.load(dirs[0] / "sample_rays.npy")
    assert 1000 < len(rows) < 32768 and np.array_equal(rows, np.load(dirs[1] / "sample_rays.npy"))
    assert np.load(dirs[0] / "weights.npy").shape == (len(rows), 192)
    assert np.load(dirs[0] / "sample_box.npy").dtype == np.float64
