"""Config object for the render path.

The reference drives every plugin from a global yacs ``cfg`` (SURVEY.md section 5; recalled key
names ``N_samples, N_importance, chunk, perturb, white_bkgd, xyz_res, view_res, network_module,
renderer_module ...``; the reference's lib/config is not in the mount so no file:line exists).
Here ``cfg`` is a plain attribute namespace with the same key names; anything attribute-style
(yacs CfgNode, SimpleNamespace, argparse Namespace) is accepted by make_network / make_renderer.
"""
from __future__ import annotations

from types import SimpleNamespace

_DEFAULTS = dict(
    task="panopticnerf",
    network_module="panopticnerf_b200.lib.networks.panopticnerf.network",
    renderer_module="panopticnerf_b200.lib.networks.renderer.panopticnerf_renderer",
    # MLP (SURVEY 8a a8)
    D=8, W=256, xyz_res=10, view_res=4, num_classes=0, num_instances=0,
    # trunk input: "frequency" = gamma(x) (the network above) | "hashgrid" = h(x), the multi-resolution hash-grid features
    # of the point (E = hash_levels * hash_features <= 64 columns in place of gamma(x); rule chosen here, the reference's
    # 360 architecture is not in the mount).  hash_aabb [lo.xyz, hi.xyz] is required with "hashgrid".
    xyz_encoding="frequency", hash_levels=16, hash_features=2, hash_log2_size=19,
    hash_base_resolution=16.0, hash_per_level_scale=1.3819, hash_aabb=None,
    # sampling / rendering (a5, a6, a9, a10)
    N_samples=64, N_importance=0, perturb=0.0, white_bkgd=False, raw_noise_std=0.0,
    near=0.05, far=80.0, max_hits=4, bound_by_primitives=False, mask_outside=False,
    # a6: "uniform" = near..far, samples tagged with the hit interval they fall in; "intervals" = the N samples are
    # placed inside the ray's hit intervals (rule in oracle/reference_renderer.py::interval_z / DESIGN.md)
    sample_mode="uniform",
    sem_activation="none", chunk=32768, return_raw=False,
    # image shape (KITTI-360 perspective, SURVEY 8d)
    H=376, W_img=1408, fx=552.554, fy=552.554, cx=682.05, cy=238.77, camera="pinhole",
    # GPU path
    # tensor-core operand format x passes: "fp16x3" (default; ~2^-21 per product, meets the 1e-4 tolerance
    # with margin, needs |activation| < 65504) | "bf16x3" (~2^-17, fp32 range) | "fp16" / "bf16" (1 pass, fast)
    precision="fp16x3",
    # Renderer.render: "fused" = one pnr_render_fused call per frame (chunked inside by the workspace, `raw` never
    # materialised for the frame); "staged" = one libpnr call per stage from Python (implied by return_raw).
    # workspace_mb = 0: pnr_workspace_bytes' default (raw ~1.5 GB per chunk).
    render_path="fused", workspace_mb=0,
    # raise if the fp16 operands overflowed in this render (costs one 4-byte D2H read per render)
    check_range=True,
    # training (lib/train/network_wrapper.py): loss weights of the photometric (fine + coarse), depth, pseudo-label
    # semantic, fixed-semantic and instance terms; a ray supervises the instance head when its dominant primitive
    # holds at least inst_min_weight of its rendering weight
    trainer_module="panopticnerf_b200.lib.train.network_wrapper",
    w_rgb=1.0, w_depth=0.1, w_sem=1.0, w_fix=1.0, w_inst=1.0, inst_min_weight=0.5,
)

# BASELINE.json "configs", in order.
PRESETS = {
    "cfg1": dict(D=4, W=64, N_samples=32, H=64, W_img=64, fx=60.0, fy=60.0, cx=32.0, cy=32.0),
    "cfg2": dict(),
    "cfg3": dict(num_classes=45, num_instances=64, N_importance=128),
    "cfg4": dict(),   # cfg2 per frame, 8 frames ray-sharded over the ranks
    "cfg5": dict(num_classes=45, num_instances=64, N_samples=192, H=1024, W_img=2048,
                 camera="equirect"),
}


def make_cfg(preset: str = "cfg2", **overrides) -> SimpleNamespace:
    d = dict(_DEFAULTS)
    d.update(PRESETS[preset])
    d.update(overrides)
    d["preset"] = preset
    return SimpleNamespace(**d)
