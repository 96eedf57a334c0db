"""Device time of the ray / primitive intersection (a5) with and without mesh primitives (DESIGN 3.2), CUDA events,
median of --reps runs after warm-up, the variants alternated in each round.  Prints the card and its power limit with
the numbers as JSON, and also writes that JSON to --out when given.

  1. the bench's synthetic scene - a cfg2 frame (529 408 rays), 64 cuboids - through pnr_intersect and through
     pnr_intersect_meshes without a table (the same kernel: the times should agree within the spread);
  2. the same frame with the 64 cuboids plus the five meshes of synthetic.make_mesh_primitives (an ellipsoid and a
     nested one, a U extrusion, the ~2000-triangle road under the camera, a cuboid as 12 triangles), with the number of
     triangle tests (rays in each mesh's cull box x its triangles);
  3. for scale, the fused render of that frame (cfg2 network) with cuboids only and with the meshes;
  4. a sequence table (pnr_intersect_frames: S static boxes, then 20 dynamic boxes for each of 300 frames) against the
     static table alone (pnr_intersect on the S boxes), for S = 64 and 2000: a 2048-ray training batch whose rays belong
     to random frames, and a cfg2 frame whose rays all belong to one frame."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import panopticnerf_b200 as PN  # noqa: E402
from panopticnerf_b200 import _capi, synthetic as S  # noqa: E402
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P  # noqa: E402

DEV = "cuda:0"


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fns, reps: int, warmup: int):
    """{name: median ms} of each fn, alternated within every round."""
    for _ in range(warmup):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    return {k: statistics.median(v) for k, v in ms.items()}, {k: (min(v), max(v)) for k, v in ms.items()}


def sequence_tables(frame_rays, M: int, reps: int, warmup: int, F: int = 300, per_frame: int = 20):
    """{case: median ms}: static-only against the sequence table, alternated, for a training batch and a frame."""
    g = torch.Generator().manual_seed(0)
    batch_rays = frame_rays[torch.randperm(frame_rays.shape[0], generator=g)[:2048].to(DEV)].contiguous()
    L = _capi.lib()
    fns, keep = {}, []
    for S_ in (64, 2000):
        prims = {k: v.to(DEV) for k, v in S.make_boxes(S_ + F * per_frame, seed=S_).items()}
        fb = torch.stack([S_ + per_frame * torch.arange(F), S_ + per_frame * torch.arange(1, F + 1)], 1)
        fb = fb.to(torch.int32).to(DEV)
        for name, rays, rf in (("batch2048", batch_rays, torch.randint(0, F, (2048,), generator=g, dtype=torch.int32)),
                               ("frame", frame_rays, torch.full((frame_rays.shape[0],), 7, dtype=torch.int32))):
            R = rays.shape[0]
            rf = rf.to(DEV)
            out = [torch.empty(R, dtype=torch.uint8, device=DEV), torch.empty(R, M, dtype=torch.int32, device=DEV),
                   torch.empty(R, M, device=DEV), torch.empty(R, M, device=DEV)]
            keep += [prims, fb, rays, rf, out]
            a = _capi.PnrIntersectFramesArgs(rays=rays.data_ptr(), R=R, box_center=prims["box_center"].data_ptr(),
                                             box_half=prims["box_half"].data_ptr(), box_rot=prims["box_rot"].data_ptr(),
                                             B=S_ + F * per_frame, M=M, hit_mask=out[0].data_ptr(),
                                             box_id=out[1].data_ptr(), t_in=out[2].data_ptr(), t_out=out[3].data_ptr())
            a.frames = _capi.PnrFrameTable(ray_frame=rf.data_ptr(), frame_boxes=fb.data_ptr(), F=F, S=S_)
            static = lambda a=a, S_=S_: _capi.check(L.pnr_intersect(a.rays, a.R, a.box_center, a.box_half, a.box_rot,
                                                                    S_, a.M, a.hit_mask, a.box_id, a.t_in, a.t_out,
                                                                    _capi.stream_ptr()))
            seq = lambda a=a: _capi.check(L.pnr_intersect_frames(C.byref(a), _capi.stream_ptr()))
            keep.append(a)
            fns[f"{name}_S{S_}_static"] = static
            fns[f"{name}_S{S_}_sequence"] = seq
    return timed(fns, reps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--M", type=int, default=4)
    ap.add_argument("--out", type=Path, default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert args.reps >= 20
    cfg = PN.make_cfg("cfg2")
    rays = S.make_rays(cfg).to(DEV)
    R, M = rays.shape[0], args.M
    bx = {k: v.to(DEV) for k, v in S.make_boxes(64, int(cfg.num_classes), int(cfg.num_instances)).items()}
    mp = {k: v.to(DEV) for k, v in S.make_mesh_primitives(64, int(cfg.num_classes), int(cfg.num_instances)).items()}
    B, Bm = bx["box_center"].shape[0], mp["box_center"].shape[0]
    out = [torch.empty(R, dtype=torch.uint8, device=DEV), torch.empty(R, M, dtype=torch.int32, device=DEV),
           torch.empty(R, M, device=DEV), torch.empty(R, M, device=DEV)]
    o = [t.data_ptr() for t in out]
    L = _capi.lib()
    p = lambda t: t.data_ptr()

    def cuboids():
        _capi.check(L.pnr_intersect(p(rays), R, p(bx["box_center"]), p(bx["box_half"]), p(bx["box_rot"]), B, M, *o,
                                    _capi.stream_ptr()))

    def no_table():
        _capi.check(L.pnr_intersect_meshes(p(rays), R, p(bx["box_center"]), p(bx["box_half"]), p(bx["box_rot"]), None,
                                           None, 0, B, M, *o, _capi.stream_ptr()))

    def meshes():
        _capi.check(L.pnr_intersect_meshes(p(rays), R, p(mp["box_center"]), p(mp["box_half"]), p(mp["box_rot"]),
                                           p(mp["mesh_tri_start"]), p(mp["mesh_tris"]), mp["mesh_tris"].shape[0], Bm,
                                           M, *o, _capi.stream_ptr()))

    med, rng = timed({"pnr_intersect": cuboids, "pnr_intersect_meshes_no_table": no_table, "mixed_scene": meshes},
                     args.reps, args.warmup)
    start = mp["mesh_tri_start"].cpu()
    tests, per_mesh = 0, {}
    for b in range(Bm):
        n = int(start[b + 1] - start[b])
        if n == 0:
            continue
        hit = P.intersect(rays, mp["box_center"][b:b + 1], mp["box_half"][b:b + 1], mp["box_rot"][b:b + 1], 1)[0]
        per_mesh[b] = dict(triangles=n, rays_in_cull_box=int(hit.sum()))
        tests += n * int(hit.sum())

    net = S.init_network_weights(PN.make_network(cfg)).to(DEV)
    ren = PN.make_renderer(cfg, net)
    base = {"rays": rays, "scene_aabb": torch.tensor(S.SCENE_AABB)}
    b_cub, b_mesh = dict(base, **bx), dict(base, **mp)
    rmed, rrng = timed({"render_cuboids": lambda: ren.render(b_cub), "render_meshes": lambda: ren.render(b_mesh)},
                       max(20, args.reps // 5), 2)
    smed, srng = sequence_tables(rays, M, args.reps, args.warmup)
    res = dict(card=card(), rays=R, M=M, cuboids=B, primitives_mixed=Bm, triangles=int(mp["mesh_tris"].shape[0]),
               triangle_tests=tests, triangle_tests_per_ray=tests / R, per_mesh=per_mesh, median_ms={**med, **rmed},
               min_max_ms={**rng, **rrng}, sequence_table=dict(frames=300, dynamic_per_frame=20, median_ms=smed,
                                                               min_max_ms=srng))
    print(json.dumps(res, indent=1))
    if args.out is not None:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
