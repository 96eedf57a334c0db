"""GPU tier of the mesh primitives of a5 (DESIGN 3.2): pnr_intersect_meshes against the torch oracle
(tests/oracle_mesh.py) bit for bit - a cfg2 frame with cuboids and meshes, B around the 512-box staging chunk, M = 1 /
4 / 8 with overflowing lists, rays through shared edges and vertices; without a table it is pnr_intersect; the fused
render with meshes against the staged one (bit for bit where the stages are, per ray against float64 for the maps);
Renderer.render against the oracle renderer; one training iteration with mesh primitives."""
import pytest
import torch

import oracle_mesh as OM
from oracle import reference_renderer as O
from panopticnerf_b200 import make_cfg, make_network, make_renderer, synthetic as S
from panopticnerf_b200.lib.networks.renderer import panopticnerf_renderer as P
from test_cpu_mesh_primitives import _dyadic_rays, comb, only_meshes
from test_gpu_render_limits import _bits_equal, _per_ray_ratio
from test_gpu_stage_limits import _report
from util import check_render_outputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _dev(d):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in d.items()}


def _gpu(rays, prims, M):
    p = _dev(prims)
    return P.intersect(rays.to(DEV), p["box_center"], p["box_half"], p["box_rot"], M, p["mesh_tri_start"],
                       p["mesh_tris"])


def _oracle(rays, prims, M):
    """The oracle on the device (the same IEEE ops as on the host; a frame of rays x 2000 triangles is too slow there)."""
    p = _dev(prims)
    r = rays.to(DEV)
    return OM.intersect(r[:, :3], r[:, 3:], p["box_center"], p["box_half"], p["box_rot"], M, p["mesh_tri_start"],
                        p["mesh_tris"])


def _same(got, ref, what):
    for a, b, k in zip(got, ref, ("hit_mask", "box_id", "t_in", "t_out")):
        _bits_equal(a, b, f"{what} {k}")


@pytest.mark.parametrize("M", [1, 4, 8])
def test_cfg2_frame_with_cuboids_and_meshes(M):
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg)
    assert rays.shape[0] == 529408
    prims = S.make_mesh_primitives()
    got = _gpu(rays, prims, M)
    _same(got, _oracle(rays, prims, M), f"frame M={M}")
    ids = got[1]
    assert bool((ids == 66).any()), "the road is never hit"
    if M > 1:
        assert bool(((ids == 65).sum(1) >= 2).any()), "no ray leaves and re-enters the U"


@pytest.mark.parametrize("B", [511, 512, 513, 1025])
def test_box_counts_around_the_staging_chunk(B):
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=60, row0=200)
    prims = S.make_mesh_primitives(num_boxes=B - 5, seed=B)
    assert prims["box_center"].shape[0] == B
    _same(_gpu(rays, prims, 8), _oracle(rays, prims, 8), f"B={B}")


@pytest.mark.parametrize("M", [1, 4, 8])
def test_overflowing_lists(M):
    combs = [comb(10), comb(10) + torch.tensor([0.5, 0.0, 0.0])]
    prims = only_meshes(combs)
    g = torch.Generator().manual_seed(M)
    o = torch.tensor([-3.0, 0.0, 2.0]) + (torch.rand(4096, 3, generator=g) - 0.5) * torch.tensor([0.0, 1.5, 1.5])
    d = torch.tensor([1.0, 0.0, 0.0]) + (torch.rand(4096, 3, generator=g) - 0.5) * 0.05
    rays = torch.cat([o, d], 1).contiguous()
    got = _gpu(rays, prims, M)
    _same(got, _oracle(rays, prims, M), f"comb M={M}")
    assert int((got[1] >= 0).all(1).sum()) > 1000


def test_rays_through_shared_edges_and_vertices():
    cube = S.box_triangles((0.0, 0.0, 8.0), (2.0, 2.0, 2.0), torch.eye(3))
    steps = [(0.5, 0.25, 8.0), (-0.75, 0.375, 16.0), (0.0, 0.0, 4.0), (1.0, -1.0, 2.0), (3.0, 1.5, -4.0)]
    v = cube.reshape(-1, 3)
    tg = [tuple(x) for x in v.tolist()]
    tg += [tuple(((a + b) / 2).tolist()) for t in cube for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0]))]
    rays = _dyadic_rays(tg, steps)
    prims = only_meshes([cube])
    ref = OM.intersect(rays[:, :3], rays[:, 3:], prims["box_center"], prims["box_half"], prims["box_rot"], 8,
                       prims["mesh_tri_start"], prims["mesh_tris"])
    _same(_gpu(rays, prims, 8), ref, "dyadic")


def test_without_a_table_it_is_pnr_intersect():
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=80, row0=100).to(DEV)
    bx = _dev(S.make_boxes(64))
    a = P.intersect(rays, bx["box_center"], bx["box_half"], bx["box_rot"], 4)
    from panopticnerf_b200 import _capi
    R = rays.shape[0]
    hit = torch.empty(R, dtype=torch.uint8, device=DEV)
    bid = torch.empty(R, 4, dtype=torch.int32, device=DEV)
    tin, tout = torch.empty(R, 4, device=DEV), torch.empty(R, 4, device=DEV)
    _capi.check(_capi.lib().pnr_intersect_meshes(rays.data_ptr(), R, bx["box_center"].data_ptr(), bx["box_half"].data_ptr(),
                                                 bx["box_rot"].data_ptr(), None, None, 0, 64, 4, hit.data_ptr(),
                                                 bid.data_ptr(), tin.data_ptr(), tout.data_ptr(), _capi.stream_ptr()))
    _same((hit.bool(), bid, tin, tout), a, "no table")


# ------------------------------------------------------------------------------------------------ render
def _with(cfg, **over):
    d = dict(vars(cfg))
    preset = d.pop("preset")
    return make_cfg(preset, **dict(d, **over))


def _mesh_batch(cfg, R, seed, row0=200, step=3):
    prims = S.make_mesh_primitives(int(64), int(cfg.num_classes), int(cfg.num_instances), seed=seed)
    rays = S.make_rays(cfg, seed=seed, row0=row0, rows=(R * step + int(cfg.W_img) - 1) // int(cfg.W_img))[::step][:R]
    b = dict(prims, rays=rays.contiguous(), scene_aabb=torch.tensor(S.SCENE_AABB))
    return b


CASES = [dict(sample_mode="uniform", bound_by_primitives=False, N_samples=64, N_importance=0),
         dict(sample_mode="intervals", bound_by_primitives=True, N_samples=64, N_importance=64),
         dict(sample_mode="uniform", bound_by_primitives=True, N_samples=32, N_importance=96, perturb=1.0),
         dict(sample_mode="intervals", bound_by_primitives=False, N_samples=64, N_importance=128, perturb=1.0)]


@pytest.mark.parametrize("i", range(len(CASES)))
def test_fused_render_with_meshes_equals_the_staged_render(i):
    cfg = make_cfg("cfg2", D=4, W=128, num_classes=45, num_instances=64, max_hits=(8, 4, 1, 8)[i], **CASES[i])
    net = S.init_network_weights(make_network(cfg), seed=i).to(DEV)
    b = _dev(_mesh_batch(cfg, 3000, seed=i))
    g = torch.Generator().manual_seed(i)
    R, N, Ni = b["rays"].shape[0], cfg.N_samples, cfg.N_importance
    b["u"] = torch.rand(R, N, generator=g).to(DEV)
    if Ni:
        b["u_fine"] = torch.sort(torch.rand(R, Ni, generator=g), -1).values.to(DEV)
    staged = make_renderer(_with(cfg, render_path="staged", return_raw=True), net).render(b)
    fused = make_renderer(cfg, net).render(b)
    chunked = make_renderer(_with(cfg, gpu_chunk=700), net).render(b)
    assert bool((staged["box_id"] >= 64).any())
    exact = ["hit_mask", "box_id", "t_in", "t_out", "sample_box", "z_vals", "z_vals_0", "weights", "weights_0",
             "fixed_semantic_map", "fixed_instance_map", "fixed_semantic_map_0", "fixed_instance_map_0", "near", "far"]
    for k in exact:
        if k in staged:
            _bits_equal(fused[k], staged[k], f"case {i} {k}")
    for k in fused:
        _bits_equal(chunked[k], fused[k], f"case {i} chunked {k}")
    flags = dict(white=cfg.white_bkgd, mask=cfg.mask_outside, softmax=False)
    worst, where = _per_ray_ratio(fused, staged["raw"], staged["z_vals"], b["rays"], cfg.num_classes, cfg.num_instances,
                                  staged["sample_box"], b["box_sem"], b["box_inst"], **flags)
    _report(f"render_fused with meshes case {i} [{where}]", worst)


def test_render_matches_the_oracle_renderer():
    cfg = make_cfg("cfg2", D=4, W=64, N_samples=64, N_importance=32, num_classes=8, num_instances=8, max_hits=4,
                   sample_mode="intervals", bound_by_primitives=True)
    net = S.init_network_weights(make_network(cfg), seed=2)
    onet = O.make_network(cfg)
    onet.load_state_dict(net.state_dict())
    b = _mesh_batch(cfg, 1500, seed=2, row0=220, step=5)
    out = make_renderer(cfg, net.to(DEV)).render(_dev(b))
    with OM.oracle_renderer_with_meshes():
        ref = O.make_renderer(cfg, onet).render(b)
    assert bool((ref["box_id"] >= 64).any())
    for k in ("hit_mask", "box_id", "z_vals_0"):
        assert torch.equal(out[k].cpu().to(ref[k].dtype), ref[k]), k
    # the fine depths are discontinuous in the coarse weights: compare what does not depend on them
    check_render_outputs(out, {k: v for k, v in ref.items() if k.endswith("_0") or k in ("near", "far", "t_in", "t_out")},
                         float(cfg.far))


# ------------------------------------------------------------------------------------------------ training
def test_one_training_iteration_with_mesh_primitives():
    from panopticnerf_b200.lib.train import NetworkWrapper
    cfg = make_cfg("cfg3", render_path="staged", bound_by_primitives=True, perturb=1.0, check_range=True)
    net = S.init_network_weights(make_network(cfg), seed=31).to(DEV)
    fine = S.init_network_weights(make_network(cfg), seed=32).to(DEV)
    R = 1200
    b = _mesh_batch(cfg, R, seed=3, row0=230, step=4)
    g = torch.Generator().manual_seed(9)
    N, Ni = int(cfg.N_samples), int(cfg.N_importance)
    b.update(u=torch.rand(R, N, generator=g), u_fine=torch.rand(R, Ni, generator=g), rgb=torch.rand(R, 3, generator=g),
             depth=torch.rand(R, generator=g) * 40 + 5, pseudo_label=torch.randint(-1, int(cfg.num_classes), (R,), generator=g))
    b["box_inst"] = torch.arange(b["box_center"].shape[0], dtype=torch.int32) % int(cfg.num_instances)
    wrapper = NetworkWrapper(cfg, net, fine)
    output, loss, stats, _ = wrapper(_dev(b))
    loss.backward()
    assert torch.isfinite(loss) and float(fine.instance_linears[1].weight.grad.norm()) > 0.0
    w, sb = output["weights"].detach().cpu().double(), output["sample_box"].cpu()
    for key, table, n in (("fixed_semantic_map", b["box_sem"], cfg.num_classes),
                          ("fixed_instance_map", b["box_inst"], cfg.num_instances)):
        ref = O._composite_onehot(w, sb, table, n)
        err = (output[key].detach().cpu().double() - ref).abs().max()
        assert float(err) <= 1e-5, (key, float(err))
    ids = output["box_id"].cpu()
    only_mesh = (ids >= 64).any(1) & ~((ids >= 0) & (ids < 64)).any(1)
    assert int(only_mesh.sum()) > 20
    fim = output["fixed_instance_map"].detach().cpu()[only_mesh]
    assert bool((fim.sum(1) > 0).any())
    assert bool((output["inst_label"].cpu()[only_mesh] >= 0).any())
