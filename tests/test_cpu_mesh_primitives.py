"""CPU tier of the mesh primitives of a5 (DESIGN 3.2): the routines of csrc/ray_math.h built for the host with
-ffp-contract=off (tests/host_emu.cpp) equal the torch oracle (tests/oracle_mesh.py) bit for bit; the intervals
agree with exact geometry; a cuboid given as 12 triangles agrees with the slab test; the KITTI-360 reader's mesh
primitives; the argument checks of pnr_intersect_meshes (refused with PNR_ERR_ARG before any CUDA call: the pointers
are placeholders that are never dereferenced) and the ctypes layout of pnr_render_args against the header."""
import ctypes as C
import shutil
import subprocess
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_mesh as OM
from host_emu import emu  # noqa: F401  (fixture)
from oracle import reference_renderer as O
from panopticnerf_b200 import _capi, make_cfg, synthetic as S
from panopticnerf_b200.lib.datasets import kitti360 as K
from panopticnerf_b200.lib.datasets.kitti360 import bboxes as KB
from panopticnerf_b200.lib.datasets.kitti360 import intersection_cache as KC

ROOT = Path(__file__).resolve().parent.parent
X = 64          # a non-null placeholder pointer
ERR_ARG = -1


def _p(t):
    return C.c_void_p(t.data_ptr())


def emu_intersect(emu, rays, prims, M):
    R, B = rays.shape[0], prims["box_center"].shape[0]
    hit = torch.zeros(R, dtype=torch.uint8)
    bid = torch.zeros(R, M, dtype=torch.int32)
    tin, tout = torch.zeros(R, M), torch.zeros(R, M)
    tris = prims["mesh_tris"].contiguous()
    emu.emu_intersect(_p(rays), C.c_int64(R), _p(prims["box_center"]), _p(prims["box_half"]),
                      _p(prims["box_rot"]), _p(prims["mesh_tri_start"]), _p(tris), C.c_int64(tris.shape[0]), B, M,
                      _p(hit), _p(bid), _p(tin), _p(tout))
    return hit.bool(), bid, tin, tout


def oracle(rays, prims, M):
    return OM.intersect(rays[:, :3], rays[:, 3:], prims["box_center"], prims["box_half"], prims["box_rot"], M,
                        prims["mesh_tri_start"], prims["mesh_tris"])


def assert_same(a, b):
    for x, y, k in zip(a, b, ("hit_mask", "box_id", "t_in", "t_out")):
        assert torch.equal(x, y), (k, int((x != y).sum()))


def only_meshes(meshes):
    """A primitive table of the given meshes alone, each with its cull box."""
    tris, starts = S.mesh_table(meshes)
    cb = [S.cull_box(m) for m in meshes]
    return dict(box_center=torch.stack([c for c, _, _ in cb]).contiguous(),
                box_half=torch.stack([h for _, h, _ in cb]).contiguous(),
                box_rot=torch.stack([r for _, _, r in cb]).contiguous(),
                mesh_tri_start=torch.tensor(starts + [tris.shape[0]], dtype=torch.int32), mesh_tris=tris)


def comb(teeth: int, y0=-1.0, y1=1.0):
    """An extruded comb (x, z): a bar [0, 2n-1] x [0, 1] with n teeth [2i, 2i+1] x [1, 3].  A ray along x at z = 2
    crosses n intervals of one primitive."""
    n = teeth
    poly = [(0.0, 0.0), (2.0 * n - 1, 0.0)]
    for i in range(n - 1, -1, -1):
        poly += [(2.0 * i + 1, 3.0), (2.0 * i, 3.0)]
        if i > 0:
            poly += [(2.0 * i, 1.0), (2.0 * i - 1, 1.0)]
    # cap: each tooth is two triangles on its own corners and the bar below it; the bar is a fan over its corners
    idx = {p: k for k, p in enumerate(poly)}
    caps = []
    for i in range(n):
        a, b = idx[(2.0 * i, 3.0)], idx[(2.0 * i + 1, 3.0)]
        lo_l = idx.get((2.0 * i, 1.0), idx[(0.0, 0.0)] if i == 0 else None)
        lo_r = idx.get((2.0 * i + 1, 1.0), idx[(2.0 * n - 1, 0.0)] if i == n - 1 else None)
        caps += [(lo_l, lo_r, b), (lo_l, b, a)]
    bar = [idx[(0.0, 0.0)], idx[(2.0 * n - 1, 0.0)]] + [idx[(float(x), 1.0)] for x in range(2 * n - 2, 0, -1)]
    for k in range(1, len(bar) - 1):
        caps.append((bar[0], bar[k], bar[k + 1]))
    return S.extrusion(poly, caps, y0, y1)


# ------------------------------------------------------------------------------------------ host build vs oracle
@pytest.mark.parametrize("M,row0", [(1, 200), (4, 240), (8, 300), (3, 330)])
def test_random_rays_match_the_oracle(emu, M, row0):
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=24, row0=row0)[::2].contiguous()
    prims = S.make_mesh_primitives(seed=1)
    ref = oracle(rays, prims, M)
    assert_same(emu_intersect(emu, rays, prims, M), ref)
    ids = ref[1]
    assert bool((ids >= 64).any()), "no ray reached a mesh"


def test_every_mesh_is_reached_and_nested_meshes_both_report(emu):
    cfg = make_cfg("cfg2")
    rays = S.make_rays(cfg, rows=120, row0=200)[::5].contiguous()
    prims = S.make_mesh_primitives(seed=0)
    ref = oracle(rays, prims, 8)
    assert_same(emu_intersect(emu, rays, prims, 8), ref)
    ids = ref[1]
    for b in range(64, 69):
        assert bool((ids == b).any(1).any()), f"mesh {b} is never hit"
    both = (ids == 64).any(1) & (ids == 68).any(1)     # the inner ellipsoid inside the outer one
    assert bool(both.any())
    inner = both.nonzero()[0, 0]
    m_in, m_out = (ids[inner] == 68).nonzero()[0, 0], (ids[inner] == 64).nonzero()[0, 0]
    assert ref[2][inner, m_out] < ref[2][inner, m_in] < ref[3][inner, m_in] < ref[3][inner, m_out]


def _dyadic_rays(targets, steps):
    """A ray through each target, from target - step: with dyadic targets and steps whose z component is a power of two
    and the largest, the shear factors d_x / d_z, d_y / d_z and every sheared coordinate are exact."""
    t = torch.tensor(targets, dtype=torch.float32)
    st = torch.tensor(steps, dtype=torch.float32)
    d = st.repeat(t.shape[0] // st.shape[0] + 1, 1)[:t.shape[0]]
    return torch.cat([t - d, d], 1).contiguous()


def test_rays_through_shared_edges_and_vertices_cross_once(emu):
    """Dyadic coordinates: every sheared coordinate is exact, so these rays pass exactly through the edges and vertices
    of the meshes.  A ray through the inside of a closed convex mesh crosses it exactly twice (entry, exit), however
    many triangles meet where it enters; one that only touches an edge or vertex crosses an even count."""
    cube = S.box_triangles((0.0, 0.0, 8.0), (2.0, 2.0, 2.0), torch.eye(3))
    oct_v = [(0, 0, 4), (0, 0, 12), (4, 0, 8), (-4, 0, 8), (0, 4, 8), (0, -4, 8)]
    oct_f = [(0, 2, 4), (0, 4, 3), (0, 3, 5), (0, 5, 2), (1, 4, 2), (1, 3, 4), (1, 5, 3), (1, 2, 5)]
    octa = S._tri_mesh(oct_v, oct_f)
    steps = [(0.5, 0.25, 8.0), (-0.75, 0.375, 16.0), (0.0, 0.0, 4.0), (1.0, -1.0, 2.0), (3.0, 1.5, -4.0)]
    for mesh in (cube, octa):
        v = mesh.reshape(-1, 3)
        tg = [tuple(x) for x in v.tolist()]                                       # vertices
        tg += [tuple(((a + b) / 2).tolist()) for t in mesh for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0]))]
        n_thru = len(tg)
        tg += [tuple(x) for x in (v.mean(0) + 0.5 * (v - v.mean(0))).tolist()]  # through the inside
        rays = _dyadic_rays(tg, steps)
        prims = only_meshes([mesh])
        ref = oracle(rays, prims, 8)
        assert_same(emu_intersect(emu, rays, prims, 8), ref)
        cross, t = OM.crossings(rays[:, :3], rays[:, 3:], mesh)
        n = cross.sum(1)
        assert bool((n % 2 == 0).all()), n
        assert bool((n[n_thru:] == 2).all())                                     # the rays through the inside
        assert bool((n <= 2).all())                                              # convex: never more than one passage
        assert bool(ref[0][n_thru:].all())
        # a ray through an edge point or vertex that lies inside the mesh's silhouette enters exactly once
        assert int((n[:n_thru] == 2).sum()) > n_thru // 3


def test_rays_in_a_face_plane_and_origins_inside_on_and_behind(emu):
    cube = S.box_triangles((0.0, 0.0, 8.0), (2.0, 2.0, 2.0), torch.eye(3))
    prims = only_meshes([cube])
    rays = torch.tensor([
        [0.0, 2.0, 0.0, 0.0, 0.0, 1.0],      # in the plane y = 2 of a face
        [-4.0, 2.0, 8.0, 1.0, 0.0, 0.0],     # in that plane, across the face
        [0.5, 0.25, 8.0, 0.0, 0.0, 1.0],     # origin inside
        [0.5, 0.25, 6.0, 0.0, 0.0, 1.0],     # origin on the entry face
        [0.5, 0.25, 10.0, 0.0, 0.0, 1.0],    # origin on the exit face, looking out
        [0.5, 0.25, 14.0, 0.0, 0.0, 1.0],    # the mesh behind the origin
        [0.5, 0.25, 14.0, 0.0, 0.0, -1.0],   # ... and in front of it
    ], dtype=torch.float32)
    ref = oracle(rays, prims, 4)
    assert_same(emu_intersect(emu, rays, prims, 4), ref)
    hit, bid, tin, tout = ref
    assert hit.tolist() == [hit[0].item(), hit[1].item(), True, True, False, False, True]
    assert (tin[2, 0].item(), tout[2, 0].item()) == (0.0, 2.0)
    assert (tin[3, 0].item(), tout[3, 0].item()) == (0.0, 4.0)
    assert (tin[6, 0].item(), tout[6, 0].item()) == (4.0, 8.0)


def test_u_extrusion_gives_two_intervals_with_one_id(emu):
    u = S.u_extrusion(0.0, 0.0, 1.0, -1.0, 1.0)
    prims = only_meshes([u])
    rays = torch.tensor([[-2.0, 0.0, 2.0, 1.0, 0.0, 0.0], [-2.0, 0.0, 0.5, 1.0, 0.0, 0.0]], dtype=torch.float32)
    ref = oracle(rays, prims, 4)
    assert_same(emu_intersect(emu, rays, prims, 4), ref)
    assert ref[1][0].tolist() == [0, 0, -1, -1]
    assert ref[2][0, :2].tolist() == [2.0, 4.0] and ref[3][0, :2].tolist() == [3.0, 5.0]
    assert ref[1][1].tolist() == [0, -1, -1, -1] and (ref[2][1, 0].item(), ref[3][1, 0].item()) == (2.0, 5.0)


@pytest.mark.parametrize("M", range(1, 9))
def test_more_intervals_than_slots(emu, M):
    """A comb of 10 teeth in front of a second one: 20 intervals on the ray, of which the M nearest are kept - from
    the inside of a tooth, from in front of the comb and from behind its first teeth."""
    combs = [comb(10), comb(10, -1.0, 1.0)]
    combs[1] = combs[1] + torch.tensor([0.5, 0.0, 0.0])            # interleaved teeth of a second primitive
    prims = only_meshes(combs)
    rays = torch.tensor([[-3.0, 0.0, 2.0, 1.0, 0.0, 0.0], [0.5, 0.25, 2.0, 1.0, 0.0, 0.0],
                         [6.25, 0.0, 2.0, 1.0, 0.0, 0.0], [-3.0, 0.0, 2.5, 1.0, 0.0, 0.0]], dtype=torch.float32)
    ref = oracle(rays, prims, M)
    assert_same(emu_intersect(emu, rays, prims, M), ref)
    assert bool((ref[1] >= 0).all())                                   # every slot taken
    assert bool((ref[2][:, 1:] >= ref[2][:, :-1]).all())
    full = oracle(rays, prims, 8)
    assert torch.equal(ref[1], full[1][:, :M]) and torch.equal(ref[2], full[2][:, :M])


# ------------------------------------------------------------------------------------------ against exact geometry
def _inside_exact(mesh, p):
    """Exact point-in-polyhedron (rational parity of a ray in a direction that meets no edge or vertex)."""
    P = [Fraction(x) for x in p]
    T = [[[Fraction(float(c)) for c in v] for v in t] for t in mesh.tolist()]
    rng = np.random.default_rng(0)
    while True:
        d = [Fraction(int(x), 1000003) for x in rng.integers(-1000, 1000, 3)]
        n, ok = 0, True
        for a, b, c in T:
            e1 = [b[i] - a[i] for i in range(3)]
            e2 = [c[i] - a[i] for i in range(3)]
            h = [d[1] * e2[2] - d[2] * e2[1], d[2] * e2[0] - d[0] * e2[2], d[0] * e2[1] - d[1] * e2[0]]
            det = sum(e1[i] * h[i] for i in range(3))
            if det == 0:
                continue                                              # parallel: no crossing (a hit would be in-plane)
            s = [P[i] - a[i] for i in range(3)]
            u = sum(s[i] * h[i] for i in range(3)) / det
            q = [s[1] * e1[2] - s[2] * e1[1], s[2] * e1[0] - s[0] * e1[2], s[0] * e1[1] - s[1] * e1[0]]
            v = sum(d[i] * q[i] for i in range(3)) / det
            t = sum(e2[i] * q[i] for i in range(3)) / det
            if u < 0 or v < 0 or u + v > 1 or t < 0:
                continue
            if u == 0 or v == 0 or u + v == 1 or t == 0:
                ok = False
                break
            n += 1
        if ok:
            return n % 2 == 1


@pytest.mark.parametrize("which", ["u", "ellipsoid", "comb"])
def test_interval_midpoints_are_inside_and_gaps_outside(emu, which):
    g = torch.Generator().manual_seed(5)
    if which == "u":
        mesh = S.u_extrusion(-3.0, 6.0, 2.0, -2.0, 2.0)
    elif which == "ellipsoid":
        mesh = S.icosphere_ellipsoid((0.5, 0.0, 10.0), (3.0, 2.0, 4.0), yaw=0.4, subdiv=1)
    else:
        mesh = comb(4) + torch.tensor([-3.0, 0.0, 8.0])
    prims = only_meshes([mesh])
    tgt = mesh.reshape(-1, 3).mean(0) + (torch.rand(60, 3, generator=g) - 0.5) * 6.0
    org = torch.tensor([[0.0, 0.0, 0.0]]).expand(60, 3).clone()
    org[40:] = mesh.reshape(-1, 3).mean(0) + (torch.rand(20, 3, generator=g) - 0.5) * 2.0   # some origins inside
    rays = torch.cat([org, tgt - org], 1).contiguous()
    ref = oracle(rays, prims, 8)
    assert_same(emu_intersect(emu, rays, prims, 8), ref)
    checked = 0
    for i in range(rays.shape[0]):
        o, d = rays[i, :3].double(), rays[i, 3:].double()
        iv = [(float(a), float(b)) for a, b, k in zip(ref[2][i], ref[3][i], ref[1][i]) if k >= 0]
        for a, b in iv:
            if b - a > 1e-3:
                assert _inside_exact(mesh, (o + d * (a + b) / 2).tolist()), (i, a, b)
                checked += 1
        for (_, b0), (a1, _) in zip(iv, iv[1:]):
            if a1 - b0 > 1e-3:
                assert not _inside_exact(mesh, (o + d * (a1 + b0) / 2).tolist()), (i, b0, a1)
                checked += 1
        if iv and iv[0][0] > 1e-3:
            assert not _inside_exact(mesh, (o + d * iv[0][0] / 2).tolist())
        if iv and iv[-1][1] < 1e3:
            assert not _inside_exact(mesh, (o + d * (iv[-1][1] + 1.0)).tolist()) or which == "comb"
    assert checked >= 20


def test_cuboid_as_12_triangles_matches_the_slab_test(emu):
    bx = S.make_boxes(24, seed=4)
    rays = S.make_rays(make_cfg("cfg2"), rows=40, row0=160)[::7].contiguous()
    meshes = [S.box_triangles(bx["box_center"][b], bx["box_half"][b], bx["box_rot"][b]) for b in range(24)]
    prims = only_meshes(meshes)
    o, d = rays[:, :3], rays[:, 3:]
    tmin, tmax, hit = O.slab_test(o, d, bx["box_center"], bx["box_half"], bx["box_rot"])
    _, _, hit_in = O.slab_test(o, d, bx["box_center"], bx["box_half"] * 0.995, bx["box_rot"])
    _, _, hit_out = O.slab_test(o, d, bx["box_center"], bx["box_half"] * 1.005, bx["box_rot"])
    clear = (hit_in == hit_out).all(1)            # no ray passes near an edge of any box
    assert int(clear.sum()) > 500
    ref = oracle(rays[clear].contiguous(), prims, 8)
    assert_same(emu_intersect(emu, rays[clear].contiguous(), prims, 8), ref)
    cub = O.intersect(o[clear], d[clear], bx["box_center"], bx["box_half"], bx["box_rot"], 8)
    assert torch.equal(ref[0], cub[0]) and torch.equal(ref[1], cub[1])
    v = cub[1] >= 0
    for a, b in ((ref[2], cub[2]), (ref[3], cub[3])):
        assert bool(((a - b).abs()[v] <= 8 * torch.finfo(torch.float32).eps * b.abs()[v].clamp(min=1.0)).all())


# ------------------------------------------------------------------------------------------ reader
def _obj(name, transform, verts, faces=None, sem=7, inst=100):
    m = lambda tag, a, t="f": (f"<{tag} type_id=\"opencv-matrix\"><rows>{a.shape[0]}</rows><cols>{a.shape[1]}</cols>"
                               f"<dt>{t}</dt><data>{' '.join(repr(float(x)) if t == 'f' else str(int(x)) for x in a.reshape(-1))}</data></{tag}>")
    f = m("faces", np.asarray(faces), "i") if faces is not None else ""
    return (f"<{name}>{m('transform', np.asarray(transform, dtype=np.float64))}{m('vertices', np.asarray(verts, dtype=np.float64))}"
            f"{f}<semanticId>{sem}</semanticId><instanceId>{inst}</instanceId><timestamp>-1</timestamp><dynamic>0</dynamic></{name}>")


def _write(tmp_path, objs):
    p = tmp_path / "boxes.xml"
    p.write_text('<?xml version="1.0"?>\n<opencv_storage>' + "".join(objs) + "</opencv_storage>\n")
    return p


def _cuboid_vf():
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
    t = S.box_triangles((0.0, 0.0, 0.0), (0.5, 0.5, 0.5), torch.eye(3)).reshape(-1, 3).numpy().astype(np.float64)
    f = np.array([[int(np.where((v == t[3 * k + j]).all(1))[0][0]) for j in range(3)] for k in range(12)])
    return v, f


def _ell_vf():
    m = S.icosphere_ellipsoid((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), subdiv=1).reshape(-1, 3).numpy().astype(np.float64)
    v, f = np.unique(m, axis=0, return_inverse=True)
    return v, f.reshape(-1, 3)


def _tf(scale=(4.0, 2.0, 1.5), yaw=0.3, t=(10.0, -2.0, 5.0), shear=0.0):
    c, s = np.cos(yaw), np.sin(yaw)
    A = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]) @ np.diag(scale)
    A[0, 1] += shear
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = A, t
    return T


def test_reader_splits_cuboids_and_meshes(tmp_path):
    cv, cf = _cuboid_vf()
    ev, ef = _ell_vf()
    objs = [_obj("object1", _tf(), cv, cf),                  # a cuboid (faces too: it stays a cuboid)
            _obj("object2", _tf(yaw=1.0), ev, ef, sem=11),    # an ellipsoid
            _obj("object3", _tf(shear=0.7), cv, cf),          # a sheared cuboid: a mesh with the world AABB
            _obj("object4", _tf(), cv)]                       # a cuboid without faces
    boxes = K.parse_bboxes_xml(_write(tmp_path, objs))
    assert boxes[0].faces.shape == (12, 3) and boxes[3].faces is None
    pr = K.boxes_to_primitives(boxes, meshes=True)
    start = pr["mesh_tri_start"]
    assert start.tolist() == [0, 0, ef.shape[0], ef.shape[0] + 12, ef.shape[0] + 12]
    assert pr["mesh_tris"].shape == (ef.shape[0] + 12, 3, 3) and pr["mesh_tris"].dtype == np.float32
    assert np.array_equal(pr["box_rot"][2], np.eye(3, dtype=np.float32))
    for b in (1, 2):
        tri = pr["mesh_tris"][start[b]:start[b + 1]].reshape(-1, 3).astype(np.float64)
        loc = (tri - pr["box_center"][b].astype(np.float64)) @ pr["box_rot"][b].astype(np.float64)
        assert np.all(np.abs(loc) <= pr["box_half"][b].astype(np.float64)), b
    wv = boxes[1].world_vertices().astype(np.float32)
    assert np.array_equal(pr["mesh_tris"][start[1]:start[2]], wv[boxes[1].faces])
    ref = K.boxes_to_primitives(boxes[:1] + boxes[3:])
    for k in ("box_center", "box_half", "box_rot"):
        assert np.array_equal(pr[k][[0, 3]], ref[k])
    bt = K.primitive_batch(pr, device="cpu")
    assert bt["mesh_tri_start"].dtype == torch.int32 and bt["mesh_tris"].shape == pr["mesh_tris"].shape
    assert "mesh_tris" not in K.primitive_batch(ref, device="cpu")


def test_reader_refusals_name_the_object(tmp_path):
    cv, cf = _cuboid_vf()
    ev, ef = _ell_vf()
    open_f = ef[:-1]
    for obj, needle in ((_obj("object9", _tf(), ev), "needs <faces>"),
                        (_obj("object9", _tf(), ev, ef + 1), "outside [0"),
                        (_obj("object9", _tf(), ev, open_f), "open or non-manifold"),
                        (_obj("object9", _tf(), ev, np.concatenate([ef, ef[:1]])), "open or non-manifold")):
        boxes = K.parse_bboxes_xml(_write(tmp_path, [_obj("object1", _tf(), cv, cf), obj]))
        with pytest.raises(ValueError, match="object9") as e:
            K.boxes_to_primitives(boxes, meshes=True)
        assert needle in str(e.value)


def test_reader_without_meshes_is_unchanged(tmp_path):
    cv, cf = _cuboid_vf()
    ev, ef = _ell_vf()
    boxes = K.parse_bboxes_xml(_write(tmp_path, [_obj("object1", _tf(), cv, cf), _obj("object2", _tf(yaw=1.0), ev, ef)]))
    a = K.boxes_to_primitives(boxes)
    stripped = [KB.Box3D(b.name, b.transform, b.vertices, b.semantic_id, b.instance_id, b.timestamp, b.dynamic)
                for b in boxes]
    b = K.boxes_to_primitives(stripped)
    assert set(a) == {"box_center", "box_half", "box_rot", "box_sem", "box_inst", "names"}
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])) if k != "names" else a[k] == b[k]
    assert K.boxes_to_primitives(boxes[:1], meshes=True).keys() == a.keys()          # cuboids only: no table
    prims = {k: v for k, v in a.items()}
    key = KC._key(prims, np.eye(4), (1.0, 1.0, 0.5, 0.5), 4, 4, 2)
    assert key == KC._key(K.boxes_to_primitives(boxes[:2], meshes=False), np.eye(4), (1.0, 1.0, 0.5, 0.5), 4, 4, 2)
    m = K.boxes_to_primitives(boxes, meshes=True)
    assert KC._key(m, np.eye(4), (1.0, 1.0, 0.5, 0.5), 4, 4, 2) != KC._key({**m, "mesh_tris": m["mesh_tris"] + 1},
                                                                          np.eye(4), (1.0, 1.0, 0.5, 0.5), 4, 4, 2)


def test_cache_key_of_cuboid_primitives_is_unchanged():
    import hashlib
    pr = {k: v.numpy() for k, v in S.make_boxes(5).items()}
    h = hashlib.sha256()
    for a in (pr["box_center"], pr["box_half"], pr["box_rot"], np.eye(4, dtype=np.float32),
              np.asarray((1.0, 2.0, 3.0, 4.0), dtype=np.float32), np.array([8, 9, 4, KC._FORMAT], dtype=np.int64)):
        h.update(np.ascontiguousarray(a).tobytes())
    assert KC._key(pr, np.eye(4), (1.0, 2.0, 3.0, 4.0), 8, 9, 4) == h.hexdigest()


# ------------------------------------------------------------------------------------------ C ABI
def _refused(rc, needle):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg, msg


def _call(**kw):
    a = dict(rays=X, R=4, bc=X, bh=X, br=X, start=X, tris=X, T=10, B=3, M=4, hit=X, bid=X, tin=X, tout=X)
    a.update(kw)
    return _capi.lib().pnr_intersect_meshes(a["rays"], a["R"], a["bc"], a["bh"], a["br"], a["start"], a["tris"], a["T"],
                                            a["B"], a["M"], a["hit"], a["bid"], a["tin"], a["tout"], None)


@pytest.mark.parametrize("kw,needle", [
    ({"start": None}, "mesh_tri_start (null)"), ({"tris": None}, "mesh_tris (null)"), ({"T": 0}, "T=0"),
    ({"start": None, "tris": None}, "T=10"), ({"T": -1}, "T=-1"), ({"T": 1 << 31}, "T=2147483648"),
    ({"M": 0}, "M=0"), ({"M": 9}, "M=9"), ({"B": -1}, "B=-1"), ({"rays": None}, "null pointer"),
    ({"bc": None}, "null box table")])
def test_intersect_meshes_refuses_bad_arguments(kw, needle):
    _refused(_call(**kw), needle)
    assert b"pnr_intersect_meshes" in _capi.lib().pnr_last_error()


def test_pnr_render_args_ctypes_layout_matches_the_header(tmp_path):
    if not shutil.which("g++"):
        pytest.skip("no host compiler")
    fields = [f for f, _ in _capi.PnrRenderArgs._fields_]
    src = tmp_path / "offsets.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(pnr_render_args, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(pnr_render_args));\n  return 0;\n}\n')
    exe = tmp_path / "offsets"
    subprocess.check_call(["g++", "-x", "c++", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got[:-1] == [getattr(_capi.PnrRenderArgs, f).offset for f in fields]
    assert got[-1] == C.sizeof(_capi.PnrRenderArgs)
    assert fields[-3:] == ["mesh_tri_start", "mesh_tris", "T"]
