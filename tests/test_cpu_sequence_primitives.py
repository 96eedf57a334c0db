"""CPU tier of sequence tables (DESIGN 3.2): kitti360.sequence_primitives on a synthetic annotation file; the host build of
pnr_intersect_frames (tests/host_emu.cpp) against the per-frame oracle (tests/oracle_sequence.py
over tests/oracle_mesh.py) bit for bit, with empty, shared, clamped and out-of-range frames, ties, overflowing lists
and meshes in the dynamic blocks; the argument refusals of pnr_intersect_frames and pnr_render_fused_frames (before
any CUDA call: the pointers are placeholders that are never dereferenced); the ctypes layouts against the header; and
the sharding of ray_frame."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_mesh as OM
import oracle_sequence as OS
from host_emu import emu  # noqa: F401  (fixture)
from panopticnerf_b200 import _capi, make_cfg, parallel, synthetic as S
from panopticnerf_b200.lib.datasets import kitti360 as K

ROOT = Path(__file__).resolve().parent.parent
X = 64          # a non-null placeholder pointer
ERR_ARG = -1


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------ sequence_primitives
def _obj(name, t, sem, inst, ts, yaw=0.3, size=(4.0, 2.0, 1.5)):
    c, s = np.cos(yaw), np.sin(yaw)
    T = np.eye(4)
    T[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]) @ np.diag(size)
    T[:3, 3] = t
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)])
    m = lambda tag, a: (f"<{tag} type_id=\"opencv-matrix\"><rows>{a.shape[0]}</rows><cols>{a.shape[1]}</cols><dt>f</dt>"
                        f"<data>{' '.join(repr(float(x)) for x in a.reshape(-1))}</data></{tag}>")
    return (f"<{name}>{m('transform', T)}{m('vertices', v)}<semanticId>{sem}</semanticId><instanceId>{inst}</instanceId>"
            f"<timestamp>{ts}</timestamp><dynamic>{int(ts != -1)}</dynamic></{name}>")


def _boxes(tmp_path):
    """Static boxes interleaved with a car moving over timestamps 10..13 and a pedestrian at 11 and 13."""
    objs = [_obj("object1", (0.0, 0.0, 5.0), 7, 100, -1), _obj("object2", (3.0, 1.0, 9.0), 11, 101, -1)]
    for k, ts in enumerate((10, 11, 12, 13)):
        objs.append(_obj(f"object{10 + k}", (2.0 * k, 0.0, 12.0), 26, 200, ts, yaw=0.1 * k))
        if ts in (11, 13):
            objs.append(_obj(f"object{20 + k}", (-1.0, 0.5, 8.0 + k), 24, 300, ts, size=(0.6, 0.6, 1.8)))
    objs.append(_obj("object3", (-4.0, 0.0, 20.0), 8, 102, -1))
    p = tmp_path / "boxes.xml"
    p.write_text('<?xml version="1.0"?>\n<opencv_storage>' + "".join(objs) + "</opencv_storage>\n")
    return K.parse_bboxes_xml(p)


def _rows(prims, idx):
    return {prims["names"][i]: tuple(np.asarray(prims[k][i]).tobytes() for k in OS.PRIM_KEYS) for i in idx}


def test_sequence_table_holds_each_frames_boxes(tmp_path):
    boxes = _boxes(tmp_path)
    frame_ids = [10, 11, 12, 13, 11, 10, 99, -1]      # two cameras share 10 and 11; 99 and -1 have no dynamic boxes
    seq = K.sequence_primitives(boxes, frame_ids)
    static = K.boxes_to_primitives(boxes, frame=None)
    S = seq["static_boxes"]
    assert S == 3 and seq["frame_boxes"].shape == (8, 2) and seq["frame_boxes"].dtype == np.int32
    for k in OS.PRIM_KEYS:
        assert np.array_equal(seq[k][:S], static[k])
    assert seq["names"][:S] == static["names"]
    fb = seq["frame_boxes"]
    for f, fid in enumerate(frame_ids):
        b0, b1 = map(int, fb[f])
        assert S <= b0 <= b1 <= seq["box_center"].shape[0]
        want = K.boxes_to_primitives(boxes, frame=fid)
        got = _rows(seq, list(range(S)) + list(range(b0, b1)))
        assert got == _rows(want, range(want["box_center"].shape[0])), fid
    assert tuple(fb[1]) == tuple(fb[4]) and tuple(fb[0]) == tuple(fb[5])          # shared timestamps share a block
    assert fb[6, 0] == fb[6, 1] and fb[7, 0] == fb[7, 1]                              # no dynamic boxes: empty
    assert int(fb[1, 1] - fb[1, 0]) == 2 and int(fb[2, 1] - fb[2, 0]) == 1
    bt = K.primitive_batch(seq, device="cpu")
    assert bt["static_boxes"] == S and bt["frame_boxes"].dtype == torch.int32
    assert "frame_boxes" not in K.primitive_batch(static, device="cpu")


def test_sequence_table_with_meshes_keeps_each_primitives_triangles(tmp_path):
    from test_cpu_mesh_primitives import _ell_vf, _obj as _mesh_obj, _tf
    ev, ef = _ell_vf()
    objs = [_mesh_obj("object1", _tf(), ev, ef, sem=7).replace("<timestamp>-1", "<timestamp>5"),
            _obj("object2", (0.0, 0.0, 4.0), 11, 101, -1),
            _mesh_obj("object3", _tf(yaw=1.0), ev, ef, sem=9)]
    p = tmp_path / "m.xml"
    p.write_text('<?xml version="1.0"?>\n<opencv_storage>' + "".join(objs) + "</opencv_storage>\n")
    boxes = K.parse_bboxes_xml(p)
    seq = K.sequence_primitives(boxes, [5, 6], meshes=True)
    S, st = seq["static_boxes"], seq["mesh_tri_start"]
    assert S == 2 and st.tolist() == [0, 0, ef.shape[0], 2 * ef.shape[0]] and seq["names"] == ["object2", "object3", "object1"]
    assert seq["frame_boxes"].tolist() == [[2, 3], [3, 3]]
    one = K.boxes_to_primitives(boxes, frame=5, meshes=True)
    for name, b in (("object1", 2), ("object3", 1)):
        i = one["names"].index(name)
        a = one["mesh_tris"][one["mesh_tri_start"][i]:one["mesh_tri_start"][i + 1]]
        assert np.array_equal(seq["mesh_tris"][st[b]:st[b + 1]], a)


# ------------------------------------------------------------------------------------------ host build vs oracle
def emu_frames(emu, rays, prims, S, fb, rf, M):
    R, B = rays.shape[0], prims["box_center"].shape[0]
    hit = torch.zeros(R, dtype=torch.uint8)
    bid = torch.zeros(R, M, dtype=torch.int32)
    tin, tout = torch.zeros(R, M), torch.zeros(R, M)
    mesh = prims.get("mesh_tri_start")
    tris = prims["mesh_tris"].contiguous() if mesh is not None else None
    emu.emu_intersect_frames(_p(rays), C.c_int64(R), _p(prims["box_center"]), _p(prims["box_half"]),
                             _p(prims["box_rot"]), _p(mesh), _p(tris),
                             C.c_int64(tris.shape[0] if mesh is not None else 0), B, S, _p(fb), fb.shape[0], _p(rf),
                             M, _p(hit), _p(bid), _p(tin), _p(tout))
    return hit.bool(), bid, tin, tout


def oracle_one(rays, table, M):
    return OM.intersect(rays[:, :3], rays[:, 3:], table["box_center"], table["box_half"], table["box_rot"], M,
                        table.get("mesh_tri_start"), table.get("mesh_tris"))


def assert_same(a, b):
    for x, y, k in zip(a, b, ("hit_mask", "box_id", "t_in", "t_out")):
        assert torch.equal(x, y), (k, int((x != y).sum()))


def _rays(n, seed):
    rays = S.make_rays(make_cfg("cfg2"), rows=40, row0=180)
    g = torch.Generator().manual_seed(seed)
    return rays[torch.randperm(rays.shape[0], generator=g)[:n]].contiguous()


@pytest.mark.parametrize("S_,M", [(0, 4), (20, 1), (40, 4), (64, 8)])
def test_random_frames_match_the_per_frame_oracle(emu, S_, M):
    prims = S.make_boxes(160, seed=S_)
    F = 12
    fb = OS.random_sequence(prims, S_, F, 40, seed=S_, shared=3)
    fb[0] = torch.tensor([S_, S_])                                       # an empty block
    fb[1] = torch.tensor([S_ - 7, S_ + 9])                               # begins below S: clamped to S
    fb[2] = torch.tensor([150, 175])                                     # ends past B: clamped to B
    fb[3] = torch.tensor([90, 80])                                       # end < begin: empty
    rays = _rays(3000, S_)
    rf = torch.randint(-1, F + 1, (rays.shape[0],), generator=torch.Generator().manual_seed(7), dtype=torch.int32)
    assert bool((rf == -1).any()) and bool((rf == F).any())            # out of range: static only
    ref = OS.per_frame(oracle_one, rays, prims, S_, fb, rf, M)
    got = emu_frames(emu, rays, prims, S_, fb, rf, M)
    assert_same(got, ref)
    assert bool((got[1] >= S_).any()), "no ray reached a dynamic box"
    if M < 8:
        assert bool((got[1] >= 0).all(1).any()), "no list overflowed"
    out = (rf < 0) | (rf >= F)
    assert bool((got[1][out] < S_).all())


def test_a_static_and_a_dynamic_box_tied_at_t_in_keep_the_static_first(emu):
    bx = S.make_boxes(8, seed=2)
    prims = {k: torch.cat([v, v[:3]]).contiguous() for k, v in bx.items()}   # dynamic 8..10 copy static 0..2
    fb = torch.tensor([[8, 11]], dtype=torch.int32)
    rays = _rays(4000, 2)
    rf = torch.zeros(rays.shape[0], dtype=torch.int32)
    got = emu_frames(emu, rays, prims, 8, fb, rf, 8)
    assert_same(got, OS.per_frame(oracle_one, rays, prims, 8, fb, rf, 8))
    ids, tin = got[1], got[2]
    tied = 0
    for b in range(3):
        has = (ids == b).any(1)
        for r in torch.nonzero(has).flatten().tolist():
            ms, md = (ids[r] == b).nonzero()[0, 0], (ids[r] == b + 8).nonzero()
            if md.numel():
                assert ms < md[0, 0] and tin[r, ms] == tin[r, md[0, 0]]
                tied += 1
    assert tied > 20


def test_meshes_in_a_dynamic_block(emu):
    prims = S.make_mesh_primitives(seed=1)          # 64 cuboids, then the meshes 64..68
    B = prims["box_center"].shape[0]
    fb = torch.tensor([[40, B], [60, 66], [64, 64], [66, B]], dtype=torch.int32)
    rays = S.make_rays(make_cfg("cfg2"), rows=24, row0=240)[::3].contiguous()
    rf = torch.arange(rays.shape[0], dtype=torch.int32) % 5 - 1           # -1 .. 3
    for M in (2, 8):
        ref = OS.per_frame(oracle_one, rays, prims, 40, fb, rf, M)
        got = emu_frames(emu, rays, prims, 40, fb, rf, M)
        assert_same(got, ref)
        assert bool((got[1] >= 64).any()), "no ray reached a mesh"


def test_without_frames_it_is_the_static_kernel(emu):
    prims = S.make_mesh_primitives(seed=3)
    B = prims["box_center"].shape[0]
    rays = _rays(1500, 3)
    rf = torch.zeros(rays.shape[0], dtype=torch.int32)
    got = emu_frames(emu, rays, prims, B, torch.tensor([[B, B]], dtype=torch.int32), rf, 4)
    assert_same(got, oracle_one(rays, prims, 4))


# ------------------------------------------------------------------------------------------ C ABI
def _refused(rc, needle, fn):
    msg = _capi.lib().pnr_last_error()
    assert rc == ERR_ARG, (rc, msg)
    assert needle.encode() in msg and fn.encode() in msg, msg


def _frames_args(**kw):
    a = _capi.PnrIntersectFramesArgs(rays=X, R=4, box_center=X, box_half=X, box_rot=X, B=10, M=4, hit_mask=X,
                                     box_id=X, t_in=X, t_out=X)
    a.frames.ray_frame, a.frames.frame_boxes, a.frames.F, a.frames.S = X, X, 3, 5
    for k, v in kw.items():
        if k in ("ray_frame", "frame_boxes", "F", "S"):
            setattr(a.frames, k, v)
        else:
            setattr(a, k, v)
    return a


FRAME_REFUSALS = [({"F": -1}, "F=-1"), ({"ray_frame": None}, "ray_frame (null)"),
                  ({"frame_boxes": None}, "frame_boxes (null)"), ({"S": -1}, "S=-1 outside [0, B=10]"),
                  ({"S": 11}, "S=11 outside"), ({"F": 0}, "F=0 (no frame table)"),
                  ({"F": 0, "ray_frame": None, "frame_boxes": None}, "S=5")]


@pytest.mark.parametrize("kw,needle", FRAME_REFUSALS + [
    ({"M": 9}, "M=9"), ({"T": 3}, "mesh_tri_start (null)"), ({"rays": None}, "null pointer"),
    ({"box_rot": None}, "null box table")])
def test_intersect_frames_refuses_bad_arguments(kw, needle):
    _refused(_capi.lib().pnr_intersect_frames(C.byref(_frames_args(**kw)), None), needle, "pnr_intersect_frames")


def test_intersect_frames_refuses_a_null_args_struct():
    _refused(_capi.lib().pnr_intersect_frames(None, None), "null args", "pnr_intersect_frames")


@pytest.mark.parametrize("kw,needle", FRAME_REFUSALS + [({"B": 0, "S": 0}, "F=3 without primitives (B=0)")])
def test_render_fused_frames_refuses_bad_frame_fields(kw, needle):
    a = _capi.PnrRenderArgs(rays=X, R=4, B=10, M=4, N=8)
    fr = _capi.PnrFrameTable(ray_frame=X, frame_boxes=X, F=3, S=5)
    for k, v in kw.items():
        setattr(a if k == "B" else fr, k, v)
    _refused(_capi.lib().pnr_render_fused_frames(X, None, C.byref(a), C.byref(fr), None), needle,
             "pnr_render_fused_frames")


@pytest.mark.parametrize("struct,cls", [("pnr_frame_table", "PnrFrameTable"),
                                        ("pnr_intersect_frames_args", "PnrIntersectFramesArgs"),
                                        ("pnr_ray_batch_args", "PnrRayBatchArgs")])
def test_ctypes_layouts_match_the_header(tmp_path, struct, cls):
    if not shutil.which("g++"):
        pytest.skip("no host compiler")
    T = getattr(_capi, cls)
    fields = [f for f, _ in T._fields_]
    src = tmp_path / "offsets.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pnr.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof({struct}, {f}));\n' for f in fields)
                   + f'  printf("%zu\\n", sizeof({struct}));\n  return 0;\n}}\n')
    exe = tmp_path / "offsets"
    subprocess.check_call(["g++", "-x", "c++", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(T, f).offset for f in fields] + [C.sizeof(T)]
    if cls == "PnrRayBatchArgs":
        assert fields[-1] == "frame"


# ------------------------------------------------------------------------------------------ sharding
def test_shard_training_batch_slices_ray_frame():
    R, G = 10, 3
    batch = {"rays": torch.randn(R, 6), "ray_frame": torch.arange(R, dtype=torch.int32),
             "frame_boxes": torch.tensor([[4, 6], [6, 6]], dtype=torch.int32), "static_boxes": 4}
    for g in range(G):
        lo, hi = parallel.shard_range(R, g, G)
        sh = parallel.shard_training_batch(batch, g, G)
        assert torch.equal(sh["ray_frame"], batch["ray_frame"][lo:hi])
        assert sh["frame_boxes"] is batch["frame_boxes"] and sh["static_boxes"] == 4
        assert torch.equal(parallel.shard_batch(batch, g, G)["ray_frame"], batch["ray_frame"][lo:hi])
    with pytest.raises(ValueError, match="ray_frame"):
        parallel.shard_training_batch(dict(batch, ray_frame=torch.zeros(R - 1, dtype=torch.int32)), 0, G)
