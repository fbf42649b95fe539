"""CPU: the textured rasteriser's entry points (DESIGN.md §4.35) are declared and exported, their limits are the
header's, they refuse bad arguments before any launch; ``TexturedMeshTable`` refuses malformed meshes before any CUDA
work; ``render_rgbd`` and ``textured_kp3ds`` refuse what is neither table; and the training paths keep refusing a
``TexturedMeshTable`` (their ``meshes=`` takes vertex-coloured meshes only)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import ffb6d_b200 as F
from conftest import ROOT
from ffb6d_b200 import _lib, objinfo, render, schedule
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, OK, last_error
from test_abi import declared_symbols
import test_render_abi as RA

_buf = (C.c_double * 4096)()
P = (C.addressof(_buf) + 15) // 16 * 16   # a fake "device" address; no call below reaches a launch


def test_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    for s in ("ffb6d_render_rgbd_textured", "ffb6d_render_texture_mips"):
        assert s in declared_symbols() and s in _lib.SYMBOLS and hasattr(raw, s), s
    assert F.render.TexturedMeshTable is render.TexturedMeshTable
    assert not issubclass(render.TexturedMeshTable, render.RenderMeshTable)
    f = lib.ffb6d_render_rgbd_textured
    assert f.restype is C.c_int and len(f.argtypes) == 30 and f.argtypes[21] is C.c_double
    assert lib.ffb6d_render_texture_mips.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                                     C.c_void_p]


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()

    def define(name):
        return re.search(r"#define FFB6D_RND_%s (.+)" % name, text).group(1).strip()

    assert int(define("MAX_TEX_SIDE")) == _lib.RND_MAX_TEX_SIDE == 16384
    assert int(define("MAX_TEX_LEVELS")) == _lib.RND_MAX_TEX_LEVELS == 15
    assert int(define("MAX_UV")) == _lib.RND_MAX_UV == 1 << 16
    # a chain at the side limit has exactly the level limit's levels
    assert len(render.tex_levels(_lib.RND_MAX_TEX_SIDE, 1)) == _lib.RND_MAX_TEX_LEVELS


def call(B=2, M=2, H=8, W=8, max_verts=16, max_faces=16, n_meshes=1, z_near=0.01, per_frame=0, depth=P + 1024,
         depth_mm=None, ws=P, ws_bytes=None, max_tex_side=64, ptrs=None):
    p = dict(xyz=P, uv=P, faces=P, vert_off=P, face_off=P, tex=P, tex_hw=P, tex_off=P, mesh_idx=P, RTs=P, label=P,
             intr=P, active=None, rgb=P + 2048, labels=P + 3072)
    p.update(ptrs or {})
    if ws_bytes is None:
        ws_bytes = lib.ffb6d_render_workspace_bytes(B, M, H, W, max_verts, max_faces)
    return lib.ffb6d_render_rgbd_textured(p["xyz"], p["uv"], p["faces"], p["vert_off"], p["face_off"], p["tex"],
                                          p["tex_hw"], p["tex_off"], max_tex_side, n_meshes, max_verts, max_faces,
                                          p["mesh_idx"], p["RTs"], p["label"], B, M, p["intr"], per_frame, H, W,
                                          z_near, p["active"], depth, depth_mm, p["rgb"], p["labels"], ws, ws_bytes,
                                          None)


@pytest.mark.parametrize("kw, what", [
    (dict(B=-1), "bad size"), (dict(B=_lib.RND_MAX_FRAMES + 1), "bad size"), (dict(H=0), "bad size"),
    (dict(M=_lib.RND_MAX_SLOTS + 1), "bad size"), (dict(max_faces=0), "bad size"), (dict(n_meshes=0), "n_meshes"),
    (dict(z_near=0.0009), "z_near"), (dict(z_near=float("nan")), "z_near"), (dict(per_frame=2), "intrinsics_per_frame"),
    (dict(max_tex_side=0), "max_tex_side"), (dict(max_tex_side=_lib.RND_MAX_TEX_SIDE + 1), "max_tex_side"),
    (dict(depth=None), "exactly one"), (dict(depth_mm=P + 1024), "exactly one"),
    (dict(ptrs=dict(xyz=None)), "null"), (dict(ptrs=dict(uv=None)), "null"), (dict(ptrs=dict(faces=None)), "null"),
    (dict(ptrs=dict(tex=None)), "null"), (dict(ptrs=dict(tex_hw=None)), "null"),
    (dict(ptrs=dict(tex_off=None)), "null"), (dict(ptrs=dict(rgb=None)), "null"),
    (dict(ptrs=dict(uv=P + 2)), "misaligned"), (dict(ptrs=dict(tex_hw=P + 2)), "misaligned"),
    (dict(ptrs=dict(tex_off=P + 4)), "misaligned"), (dict(ptrs=dict(xyz=P + 2)), "misaligned"),
    (dict(depth=P + 2), "misaligned"), (dict(ws=P + 8), "misaligned"),
])
def test_render_textured_refuses(kw, what):
    n0 = _lib.launch_count()
    assert call(**kw) == ERR_INVALID
    assert what in last_error() and "render_rgbd_textured" in last_error(), last_error()
    assert _lib.launch_count() == n0


def test_workspace_limits_and_empty_batch():
    n0 = _lib.launch_count()
    need = lib.ffb6d_render_workspace_bytes(2, 2, 8, 8, 16, 16)
    assert call(ws_bytes=need - 1) == ERR_WORKSPACE and "workspace" in last_error()
    assert call(ws=None) == ERR_WORKSPACE
    # B = 0: a no-op once the sizes pass, whatever the pointers
    assert call(B=0, depth=None, ws=None, ws_bytes=0, ptrs=dict(xyz=None, uv=None, tex=None, tex_hw=None)) == OK
    assert call(B=0, max_tex_side=0) == ERR_INVALID
    for side in (1, _lib.RND_MAX_TEX_SIDE):            # admitted up to the pointer checks
        assert call(max_tex_side=side, ptrs=dict(tex=None)) == ERR_INVALID and "null" in last_error()
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("kw, what", [
    (dict(n=0), "n_meshes"), (dict(n=1 << 31), "n_meshes"), (dict(side=0), "max_tex_side"),
    (dict(side=_lib.RND_MAX_TEX_SIDE + 1), "max_tex_side"), (dict(tex=None), "null"), (dict(hw=None), "null"),
    (dict(off=None), "null"), (dict(hw=P + 1), "misaligned"), (dict(off=P + 4), "misaligned"),
])
def test_mips_refuse(kw, what):
    n0 = _lib.launch_count()
    a = dict(tex=P, hw=P, off=P, n=1, side=64)
    a.update(kw)
    assert lib.ffb6d_render_texture_mips(a["tex"], a["hw"], a["off"], a["n"], a["side"], None) == ERR_INVALID
    assert what in last_error() and "render_texture_mips" in last_error(), last_error()
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- the Python surface
def _mesh(V=4, th=4, tw=6):
    xyz = np.zeros((V, 3), np.float32)
    faces = np.array([[0, 1, 2], [1, 2, 3]])
    uv = np.zeros((V, 2), np.float32)
    return xyz, faces, uv, np.zeros((th, tw, 3), np.uint8)


def test_table_refuses_malformed_meshes():
    xyz, faces, uv, tex = _mesh()
    n0 = _lib.launch_count()
    bad = [((xyz, np.array([[0, 1, 4]]), uv, tex), "face indices"), ((xyz, np.array([[0, -1, 2]]), uv, tex),
                                                                     "face indices"),
           ((xyz[:, :2], faces, uv, tex), "xyz"), ((xyz, faces[:, :2], uv, tex), "faces"),
           ((xyz, faces.astype(np.float32), uv, tex), "faces"),
           ((xyz, faces, uv[:3], tex), "uv must be"), ((xyz, faces, uv.astype(np.int32), tex), "uv must be"),
           ((xyz, faces, np.where(np.eye(4, 2) > 0, np.nan, 0.0), tex), "finite"),
           ((xyz, faces, np.full((4, 2), np.inf), tex), "finite"),
           ((xyz, faces, np.full((4, 2), 65536.5), tex), "finite"),
           ((xyz, faces, np.full((4, 2), -70000.0), tex), "finite"),
           ((xyz, faces, uv, np.zeros((4, 6, 4), np.uint8)), "RGBA"),
           ((xyz, faces, uv, tex.astype(np.float32)), "uint8"), ((xyz, faces, uv, tex[:, :, 0]), "uint8"),
           ((xyz, faces, uv, np.zeros((0, 6, 3), np.uint8)), "sides"),
           ((xyz, faces, uv, np.zeros((1, _lib.RND_MAX_TEX_SIDE + 1, 3), np.uint8)), "sides"),
           ((xyz, faces, uv), "must be")]
    for mesh, what in bad:
        with pytest.raises(ValueError, match=what):
            render.TexturedMeshTable([mesh], device="cpu")
    with pytest.raises(ValueError, match="no meshes"):
        render.TexturedMeshTable([], device="cpu")
    with pytest.raises(ValueError, match="list of"):
        render.TexturedMeshTable(_mesh(), device="cpu")
    # at the limits: |uv| = 2^16, a 1 x 16384 texture
    t = render.TexturedMeshTable([(xyz, faces, np.full((4, 2), -65536.0), np.zeros((1, 16384, 3), np.uint8))],
                                 device="cpu")
    assert t.max_tex_side == 16384 and t.tex.numel() == 3 * sum(h * w for h, w in render.tex_levels(1, 16384))
    assert _lib.launch_count() == n0


def test_table_layout():
    xyz, faces, uv, _ = _mesh()
    t = render.TexturedMeshTable([(xyz, faces, uv, np.full((5, 3, 3), 9, np.uint8)),
                                  (xyz[:3], faces[:1], uv[:3], np.full((1, 7, 3), 4, np.uint8))], device="cpu")
    assert len(t) == 2 and t.max_verts == 4 and t.max_faces == 2 and t.max_tex_side == 7
    assert t.tex_hw.tolist() == [[5, 3], [1, 7]]
    # chains: 5x3, 2x1, 1x1 (8 texels in all), then 1x7, 1x3, 1x1; unused slots repeat the last offset
    assert t.tex_off[0].tolist() == [0, 15, 17] + [17] * 12
    assert t.tex_off[1].tolist() == [18, 25, 28] + [28] * 12
    assert t.tex.numel() == 3 * 29 and (t.level(0, 0) == 9).all() and (t.level(1, 0) == 4).all()
    assert t.uv.dtype == F.render.torch.float32 and t.vert_off.tolist() == [0, 4, 7]


def test_render_rgbd_and_kp3ds_refuse():
    xyz, faces, uv, tex = _mesh()
    t = render.TexturedMeshTable([(xyz, faces, uv, tex)], device="cpu")
    n0 = _lib.launch_count()
    RT = np.zeros((1, 1, 3, 4), np.float32)
    lab = np.zeros((1, 1), np.uint8)
    with pytest.raises(ValueError, match="RenderMeshTable"):
        F.render_rgbd([(0, 0, 0)], np.array([[0]]), RT, lab, np.eye(3), 8, 8)
    with pytest.raises(ValueError, match="CUDA device"):
        F.render_rgbd(t, np.array([[0]]), RT, lab, np.eye(3), 8, 8)
    with pytest.raises(ValueError, match="RenderMeshTable or a TexturedMeshTable"):
        objinfo.textured_kp3ds("table", 0)
    with pytest.raises(ValueError, match=r"centre must be \[3\] or \[2,3\]"):
        objinfo.textured_kp3ds(t, [0, 0], radius=[1.0, 1.0], centre=[[0, 0, 0]] * 3)
    with pytest.raises(ValueError, match="centre must be"):
        objinfo.textured_kp3ds(t, 0, radius=1.0, centre=[0, 0])
    assert _lib.launch_count() == n0


def test_centred_poses():
    # the pyrender branch's pose: get_o2c_pose_cv(cam_pose, T(-mean)); no centre keeps the raster_triangle branch's
    r = np.float32(0.12)
    plain = objinfo.sphere_poses(r)
    c = np.array([0.01, -0.02, 0.005])
    got = objinfo.sphere_poses(r, centre=c)
    T = np.eye(4)
    T[:3, 3] = -c
    cams = [objinfo.camera_pose(p) for p in objinfo.camera_positions(3, 3, r / 0.035 * 0.18)]
    assert np.array_equal(got, np.stack([objinfo.o2c_pose(cp) @ T for cp in cams]))
    assert np.array_equal(plain, np.stack([objinfo.o2c_pose(cp, np.eye(4)) for cp in cams]))
    assert np.array_equal(got[:, :3, :3], plain[:, :3, :3])


@pytest.mark.parametrize("entry", ["build_ffb6d_train_item", "GraphedFrameTrainStep"])
def test_train_paths_refuse_a_textured_table(entry):
    f = RA._entries()[entry]
    xyz, faces, uv, tex = _mesh(3)
    t = render.TexturedMeshTable([(xyz, faces[:1], uv, tex)], device="cpu")
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="RenderMeshTable"):
        f(RA._train_batch(), "linemod", t)
    with pytest.raises(ValueError, match="RenderMeshTable"):
        schedule.check_render_batch(RA._train_batch(), "linemod", "x", t, "device")
    assert _lib.launch_count() == n0
