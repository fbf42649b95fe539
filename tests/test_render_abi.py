"""CPU: the rasteriser's entry points (DESIGN.md §4.31) are declared and exported, their limits are the header's, they
refuse bad arguments before any launch and return OK for an empty batch; the training paths refuse meshes with YCB,
render keys without meshes (and meshes without the keys), meshes with the batch's normal map (``normals="input"``)
and host mesh indices outside the table, before any CUDA work."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import ROOT
from ffb6d_b200 import _lib, graphed, render
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, OK, last_error
from ffb6d_b200.model import FFB6D
from test_abi import declared_symbols

_buf = (C.c_double * 4096)()
P = C.addressof(_buf)                 # a fake "device" address; no call below reaches a launch
P = (P + 15) // 16 * 16


def test_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    for s in ("ffb6d_render_rgbd", "ffb6d_render_workspace_bytes"):
        assert s in declared_symbols() and s in _lib.SYMBOLS and hasattr(raw, s), s
    assert "render_rgbd" in dir(F) and F.render_rgbd is render.render_rgbd
    assert F.render.RenderMeshTable is render.RenderMeshTable


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()

    def define(name):
        return re.search(r"#define FFB6D_RND_%s (.+)" % name, text).group(1).strip()

    assert int(define("MAX_FRAMES")) == _lib.RND_MAX_FRAMES
    assert define("MAX_FRAME_PIXELS") == "2147483647ll" and _lib.RND_MAX_FRAME_PIXELS == 2 ** 31 - 1
    assert int(define("MAX_SLOTS")) == _lib.RND_MAX_SLOTS
    assert define("MAX_MESH_VERTS") == "2147483647ll" and _lib.RND_MAX_MESH_VERTS == 2 ** 31 - 1
    assert define("MAX_FRAME_FACES") == "4294967296ll" and _lib.RND_MAX_FRAME_FACES == 2 ** 32
    assert int(define("GUARD_BAND")) == _lib.RND_GUARD_BAND
    assert int(define("BIG_FACE_PIXELS")) == _lib.RND_BIG_FACE_PIXELS
    assert define("QUEUE_CAP") == "(1 << 20)" and _lib.RND_QUEUE_CAP == 1 << 20
    from oracle import render_oracle
    assert render_oracle.GUARD_BAND == _lib.RND_GUARD_BAND


SIZES = dict(B=2, M=2, H=8, W=8, max_verts=16, max_faces=16)


def call(B=2, M=2, H=8, W=8, max_verts=16, max_faces=16, n_meshes=1, z_near=0.01, per_frame=0, depth=P + 1024,
         depth_mm=None, ws=P, ws_bytes=None, ptrs=None):
    p = dict(xyz=P, vrgb=P, faces=P, vert_off=P, face_off=P, mesh_idx=P, RTs=P, label=P, intr=P, active=None,
             rgb=P + 2048, labels=P + 3072)
    p.update(ptrs or {})
    if ws_bytes is None:
        ws_bytes = lib.ffb6d_render_workspace_bytes(B, M, H, W, max_verts, max_faces)
    return lib.ffb6d_render_rgbd(p["xyz"], p["vrgb"], p["faces"], p["vert_off"], p["face_off"], n_meshes, max_verts,
                                 max_faces, p["mesh_idx"], p["RTs"], p["label"], B, M, p["intr"], per_frame, H, W,
                                 z_near, p["active"], depth, depth_mm, p["rgb"], p["labels"], ws, ws_bytes, None)


@pytest.mark.parametrize("kw, what", [
    (dict(B=-1), "bad size"), (dict(B=_lib.RND_MAX_FRAMES + 1), "bad size"), (dict(H=0), "bad size"),
    (dict(W=0), "bad size"), (dict(H=1 << 16, W=1 << 15), "bad size"), (dict(M=0), "bad size"),
    (dict(M=_lib.RND_MAX_SLOTS + 1), "bad size"), (dict(max_verts=0), "bad size"),
    (dict(max_verts=_lib.RND_MAX_MESH_VERTS + 1), "bad size"), (dict(max_faces=0), "bad size"),
    (dict(M=2, max_faces=(1 << 31) + 1), "bad size"), (dict(M=1, max_faces=(1 << 32) + 1), "bad size"),
    (dict(n_meshes=0), "n_meshes"), (dict(z_near=0.0009), "z_near"), (dict(z_near=float("inf")), "z_near"),
    (dict(z_near=float("nan")), "z_near"), (dict(z_near=-1.0), "z_near"), (dict(per_frame=2), "intrinsics_per_frame"),
    (dict(depth=None), "exactly one"), (dict(depth_mm=P + 1024), "exactly one"),
    (dict(ptrs=dict(xyz=None)), "null"), (dict(ptrs=dict(faces=None)), "null"), (dict(ptrs=dict(intr=None)), "null"),
    (dict(ptrs=dict(rgb=None)), "null"), (dict(ptrs=dict(labels=None)), "null"), (dict(ptrs=dict(label=None)), "null"),
    (dict(ptrs=dict(mesh_idx=None)), "null"), (dict(ptrs=dict(RTs=None)), "null"),
    (dict(ptrs=dict(xyz=P + 2)), "misaligned"), (dict(ptrs=dict(vert_off=P + 4)), "misaligned"),
    (dict(ptrs=dict(intr=P + 4)), "misaligned"), (dict(ptrs=dict(mesh_idx=P + 2)), "misaligned"),
    (dict(depth=P + 2), "misaligned"), (dict(depth=None, depth_mm=P + 1), "misaligned"), (dict(ws=P + 8), "misaligned"),
])
def test_render_refuses(kw, what):
    n0 = _lib.launch_count()
    assert call(**kw) == ERR_INVALID
    assert what in last_error(), last_error()
    assert _lib.launch_count() == n0


def test_workspace_refused_and_sized():
    n0 = _lib.launch_count()
    need = lib.ffb6d_render_workspace_bytes(2, 2, 8, 8, 16, 16)
    assert need == 16 + 2 * 8 * 8 * 8 + 2 * 2 * 16 * 16 + _lib.RND_QUEUE_CAP * 8
    # an odd pixel count: the keys are padded to 16 bytes, so the vertex records after them stay 16-byte aligned
    odd = lib.ffb6d_render_workspace_bytes(1, 2, 481, 641, 16, 16)
    assert odd == 16 + (481 * 641 * 8 + 8) + 2 * 16 * 16 + _lib.RND_QUEUE_CAP * 8 and (481 * 641 * 8 + 8) % 16 == 0
    assert call(ws_bytes=need - 1) == ERR_WORKSPACE and "workspace" in last_error()
    assert call(ws=None) == ERR_WORKSPACE
    assert lib.ffb6d_render_workspace_bytes(-1, 2, 8, 8, 16, 16) == 0
    assert lib.ffb6d_render_workspace_bytes(1, _lib.RND_MAX_SLOTS + 1, 8, 8, 16, 16) == 0
    assert _lib.launch_count() == n0


def test_limits_admitted_and_empty_batch():
    n0 = _lib.launch_count()
    assert call(B=0, depth=None, ws=None, ws_bytes=0, ptrs=dict(xyz=None, rgb=None, labels=None)) == OK
    assert call(B=0, z_near=0.0) == ERR_INVALID           # argument checks come before the empty-batch return
    lim = (dict(B=_lib.RND_MAX_FRAMES, H=1, W=1), dict(B=1, H=1, W=_lib.RND_MAX_FRAME_PIXELS),
           dict(B=1, H=_lib.RND_MAX_FRAME_PIXELS, W=1), dict(M=_lib.RND_MAX_SLOTS, max_faces=1 << 20),
           dict(M=1, max_faces=1 << 32), dict(max_verts=_lib.RND_MAX_MESH_VERTS, M=1, B=1), dict(z_near=0.001))
    for kw in lim:
        assert lib.ffb6d_render_workspace_bytes(*[kw.get(k, v) for k, v in SIZES.items()]) > 0, kw
        # admitted up to the pointer checks
        assert call(**dict(kw, ptrs=dict(xyz=None))) == ERR_INVALID and "null" in last_error(), kw
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- the Python surface
def test_mesh_table_checks_faces_on_the_host():
    xyz, faces, rgb = np.zeros((4, 3), np.float32), np.array([[0, 1, 2], [1, 2, 3]]), np.zeros((4, 3), np.uint8)
    for bad, what in (((xyz, np.array([[0, 1, 4]]), rgb), "face indices"), ((xyz, np.array([[0, -1, 2]]), rgb),
                                                                            "face indices"),
                      ((xyz, faces, rgb.astype(np.int32)), "rgb"), ((xyz[:, :2], faces, rgb), "xyz"),
                      ((xyz, faces[:, :2], rgb), "faces"), ((xyz, faces.astype(np.float32), rgb), "faces")):
        with pytest.raises(ValueError, match=what):
            render.RenderMeshTable([bad], device="cpu")
    with pytest.raises(ValueError, match="no meshes"):
        render.RenderMeshTable([], device="cpu")
    t = _two_meshes()
    assert len(t) == 2 and t.max_verts == 4 and t.max_faces == 2
    assert t.vert_off.tolist() == [0, 4, 7] and t.face_off.tolist() == [0, 2, 3]


def _two_meshes():
    xyz, faces, rgb = np.zeros((4, 3), np.float32), np.array([[0, 1, 2], [1, 2, 3]]), np.zeros((4, 3), np.uint8)
    return render.RenderMeshTable([(xyz, faces, rgb), (xyz[:3], faces[:1], rgb[:3])], device="cpu")


def test_render_rgbd_refuses_before_cuda_work():
    t = _two_meshes()
    n0 = _lib.launch_count()
    RT = np.zeros((1, 2, 3, 4), np.float32)
    lab = np.zeros((1, 2), np.uint8)
    for mesh_idx, what in ((np.array([[0, 2]]), "mesh indices"), (np.array([[-2, 0]]), "mesh indices"),
                           (np.array([0, 1]), r"\[B,M\]")):
        with pytest.raises(ValueError, match=what):
            F.render_rgbd(t, mesh_idx, RT, lab, np.eye(3), 8, 8)
    with pytest.raises(ValueError, match="z_near"):
        F.render_rgbd(t, np.array([[0, 1]]), RT, lab, np.eye(3), 8, 8, z_near=0.0005)
    with pytest.raises(ValueError, match="RenderMeshTable"):
        F.render_rgbd([(0, 0, 0)], np.array([[0, 1]]), RT, lab, np.eye(3), 8, 8)
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- the training paths
B, H, W = 2, 16, 20


def _train_batch(dataset="linemod", render_keys=True, mesh_idx=None, nrm_map=False):
    n_obj = 2 if dataset == "linemod" else 4
    b = {"dpt": torch.zeros((B, H, W), dtype=torch.uint16), "rgb": torch.zeros((B, H, W, 3), dtype=torch.uint8),
         "labels": torch.zeros((B, H, W), dtype=torch.uint8),
         "back_rgb": torch.zeros((B, H, W, 3)), "back_labels": torch.zeros((B, H, W)), "back_dpt": torch.zeros((B, H, W)),
         "jitter": np.zeros((B, 8)), "jittered": np.zeros(B, bool), "plans": np.zeros((B, 2, 4)),
         "augment": np.zeros(B, bool), "apply_rgb": np.zeros(B, bool),
         "RTs": torch.zeros((B, n_obj, 3, 4)), "kp_3ds": torch.zeros((B, n_obj, 8, 3)),
         "ctr_3ds": torch.zeros((B, n_obj, 3)), "cls_ids": torch.zeros((B, n_obj, 1), dtype=torch.int32),
         "obj_cls": torch.zeros((B, n_obj), dtype=torch.int32), "obj_kps": torch.zeros((B, n_obj, 8, 3), dtype=torch.float64),
         "obj_ctr": torch.zeros((B, n_obj, 3), dtype=torch.float64)}
    if nrm_map:
        b["nrm_map"] = torch.zeros((B, H, W, 3))
    if render_keys:
        b.update(rendered=np.array([True, False]),
                 render_mesh=np.zeros((B, 1), np.int32) if mesh_idx is None else mesh_idx,
                 render_RTs=np.zeros((B, 1, 3, 4), np.float32), render_label=np.ones((B, 1), np.uint8))
    return b


def _table():
    return render.RenderMeshTable([(np.zeros((3, 3), np.float32), np.array([[0, 1, 2]]), np.zeros((3, 3), np.uint8))],
                                  device="cpu")


def _entries():
    model = FFB6D(n_classes=2, n_pts=64, n_kps=8)
    opt = torch.optim.Adam(model.parameters(), capturable=True)
    kw = dict(cam_scale=1e3, K=np.eye(3))
    return {
        "build_ffb6d_train_item": lambda batch, dataset, meshes, normals="device": F.build_ffb6d_train_item(
            batch, dataset=dataset, n_points=64, seed=0, meshes=meshes, normals=normals, **kw),
        "GraphedFrameTrainStep": lambda batch, dataset, meshes, normals="device": graphed.GraphedFrameTrainStep(
            model, opt, batch, dataset=dataset, meshes=meshes, normals=normals, **kw),
    }


@pytest.mark.parametrize("entry", ["build_ffb6d_train_item", "GraphedFrameTrainStep"])
def test_train_paths_refuse_before_cuda_work(entry):
    f = _entries()[entry]
    t = _table()
    n0 = _lib.launch_count()
    cases = [((_train_batch("ycb"), "ycb", t), "YCB ships"),
             ((_train_batch("ycb", render_keys=False), "ycb", t), "YCB ships"),
             ((_train_batch(), "linemod", None), "no meshes were given"),
             ((_train_batch(render_keys=False), "linemod", t), "lacks the render keys"),
             ((_train_batch(mesh_idx=np.array([[0], [1]], np.int32)), "linemod", t), r"mesh indices must lie in \[-1, 1\)"),
             ((_train_batch(mesh_idx=np.array([[0], [-2]], np.int32)), "linemod", t), "mesh indices"),
             ((_train_batch(mesh_idx=np.zeros((B, 1), np.int64)), "linemod", t), "render_mesh"),
             ((dict(_train_batch(), rendered=np.zeros(3, bool)), "linemod", t), "rendered"),
             ((dict(_train_batch(), render_RTs=np.zeros((B, 1, 3, 4))), "linemod", t), "render_RTs"),
             ((_train_batch(), "linemod", "table"), "RenderMeshTable"),
             # a rendered frame's normals must come from its own depth: the batch's normal map cannot be its
             ((_train_batch(nrm_map=True), "linemod", t, "input"), "meshes= needs normals='device'"),
             ((_train_batch(), "linemod", t, "input"), "meshes= needs normals='device'")]
    for args, what in cases:
        with pytest.raises(ValueError, match=what):
            f(*args)
    # accepted: past the render checks, failing later on the CPU tensors
    for args in ((_train_batch(), "linemod", t),
                 (_train_batch(render_keys=False, nrm_map=True), "linemod", None, "input"),
                 (_train_batch(render_keys=False), "linemod", None)):
        with pytest.raises((ValueError, RuntimeError, TypeError)) as e:
            f(*args)
        assert "render" not in str(e.value) and "mesh" not in str(e.value), str(e.value)
    assert _lib.launch_count() == n0
