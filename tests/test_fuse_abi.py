"""CPU: the fuse compositor's entry point (DESIGN.md §4.34) is declared and exported, its limits are the header's and
``_lib``'s alike, it refuses bad arguments before any launch and returns OK for an empty batch; ``fuse_rgbd`` refuses
the same sizes first; the training paths refuse ``crops=`` with YCB or with the batch's normal map, fuse keys without
``crops=`` (and ``crops=`` without the keys), a batch without a per-frame ``K``, wrong dtypes and shapes, host crop
indices outside the table and frames flagged both rendered and fused, before any CUDA work."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import ROOT
from ffb6d_b200 import _lib, fuse_frames, graphed, render
from ffb6d_b200._lib import lib, ERR_INVALID, OK, last_error
from ffb6d_b200.model import FFB6D
from test_abi import declared_symbols

_buf = (C.c_double * 4096)()
P = C.addressof(_buf)                 # a fake "device" address; no call below reaches a launch
P = (P + 15) // 16 * 16


def test_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    assert "ffb6d_fuse_rgbd" in declared_symbols() and "ffb6d_fuse_rgbd" in _lib.SYMBOLS
    assert hasattr(raw, "ffb6d_fuse_rgbd")
    assert "fuse_rgbd" in dir(F) and F.fuse_rgbd is fuse_frames.fuse_rgbd
    assert F.fuse_frames.FuseCropTable is fuse_frames.FuseCropTable


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()

    def define(name):
        return re.search(r"#define FFB6D_FUSE_%s (.+)" % name, text).group(1).strip()

    assert int(define("MAX_FRAMES")) == _lib.FUSE_MAX_FRAMES == 65535
    assert define("MAX_FRAME_PIXELS") == "2147483647ll" and _lib.FUSE_MAX_FRAME_PIXELS == 2 ** 31 - 1
    assert int(define("MAX_SLOTS")) == _lib.FUSE_MAX_SLOTS and _lib.FUSE_MAX_SLOTS >= 64
    assert define("MAX_CROPS") == "2147483647ll" and _lib.FUSE_MAX_CROPS == 2 ** 31 - 1


def call(B=2, M=2, H=8, W=8, n_crops=1, ptrs=None):
    p = dict(rgb=P, dpt=P, sil=P, off=P, hw=P, crop=P, offset=P, label=P, active=None, dpt_mm=P + 1024,
             out_rgb=P + 2048, labels=P + 3072)
    p.update(ptrs or {})
    return lib.ffb6d_fuse_rgbd(p["rgb"], p["dpt"], p["sil"], p["off"], p["hw"], n_crops, p["crop"], p["offset"],
                               p["label"], B, M, H, W, p["active"], p["dpt_mm"], p["out_rgb"], p["labels"], None)


@pytest.mark.parametrize("kw, what", [
    (dict(B=-1), "bad size"), (dict(B=_lib.FUSE_MAX_FRAMES + 1), "bad size"), (dict(H=0), "bad size"),
    (dict(W=0), "bad size"), (dict(H=-1, W=-1), "bad size"), (dict(H=1 << 16, W=1 << 15), "bad size"),
    (dict(H=1, W=_lib.FUSE_MAX_FRAME_PIXELS + 1), "bad size"), (dict(M=0), "bad size"),
    (dict(M=_lib.FUSE_MAX_SLOTS + 1), "bad size"), (dict(n_crops=0), "n_crops"),
    (dict(n_crops=_lib.FUSE_MAX_CROPS + 1), "n_crops"),
    (dict(ptrs=dict(rgb=None)), "null"), (dict(ptrs=dict(dpt=None)), "null"), (dict(ptrs=dict(sil=None)), "null"),
    (dict(ptrs=dict(off=None)), "null"), (dict(ptrs=dict(hw=None)), "null"), (dict(ptrs=dict(crop=None)), "null"),
    (dict(ptrs=dict(offset=None)), "null"), (dict(ptrs=dict(label=None)), "null"),
    (dict(ptrs=dict(dpt_mm=None)), "null"), (dict(ptrs=dict(out_rgb=None)), "null"),
    (dict(ptrs=dict(labels=None)), "null"),
    (dict(ptrs=dict(dpt=P + 1)), "misaligned"), (dict(ptrs=dict(off=P + 4)), "misaligned"),
    (dict(ptrs=dict(hw=P + 2)), "misaligned"), (dict(ptrs=dict(crop=P + 2)), "misaligned"),
    (dict(ptrs=dict(offset=P + 2)), "misaligned"), (dict(ptrs=dict(dpt_mm=P + 1)), "misaligned"),
])
def test_fuse_refuses(kw, what):
    n0 = _lib.launch_count()
    assert call(**kw) == ERR_INVALID
    assert what in last_error(), last_error()
    assert _lib.launch_count() == n0


def test_limits_admitted_and_empty_batch():
    n0 = _lib.launch_count()
    assert call(B=0, ptrs=dict(rgb=None, dpt_mm=None, labels=None)) == OK
    assert call(B=0, M=0) == ERR_INVALID                  # size checks come before the empty-batch return
    for kw in (dict(B=_lib.FUSE_MAX_FRAMES, H=1, W=1), dict(B=1, H=1, W=_lib.FUSE_MAX_FRAME_PIXELS),
               dict(B=1, H=_lib.FUSE_MAX_FRAME_PIXELS, W=1), dict(B=1, H=46340, W=46341),
               dict(M=_lib.FUSE_MAX_SLOTS), dict(n_crops=_lib.FUSE_MAX_CROPS)):
        # admitted up to the pointer checks
        assert call(**dict(kw, ptrs=dict(rgb=None))) == ERR_INVALID and "null" in last_error(), kw
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- the Python surface
def _frames():
    out = []
    for cls in (1, 1, 4):
        m = np.zeros((6, 7), np.uint8)
        m[1:4, 2:6] = 255
        out.append((np.zeros((6, 7, 3), np.uint8), np.zeros((6, 7), np.uint16), m, cls))
    return out


def _table():
    return fuse_frames.FuseCropTable(_frames(), device="cpu")


def test_fuse_rgbd_refuses_what_the_abi_refuses_before_cuda_work():
    t = _table()
    n0 = _lib.launch_count()
    off = np.zeros((1, 2, 2), np.int32)
    lab = np.zeros((1, 2), np.uint8)
    ok = np.zeros((1, 2), np.int32)
    cases = [((t, np.array([[0, 3]]), off, lab, 8, 8), r"crop indices must lie in \[-1, 3\)"),
             ((t, np.array([[-2, 0]]), off, lab, 8, 8), "crop indices"),
             ((t, np.array([0, 1]), off, lab, 8, 8), r"\[B,M\]"),
             ((t, ok, off, lab, 0, 8), "H=0"), ((t, ok, off, lab, 8, 0), "W=0"),
             ((t, ok, off, lab, 1 << 16, 1 << 15), "H W"),
             ((t, np.zeros((1, 0), np.int32), np.zeros((1, 0, 2)), np.zeros((1, 0)), 8, 8), "slots"),
             ((t, np.zeros((1, _lib.FUSE_MAX_SLOTS + 1), np.int32), np.zeros((1, _lib.FUSE_MAX_SLOTS + 1, 2)),
               np.zeros((1, _lib.FUSE_MAX_SLOTS + 1)), 8, 8), "slots"),
             ((t, np.zeros((_lib.FUSE_MAX_FRAMES + 1, 1), np.int32), np.zeros((1, 1, 2)), np.zeros((1, 1)), 1, 1),
              "frames"),
             (([(0, 0, 0)], ok, off, lab, 8, 8), "FuseCropTable")]
    for args, what in cases:
        with pytest.raises(ValueError, match=what):
            F.fuse_rgbd(*args)
    assert _lib.launch_count() == n0


def test_python_limits_match_the_abi():
    """Each size the Python entry point admits, the ABI admits (up to the pointer checks), and one past it both
    refuse."""
    for B, M, H, W in ((_lib.FUSE_MAX_FRAMES, 1, 1, 1), (1, _lib.FUSE_MAX_SLOTS, 1, 1),
                       (1, 1, 1, _lib.FUSE_MAX_FRAME_PIXELS)):
        assert call(B=B, M=M, H=H, W=W, ptrs=dict(rgb=None)) == ERR_INVALID and "null" in last_error()
    for B, M, H, W in ((_lib.FUSE_MAX_FRAMES + 1, 1, 1, 1), (1, _lib.FUSE_MAX_SLOTS + 1, 1, 1),
                       (1, 1, 1, _lib.FUSE_MAX_FRAME_PIXELS + 1)):
        assert call(B=B, M=M, H=H, W=W) == ERR_INVALID and "bad size" in last_error()


# ---------------------------------------------------------------------------------------------- the training paths
B, H, W = 2, 16, 20


def _train_batch(dataset="linemod", fuse_keys=True, crop=None, K=True, nrm_map=False, render_keys=False):
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
    if K:
        b["K"] = np.tile(np.eye(3), (B, 1, 1))
    if fuse_keys:
        b.update(fused=np.array([True, False]),
                 fuse_crop=np.array([[0, 2], [-1, -1]], np.int32) if crop is None else crop,
                 fuse_offset=np.zeros((B, 2, 2), np.int32), fuse_label=np.array([[1, 0], [0, 0]], np.uint8))
    if render_keys:
        b.update(rendered=np.array([True, True]), render_mesh=np.zeros((B, 1), np.int32),
                 render_RTs=np.zeros((B, 1, 3, 4), np.float32), render_label=np.ones((B, 1), np.uint8))
    return b


def _mesh_table():
    return render.RenderMeshTable([(np.zeros((3, 3), np.float32), np.array([[0, 1, 2]]), np.zeros((3, 3), np.uint8))],
                                  device="cpu")


def _entries():
    model = FFB6D(n_classes=2, n_pts=64, n_kps=8)
    opt = torch.optim.Adam(model.parameters(), capturable=True)
    kw = dict(cam_scale=1e3, K=np.eye(3))
    return {
        "build_ffb6d_train_item": lambda batch, dataset, crops, normals="device", meshes=None: F.build_ffb6d_train_item(
            batch, dataset=dataset, n_points=64, seed=0, crops=crops, normals=normals, meshes=meshes, **kw),
        "GraphedFrameTrainStep": lambda batch, dataset, crops, normals="device", meshes=None: graphed.GraphedFrameTrainStep(
            model, opt, batch, dataset=dataset, crops=crops, normals=normals, meshes=meshes, **kw),
    }


def refusal_cases(t, mesh_table):
    """(args, message) of every batch the training paths refuse with crops= or with fuse keys."""
    return [((_train_batch("ycb"), "ycb", t), "YCB ships"),
            ((_train_batch("ycb", fuse_keys=False), "ycb", t), "YCB ships"),
            ((_train_batch(), "linemod", None), "no crops were given"),
            ((_train_batch(fuse_keys=False), "linemod", t), "lacks the fuse keys"),
            ((_train_batch(K=False), "linemod", t), "per-frame K"),
            ((dict(_train_batch(), K=np.eye(3)), "linemod", t), r"batch\['K'\]"),
            ((dict(_train_batch(), K=np.tile(np.eye(3, dtype=np.float32), (B, 1, 1))), "linemod", t), r"batch\['K'\]"),
            ((_train_batch(crop=np.array([[0, 3], [-1, -1]], np.int32)), "linemod", t),
             r"crop indices must lie in \[-1, 3\)"),
            ((_train_batch(crop=np.array([[0, -2], [-1, -1]], np.int32)), "linemod", t), "crop indices"),
            ((_train_batch(crop=np.zeros((B, 2), np.int64)), "linemod", t), "fuse_crop"),
            ((dict(_train_batch(), fused=np.zeros(3, bool)), "linemod", t), "fused"),
            ((dict(_train_batch(), fused=np.zeros(B, np.uint8)), "linemod", t), "fused"),
            ((dict(_train_batch(), fuse_offset=np.zeros((B, 2, 3), np.int32)), "linemod", t), "fuse_offset"),
            ((dict(_train_batch(), fuse_offset=np.zeros((B, 2, 2), np.int64)), "linemod", t), "fuse_offset"),
            ((dict(_train_batch(), fuse_label=np.zeros((B, 3), np.uint8)), "linemod", t), "fuse_label"),
            ((_train_batch(), "linemod", "table"), "FuseCropTable"),
            ((_train_batch(nrm_map=True), "linemod", t, "input"), "crops= needs normals='device'"),
            ((_train_batch(), "linemod", t, "input"), "crops= needs normals='device'"),
            ((_train_batch(render_keys=True), "linemod", t, "device", mesh_table), r"frames \[0\] are flagged both")]


@pytest.mark.parametrize("entry", ["build_ffb6d_train_item", "GraphedFrameTrainStep"])
def test_train_paths_refuse_before_cuda_work(entry):
    f = _entries()[entry]
    t = _table()
    n0 = _lib.launch_count()
    for args, what in refusal_cases(t, _mesh_table()):
        with pytest.raises(ValueError, match=what):
            f(*args)
    # accepted: past the fuse checks, failing later on the CPU tensors
    both_ok = dict(_train_batch(render_keys=True), rendered=np.array([False, True]))
    for args in ((_train_batch(), "linemod", t), (both_ok, "linemod", t, "device", _mesh_table()),
                 (_train_batch(fuse_keys=False, nrm_map=True), "linemod", None, "input"),
                 (_train_batch(fuse_keys=False, K=False), "linemod", None)):
        with pytest.raises((ValueError, RuntimeError, TypeError)) as e:
            f(*args)
        assert "fuse" not in str(e.value) and "crop" not in str(e.value), str(e.value)
    assert _lib.launch_count() == n0
