"""CPU: the depth-normal entry points (DESIGN.md §4.30) are declared and exported, their limits are the header's, they
refuse bad arguments before any launch and return OK for an empty batch; every Python entry point that takes
``normals`` refuses a bad value, and a normal map given together with ``normals="device"``, before any CUDA work."""
import ctypes as C
import functools
import os
import re

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import ROOT
from ffb6d_b200 import _lib, estimate, evaluate, graphed
from ffb6d_b200._lib import lib, ERR_INVALID, OK, last_error
from ffb6d_b200.model import FFB6D
from test_abi import declared_symbols

_buf = (C.c_double * 1024)()
P = C.addressof(_buf)                 # a fake "device" address; no call below reaches a launch


def test_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    for s in ("ffb6d_depth_normal", "ffb6d_depth_to_mm"):
        assert s in declared_symbols() and s in _lib.SYMBOLS and hasattr(raw, s), s
    assert "depth_normal" in dir(F) and F.depth_normal is F.ops.depth_normal


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()
    assert int(re.search(r"#define FFB6D_NRM_MAX_KSIZE (\d+)", text).group(1)) == _lib.NRM_MAX_KSIZE
    assert int(re.search(r"#define FFB6D_NRM_MAX_FRAMES (\d+)", text).group(1)) == _lib.NRM_MAX_FRAMES
    assert re.search(r"#define FFB6D_NRM_MAX_HEIGHT \(65535 \* 8 - 1\)", text) and _lib.NRM_MAX_HEIGHT == 65535 * 8 - 1
    assert re.search(r"#define FFB6D_NRM_MAX_FRAME_PIXELS 2147483647ll", text)
    assert _lib.NRM_MAX_FRAME_PIXELS == 2 ** 31 - 1


def normal(B=2, H=8, W=8, depth=P, intr=P + 64, per_frame=1, k=5, dist=2000, diff=20, into=0, out=P + 128):
    return lib.ffb6d_depth_normal(depth, B, H, W, intr, per_frame, k, dist, diff, into, out, None)


@pytest.mark.parametrize("kw, what", [
    (dict(B=-1), "bad size"), (dict(B=_lib.NRM_MAX_FRAMES + 1), "bad size"), (dict(H=0), "bad size"),
    (dict(W=0), "bad size"), (dict(H=_lib.NRM_MAX_HEIGHT + 1, W=1), "bad size"),
    (dict(H=1 << 16, W=1 << 15), "bad size"),
    (dict(k=0), "k_size"), (dict(k=_lib.NRM_MAX_KSIZE + 1), "k_size"), (dict(k=-5), "k_size"),
    (dict(dist=0), "distance_threshold"), (dict(dist=65537), "distance_threshold"),
    (dict(diff=0), "difference_threshold"), (dict(diff=65536), "difference_threshold"),
    (dict(per_frame=2), "intrinsics_per_frame"), (dict(into=2), "point_into_surface"),
    (dict(depth=None), "null"), (dict(intr=None), "null"), (dict(out=None), "null"),
    (dict(depth=P + 1), "misaligned"), (dict(intr=P + 4), "misaligned"), (dict(out=P + 2), "misaligned"),
])
def test_depth_normal_refuses(kw, what):
    n0 = _lib.launch_count()
    assert normal(**kw) == ERR_INVALID
    assert what in last_error(), last_error()
    assert _lib.launch_count() == n0


def test_depth_normal_limits_admitted_and_empty_batch():
    n0 = _lib.launch_count()
    # B = 0 is a no-op, with null pointers; the limits themselves are admitted up to the pointer checks
    assert normal(B=0, depth=None, intr=None, out=None) == OK
    for kw in (dict(k=1), dict(k=_lib.NRM_MAX_KSIZE), dict(dist=1), dict(dist=65536), dict(diff=1), dict(diff=65535),
               dict(B=_lib.NRM_MAX_FRAMES), dict(H=_lib.NRM_MAX_HEIGHT, W=1), dict(H=1, W=_lib.NRM_MAX_FRAME_PIXELS)):
        assert normal(**dict(kw, depth=None)) == ERR_INVALID and "null" in last_error(), kw
    assert normal(B=0, k=0) == ERR_INVALID          # argument checks come before the empty-batch return
    assert _lib.launch_count() == n0


def test_depth_to_mm_refuses():
    n0 = _lib.launch_count()
    f = lib.ffb6d_depth_to_mm
    assert f(None, 0, 10.0, None, None) == OK
    for args, what in (((P, -1, 10.0, P + 64), "bad size"), ((P, 8, 0.0, P + 64), "divisor"),
                       ((P, 8, float("inf"), P + 64), "divisor"), ((P, 8, float("nan"), P + 64), "divisor"),
                       ((P, 8, -1.0, P + 64), "divisor"), ((None, 8, 10.0, P + 64), "null"),
                       ((P, 8, 10.0, None), "null"), ((P + 2, 8, 10.0, P + 64), "misaligned"),
                       ((P, 8, 10.0, P + 65), "misaligned")):
        assert f(*args, None) == ERR_INVALID and what in last_error(), (args, last_error())
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------- the Python surface
B, H, W = 2, 16, 20
BAD = ("host", "", None, 1, "Device", ("device",))


def _frames():
    return {"dpt": torch.zeros((B, H, W), dtype=torch.uint16), "rgb": torch.zeros((B, H, W, 3), dtype=torch.uint8),
            "nrm_map": torch.zeros((B, H, W, 3))}


def _objects():
    return {"RTs": torch.zeros((B, 2, 3, 4)), "kp_3ds": torch.zeros((B, 2, 8, 3)), "ctr_3ds": torch.zeros((B, 2, 3)),
            "cls_ids": torch.zeros((B, 2, 1), dtype=torch.int32), "obj_cls": torch.zeros((B, 2), dtype=torch.int32),
            "obj_kps": torch.zeros((B, 2, 8, 3), dtype=torch.float64),
            "obj_ctr": torch.zeros((B, 2, 3), dtype=torch.float64)}


def _train_batch():
    b = dict(_frames(), labels=torch.zeros((B, H, W), dtype=torch.uint8), back_rgb=torch.zeros((B, H, W, 3)),
             back_labels=torch.zeros((B, H, W)), back_dpt=torch.zeros((B, H, W)), jitter=np.zeros((B, 8)),
             jittered=np.zeros(B, bool), plans=np.zeros((B, 2, 4)), augment=np.zeros(B, bool),
             apply_rgb=np.zeros(B, bool))
    b.update(_objects())
    return b


@functools.lru_cache(maxsize=None)
def _models():
    return FFB6D(n_classes=2, n_pts=64, n_kps=8).eval(), FFB6D(n_classes=2, n_pts=64, n_kps=8)


def _calls():
    """Every entry point taking ``normals``, as ``f(normals, with_nrm_map)``, on CPU tensors: each must fail on the
    normals argument before it looks at the devices."""
    model, train_model = _models()
    opt = torch.optim.Adam(train_model.parameters(), capturable=True)
    K = np.eye(3)
    fr = _frames()
    labels = torch.zeros((B, H, W), dtype=torch.uint8)
    test_kw = dict(dataset="ycb", cam_scale=1e4, K=K, mesh_pts={1: [[0, 0, 0]]}, mesh_kps={}, capacity=4)
    pose_kw = dict(dataset="ycb", cam_scale=1e4, K=K, mesh_kps={})

    def frames(nrm):
        return fr if nrm else {k: v for k, v in fr.items() if k != "nrm_map"}

    def test_batch(nrm):
        return dict(frames(nrm), labels=labels, **_objects())

    def train_batch(nrm):
        b = _train_batch()
        if not nrm:
            del b["nrm_map"]
        return b

    return {
        "build_ffb6d_inputs": lambda n, nrm: F.build_ffb6d_inputs(fr["dpt"], 1e4, K, fr["rgb"],
                                                                  fr["nrm_map"] if nrm else None, 64, normals=n),
        "build_ffb6d_item": lambda n, nrm: F.build_ffb6d_item(fr["dpt"], 1e4, K, fr["rgb"], labels,
                                                              fr["nrm_map"] if nrm else None, _objects(), 64,
                                                              normals=n),
        "build_ffb6d_train_item": lambda n, nrm: F.build_ffb6d_train_item(train_batch(nrm), dataset="ycb",
                                                                          cam_scale=1e4, K=K, n_points=64, seed=0,
                                                                          normals=n),
        "estimate_poses": lambda n, nrm: estimate.estimate_poses(model, frames(nrm), normals=n, **pose_kw),
        "GraphedPoseStep": lambda n, nrm: estimate.GraphedPoseStep(model, frames(nrm), normals=n, **pose_kw),
        "GraphedTestStep": lambda n, nrm: evaluate.GraphedTestStep(model, test_batch(nrm), normals=n, **test_kw),
        "GraphedFrameTrainStep": lambda n, nrm: graphed.GraphedFrameTrainStep(
            train_model, opt, train_batch(nrm), dataset="ycb", cam_scale=1e4, K=K, normals=n),
    }


@pytest.mark.parametrize("entry", ["build_ffb6d_inputs", "build_ffb6d_item", "build_ffb6d_train_item",
                                   "estimate_poses", "GraphedPoseStep", "GraphedTestStep", "GraphedFrameTrainStep"])
def test_normals_refused_before_cuda_work(entry):
    call = _calls()[entry]
    n0 = _lib.launch_count()
    for bad in BAD:
        for nrm in (True, False):
            with pytest.raises(ValueError, match="normals must be 'input' or 'device'"):
                call(bad, nrm)
    with pytest.raises(ValueError, match="nrm_map .*normals='device'"):
        call("device", True)
    # the accepted combinations get past the normals check and fail later, on the CPU tensors
    for n, nrm in (("device", False), ("input", True)):
        with pytest.raises((ValueError, RuntimeError, TypeError)) as e:
            call(n, nrm)
        assert "normals" not in str(e.value), (n, str(e.value))
    assert _lib.launch_count() == n0


def test_default_still_needs_nrm_map():
    fr = {k: v for k, v in _frames().items() if k != "nrm_map"}
    with pytest.raises(ValueError, match="lacks"):
        estimate.estimate_poses(_models()[0], fr, dataset="ycb", cam_scale=1e4,
                                K=np.eye(3), mesh_kps={})
    b = _train_batch()
    del b["nrm_map"]
    with pytest.raises(ValueError, match="lacks"):
        F.build_ffb6d_train_item(b, dataset="ycb", cam_scale=1e4, K=np.eye(3), n_points=64, seed=0)
