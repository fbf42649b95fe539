"""CPU: ``ffb6d_point_input`` is exported with its header signature and rejects bad arguments before any launch;
``ops.point_input``, ``estimate_poses`` and ``GraphedPoseStep`` reject wrong arguments before any CUDA work."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import ROOT
from ffb6d_b200 import _lib

B, H, W, N = 2, 8, 10, 100


def _buf(nbytes=1 << 16):
    b = (C.c_double * (nbytes // 8))()
    return b, C.addressof(b)


_keep, P = _buf()


def call(**kw):
    a = dict(depth=P, B=B, H=H, W=W, intr=P, per_frame=0, choose=P, N=N, rgb=P, nrm=P, out=P)
    a.update(kw)
    return _lib.lib.ffb6d_point_input(a["depth"], a["B"], a["H"], a["W"], a["intr"], a["per_frame"], a["choose"],
                                      a["N"], a["rgb"], a["nrm"], a["out"], None)


def test_symbol_and_signature():
    assert "ffb6d_point_input" in _lib.SYMBOLS
    text = re.sub(r"\s+", " ", open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read())
    assert ("int ffb6d_point_input(const float *depth_m, int64_t B, int64_t H, int64_t W, const double *intrinsics, "
            "int intrinsics_per_frame, const int *choose, int64_t N, const uint8_t *rgb, const float *nrm, "
            "float *cld_rgb_nrm, ffb6d_stream_t stream);") in text
    fn = _lib.lib.ffb6d_point_input
    assert fn.restype is C.c_int
    assert fn.argtypes == [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_int64,
                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]


@pytest.mark.parametrize("kw", [dict(B=-1), dict(B=65536), dict(H=0), dict(W=0), dict(H=1 << 16, W=1 << 15),
                                dict(N=-1), dict(N=1 << 31)])
def test_bad_sizes(kw):
    assert call(**kw) == _lib.ERR_INVALID
    assert "point_input: bad size" in _lib.last_error()


def test_intrinsics_per_frame_flag():
    assert call(per_frame=2) == _lib.ERR_INVALID
    assert "intrinsics_per_frame" in _lib.last_error()


@pytest.mark.parametrize("name", ["depth", "intr", "choose", "rgb", "nrm", "out"])
def test_null_pointers(name):
    assert call(**{name: None}) == _lib.ERR_INVALID
    assert "point_input: null pointer" in _lib.last_error()


@pytest.mark.parametrize("name,off", [("intr", 4), ("depth", 2), ("choose", 2), ("nrm", 1), ("out", 2)])
def test_misaligned_pointers(name, off):
    assert call(**{name: P + off}) == _lib.ERR_INVALID
    assert "point_input: misaligned" in _lib.last_error()


def test_empty_batch_or_points_is_a_no_op():
    nulls = {k: None for k in ("depth", "intr", "choose", "rgb", "nrm", "out")}
    assert call(B=0, **nulls) == _lib.OK
    assert call(N=0, **nulls) == _lib.OK


def _args(**kw):
    a = dict(depth_m=torch.zeros(B, H, W), K=torch.eye(3, dtype=torch.float64).numpy(),
             choose=torch.zeros(B, 1, N, dtype=torch.int32), rgb=torch.zeros(B, H, W, 3, dtype=torch.uint8),
             nrm_map=torch.zeros(B, H, W, 3))
    a.update(kw)
    return a


@pytest.mark.parametrize("kw", [
    dict(depth_m=torch.zeros(B, H, W, dtype=torch.float64)), dict(depth_m=torch.zeros(H, W)),
    dict(choose=torch.zeros(B, 1, N, dtype=torch.float32)), dict(choose=torch.zeros(B, 2, N, dtype=torch.int32)),
    dict(choose=torch.zeros(B + 1, N, dtype=torch.int32)), dict(rgb=torch.zeros(B, H, W, 3, dtype=torch.int32)),
    dict(rgb=torch.zeros(B, 3, H, W, dtype=torch.uint8)), dict(nrm_map=torch.zeros(B, H, W, 3, dtype=torch.float16)),
    dict(nrm_map=torch.zeros(B, H, W, 4)),
])
def test_point_input_rejects_dtype_and_shape(kw):
    import ffb6d_b200 as F
    with pytest.raises(ValueError):
        F.point_input(**_args(**kw))


def test_point_input_needs_cuda_tensors():
    import ffb6d_b200 as F
    with pytest.raises(RuntimeError, match="CUDA"):
        F.point_input(**_args())
    with pytest.raises(TypeError):
        F.point_input(**_args(nrm_map=None))


# ------------------------------------------------------------------------------------------ estimate_poses
def _frames(**kw):
    f = dict(dpt=torch.zeros(B, H, W, dtype=torch.uint16), rgb=torch.zeros(B, H, W, 3, dtype=torch.uint8),
             nrm_map=torch.zeros(B, H, W, 3))
    f.update(kw)
    return {k: v for k, v in f.items() if v is not None}


def _estimate(frames, dataset="ycb"):
    import ffb6d_b200 as F
    return F.estimate_poses(None, frames, dataset=dataset, cam_scale=10000.0, K=torch.eye(3).numpy(), mesh_kps={})


@pytest.mark.parametrize("dataset", ["YCB", "lm", None, "occlusion_linemod"])
def test_estimate_rejects_unknown_dataset(dataset):
    with pytest.raises(ValueError, match="dataset"):
        _estimate(_frames(), dataset)


@pytest.mark.parametrize("frames,what", [
    (_frames(dpt=None), "lack"), (_frames(rgb=None), "lack"), (_frames(nrm_map=None), "lack"),
    (dict(_frames(), labels=torch.zeros(B, H, W, dtype=torch.uint8)), "unknown"),
    ([torch.zeros(1)], "must be a dict"), (_frames(rgb=torch.zeros(B, H, W, 3).numpy()), "must be a tensor"),
    (_frames(dpt=torch.zeros(B, H, W, dtype=torch.int32)), "dpt"), (_frames(dpt=torch.zeros(H, W, dtype=torch.uint16)),
                                                                   "dpt"),
    (_frames(rgb=torch.zeros(B, H, W, 3)), "rgb"), (_frames(rgb=torch.zeros(B, 3, H, W, dtype=torch.uint8)), "rgb"),
    (_frames(nrm_map=torch.zeros(B, H, W, 3, dtype=torch.float16)), "nrm_map"),
    (_frames(nrm_map=torch.zeros(B, H, W + 1, 3)), "nrm_map"),
    (dict(_frames(), K=torch.eye(3).expand(B, 3, 3)), "K"), (dict(_frames(), K=torch.eye(3, dtype=torch.float64)), "K"),
    (_frames(), "CUDA device"),
])
def test_estimate_rejects_frames_before_cuda_work(frames, what):
    with pytest.raises(ValueError, match=what):
        _estimate(frames)


def test_graphed_step_rejects_before_cuda_work():
    import ffb6d_b200 as F
    from ffb6d_b200.model import FFB6DFusionNet
    kw = dict(dataset="ycb", cam_scale=10000.0, K=torch.eye(3).numpy(), mesh_kps={})
    with pytest.raises(ValueError, match="no image branch"):
        F.GraphedPoseStep(FFB6DFusionNet(n_classes=2), _frames(), **kw)
    with pytest.raises(ValueError, match="DataParallel"):
        F.GraphedPoseStep(torch.nn.DataParallel(torch.nn.Linear(1, 1)), _frames(), **kw)
    with pytest.raises(ValueError, match="dataset"):
        F.GraphedPoseStep(FFB6DFusionNet(n_classes=2), _frames(), **dict(kw, dataset="lm"))
