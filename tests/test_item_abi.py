"""CPU: ``ffb6d_point_item`` rejects bad arguments before any launch, and ``ops.point_item`` rejects wrong dtypes
and shapes before touching a GPU."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib

B, H, W, N, NOBJ, NKPS = 2, 8, 10, 100, 22, 8


def _buf(nbytes=1 << 16):
    b = (C.c_double * (nbytes // 8))()
    return b, C.addressof(b)


_keep, P = _buf()


def call(**kw):
    a = dict(depth=P, B=B, H=H, W=W, intr=P, per_frame=0, choose=P, N=N, rgb=P, labels=P, nrm=P, cls=P, kps=P,
             ctr=P, n_obj=NOBJ, n_kps=NKPS, out_cld=P, out_lab=P, out_kp=P, out_ctr=P)
    a.update(kw)
    return _lib.lib.ffb6d_point_item(a["depth"], a["B"], a["H"], a["W"], a["intr"], a["per_frame"], a["choose"], a["N"],
                                     a["rgb"], a["labels"], a["nrm"], a["cls"], a["kps"], a["ctr"], a["n_obj"],
                                     a["n_kps"], a["out_cld"], a["out_lab"], a["out_kp"], a["out_ctr"], None)


@pytest.mark.parametrize("kw", [dict(B=-1), dict(B=65536), dict(H=0), dict(W=0), dict(H=1 << 16, W=1 << 15),
                                dict(N=-1), dict(N=1 << 31)])
def test_bad_sizes(kw):
    assert call(**kw) == _lib.ERR_INVALID
    assert "bad size" in _lib.last_error()


@pytest.mark.parametrize("n_kps", [0, -1, 33])
def test_n_kps_out_of_range(n_kps):
    assert call(n_kps=n_kps) == _lib.ERR_INVALID
    assert "n_kps" in _lib.last_error()


@pytest.mark.parametrize("n_obj", [0, -3, 257])
def test_n_obj_out_of_range(n_obj):
    assert call(n_obj=n_obj) == _lib.ERR_INVALID
    assert "n_obj" in _lib.last_error()


def test_intrinsics_per_frame_flag():
    assert call(per_frame=2) == _lib.ERR_INVALID


@pytest.mark.parametrize("name", ["depth", "intr", "choose", "rgb", "labels", "nrm", "cls", "kps", "ctr", "out_cld",
                                  "out_lab", "out_kp", "out_ctr"])
def test_null_pointers(name):
    assert call(**{name: None}) == _lib.ERR_INVALID
    assert "null pointer" in _lib.last_error()


@pytest.mark.parametrize("name,off", [("intr", 4), ("kps", 4), ("ctr", 2), ("depth", 2), ("out_kp", 1),
                                      ("choose", 2)])
def test_misaligned_pointers(name, off):
    assert call(**{name: P + off}) == _lib.ERR_INVALID
    assert "misaligned" in _lib.last_error()


def test_empty_batch_or_points_is_a_no_op():
    nulls = {k: None for k in ("depth", "intr", "choose", "rgb", "labels", "nrm", "cls", "kps", "ctr", "out_cld",
                               "out_lab", "out_kp", "out_ctr")}
    assert call(B=0, **nulls) == _lib.OK
    assert call(N=0, **nulls) == _lib.OK


def _args(**kw):
    a = dict(depth_m=torch.zeros(B, H, W), K=torch.eye(3, dtype=torch.float64).numpy(),
             choose=torch.zeros(B, 1, N, dtype=torch.int32), rgb=torch.zeros(B, H, W, 3, dtype=torch.uint8),
             labels=torch.zeros(B, H, W, dtype=torch.uint8), nrm_map=torch.zeros(B, H, W, 3),
             obj_cls=torch.full((B, NOBJ), -1, dtype=torch.int32),
             obj_kps=torch.zeros(B, NOBJ, NKPS, 3, dtype=torch.float64),
             obj_ctr=torch.zeros(B, NOBJ, 3, dtype=torch.float64))
    a.update(kw)
    return a


@pytest.mark.parametrize("kw", [
    dict(depth_m=torch.zeros(B, H, W, dtype=torch.float64)), dict(depth_m=torch.zeros(H, W)),
    dict(choose=torch.zeros(B, 1, N, dtype=torch.float32)), dict(choose=torch.zeros(B, 2, N, dtype=torch.int32)),
    dict(choose=torch.zeros(B + 1, N, dtype=torch.int32)), dict(choose=torch.zeros(B, 1, 1, N, dtype=torch.int32)),
    dict(rgb=torch.zeros(B, H, W, 3, dtype=torch.int32)), dict(rgb=torch.zeros(B, 3, H, W, dtype=torch.uint8)),
    dict(labels=torch.zeros(B, H, W, dtype=torch.int32)), dict(labels=torch.zeros(B, H, W + 1, dtype=torch.uint8)),
    dict(nrm_map=torch.zeros(B, H, W, 3, dtype=torch.float16)), dict(nrm_map=torch.zeros(B, H, W, 4)),
    dict(obj_cls=torch.zeros(B, NOBJ, dtype=torch.int64)), dict(obj_cls=torch.zeros(B, NOBJ, 1, dtype=torch.int32)),
    dict(obj_kps=torch.zeros(B, NOBJ, NKPS, 3)), dict(obj_kps=torch.zeros(B, NOBJ + 1, NKPS, 3, dtype=torch.float64)),
    dict(obj_kps=torch.zeros(B, NOBJ, NKPS, 2, dtype=torch.float64)),
    dict(obj_ctr=torch.zeros(B, NOBJ, 3)), dict(obj_ctr=torch.zeros(B, NOBJ, 4, dtype=torch.float64)),
])
def test_point_item_rejects_dtype_and_shape(kw):
    import ffb6d_b200 as F
    with pytest.raises(ValueError):
        F.point_item(**_args(**kw))


def test_point_item_needs_cuda_tensors():
    import ffb6d_b200 as F
    with pytest.raises(RuntimeError, match="CUDA"):
        F.point_item(**_args())
    with pytest.raises(TypeError):
        F.point_item(**_args(rgb=None))
