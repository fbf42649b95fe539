"""CPU: the training-side entry points of the PSP head and of PSPUpsample (``ffb6d_psp_bottleneck_bwd``,
``ffb6d_psp_pool_bwd``, ``ffb6d_log_softmax_bwd``, ``ffb6d_upsample_bilinear2d_bwd``) reject bad sizes, null pointers
and misaligned pointers before any launch, and their Python wrappers reject host tensors (there is no CPU path)."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib, cnn, ops

_buf = (C.c_double * 64)()
P = C.addressof(_buf)              # fake "device" addresses, 16-byte aligned; no call below reaches a launch


def call(name, *args):
    n0 = _lib.launch_count()
    rc = getattr(_lib.lib, name)(*args, None)
    assert _lib.launch_count() == n0
    return rc


def bad(name, args, text):
    assert call(name, *args) == _lib.ERR_INVALID, args
    assert text in _lib.last_error(), _lib.last_error()


BOTTLE = dict(grad_out=P, out=P, B=8, Co=1024, H=60, W=80, grad_z=P, grad_table=P, grad_sum=P)
POOL = dict(grad_pooled=P, B=8, C=512, H=60, W=80, grad_x=P)
LSM = dict(grad_out=P, out=P, B=8, C=64, P=480 * 640, grad_in=P)
UP = dict(grad_out=P, B=8, C=1024, Hi=60, Wi=80, Ho=120, Wo=160, grad_in=P)
ENTRY = {"ffb6d_psp_bottleneck_bwd": BOTTLE, "ffb6d_psp_pool_bwd": POOL, "ffb6d_log_softmax_bwd": LSM,
         "ffb6d_upsample_bilinear2d_bwd": UP}
POINTERS = {name: [k for k, v in base.items() if v == P] for name, base in ENTRY.items()}
SIZES = {name: [k for k, v in base.items() if v != P] for name, base in ENTRY.items()}


def args(base, **kw):
    a = dict(base)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_bad_sizes(name):
    for k in SIZES[name]:
        for v in (0, -1, -(1 << 40)):
            bad(name, args(ENTRY[name], **{k: v}), "bad size")


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_null_pointers(name):
    for k in POINTERS[name]:
        bad(name, args(ENTRY[name], **{k: None}), "null pointer")


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_misaligned_pointers(name):
    for k in POINTERS[name]:
        bad(name, args(ENTRY[name], **{k: P + 2}), "4-byte aligned")


@pytest.mark.parametrize("kw", [dict(H=1025), dict(W=1025), dict(H=1024, W=1024), dict(B=1 << 16, Co=1 << 15)])
def test_bottleneck_bwd_too_large(kw):
    bad("ffb6d_psp_bottleneck_bwd", args(BOTTLE, **kw), "too large")


@pytest.mark.parametrize("kw", [dict(H=1025), dict(W=16385), dict(B=1 << 16, C=1 << 15)])
def test_pool_bwd_too_large(kw):
    bad("ffb6d_psp_pool_bwd", args(POOL, **kw), "too large")


@pytest.mark.parametrize("kw", [dict(B=1 << 16), dict(P=1 << 38)])
def test_log_softmax_bwd_too_large(kw):
    bad("ffb6d_log_softmax_bwd", args(LSM, **kw), "too large")


@pytest.mark.parametrize("kw", [dict(Hi=1 << 24), dict(Wo=1 << 24), dict(B=1 << 20, C=1 << 20)])
def test_upsample_bwd_too_large(kw):
    bad("ffb6d_upsample_bilinear2d_bwd", args(UP, **kw), "too large")


def test_ops_have_no_cpu_path():
    x = torch.zeros(1, 8, 6, 6)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.psp_bottleneck_bwd(x, x)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.psp_pool_bwd(torch.zeros(50 * 8), x)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.log_softmax_bwd(x, x)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.upsample_bilinear2d_bwd(x, (3, 3))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.upsample_bilinear2d(x)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        cnn.PSPUpsample(8, 4).forward_fused(x)
