"""CPU: the PSP-head entry points (``ffb6d_psp_pool``, ``ffb6d_psp_bottleneck_fwd``, ``ffb6d_conv1x1_log_softmax_fwd``)
reject bad sizes, null pointers and a ``final`` wider than one output tile before any launch, and the Python layer
rejects host tensors (there is no CPU path)."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib, ops

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


POOL = dict(x=P, B=8, C=512, H=60, W=80, out=P)
BOTTLE = dict(x=P, B=8, C=512, H=60, W=80, packed=P, bias=P, Co=1024, table=P, out=P)
LSM = dict(x=P, B=8, Ci=64, P=240 * 320, packed=P, bias=P, Co=64, out=P)


def args(base, **kw):
    a = dict(base)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("kw", [dict(B=0), dict(C=0), dict(H=0), dict(W=0), dict(B=-1), dict(H=-6)])
def test_pool_bad_sizes(kw):
    bad("ffb6d_psp_pool", args(POOL, **kw), "bad size")


@pytest.mark.parametrize("kw", [dict(H=1025), dict(W=1 << 24), dict(B=1 << 16, C=1 << 15)])
def test_pool_too_large(kw):
    bad("ffb6d_psp_pool", args(POOL, **kw), "too large")


@pytest.mark.parametrize("kw", [dict(x=None), dict(out=None)])
def test_pool_null(kw):
    bad("ffb6d_psp_pool", args(POOL, **kw), "null pointer")


@pytest.mark.parametrize("kw", [dict(B=0), dict(C=0), dict(H=0), dict(W=0), dict(Co=0), dict(C=-512)])
def test_bottleneck_bad_sizes(kw):
    bad("ffb6d_psp_bottleneck_fwd", args(BOTTLE, **kw), "bad size")


@pytest.mark.parametrize("kw", [dict(B=1 << 16), dict(H=2000, W=1073), dict(B=4096, Co=65536)])
def test_bottleneck_too_large(kw):
    bad("ffb6d_psp_bottleneck_fwd", args(BOTTLE, **kw), "too large")


@pytest.mark.parametrize("kw", [dict(x=None), dict(packed=None), dict(bias=None), dict(table=None), dict(out=None)])
def test_bottleneck_null(kw):
    bad("ffb6d_psp_bottleneck_fwd", args(BOTTLE, **kw), "null pointer")


def test_bottleneck_misaligned_pack():
    bad("ffb6d_psp_bottleneck_fwd", args(BOTTLE, packed=P + 4), "16-byte aligned")


@pytest.mark.parametrize("kw", [dict(B=0), dict(Ci=0), dict(P=0), dict(Co=0), dict(Co=-64)])
def test_log_softmax_bad_sizes(kw):
    bad("ffb6d_conv1x1_log_softmax_fwd", args(LSM, **kw), "bad size")


@pytest.mark.parametrize("co", [129, 256, 1 << 20])
def test_log_softmax_rejects_wide_output(co):
    bad("ffb6d_conv1x1_log_softmax_fwd", args(LSM, Co=co), "at most 128 channels")


@pytest.mark.parametrize("kw", [dict(x=None), dict(packed=None), dict(bias=None), dict(out=None)])
def test_log_softmax_null(kw):
    bad("ffb6d_conv1x1_log_softmax_fwd", args(LSM, **kw), "null pointer")


def test_ops_have_no_cpu_path():
    x = torch.zeros(1, 8, 6, 6)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.psp_pool(x)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.conv1x1_log_softmax(x, torch.zeros(8, 8), torch.zeros(8))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.psp_bottleneck(x, None, None)
