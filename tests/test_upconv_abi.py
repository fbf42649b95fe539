"""CPU: the entry points of PSPUpsample at the input's resolution (``ffb6d_upconv_taps_fwd``, ``ffb6d_upconv_taps_bwd``,
``ffb6d_prelu_fwd``, ``ffb6d_bn_prelu_bwd``) reject bad sizes, null and misaligned pointers and oversized shapes before
any launch, and their Python wrappers and ``PSPUpsample.forward_restructured`` reject host tensors (there is no CPU
path) and modules the restructured order does not cover."""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from ffb6d_b200 import _lib, cnn, ops

_buf = (C.c_double * 64)()
P = C.addressof(_buf)              # fake "device" addresses, 16-byte aligned; no call below reaches a launch

TAPS_FWD = dict(table=P, B=8, Co=64, co0=0, Cc=28, Hi=240, Wi=320, bias=P, scale=P, shift=P, alpha=P, out=P)
TAPS_BWD = dict(grad_z=P, B=8, Co=64, co0=0, Cc=28, Hi=240, Wi=320, grad_table=P)
PRELU = dict(x=P, n=8 * 64 * 480 * 640, alpha=P, y=P)
BN_PRELU = dict(z=P, grad_y=P, stats=P, B=8, C=64, P=480 * 640, alpha=P, grad_u=P, grad_alpha_part=P)
ENTRY = {"ffb6d_upconv_taps_fwd": TAPS_FWD, "ffb6d_upconv_taps_bwd": TAPS_BWD, "ffb6d_prelu_fwd": PRELU,
         "ffb6d_bn_prelu_bwd": BN_PRELU}
OPTIONAL = {"bias", "scale", "shift", "alpha"} & set(TAPS_FWD)
POINTERS = {name: [k for k, v in base.items() if v == P] for name, base in ENTRY.items()}
SIZES = {name: [k for k, v in base.items() if v != P and k != "co0"] for name, base in ENTRY.items()}


def call(name, *args):
    n0 = _lib.launch_count()
    rc = getattr(_lib.lib, name)(*args, None)
    assert _lib.launch_count() == n0
    return rc


def bad(name, args, text):
    assert call(name, *args) == _lib.ERR_INVALID, args
    assert text in _lib.last_error(), _lib.last_error()


def args(base, **kw):
    a = dict(base)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_bad_sizes(name):
    for k in SIZES[name]:
        for v in (0, -1, -(1 << 40)):
            bad(name, args(ENTRY[name], **{k: v}), "bad size")


@pytest.mark.parametrize("name", ["ffb6d_upconv_taps_fwd", "ffb6d_upconv_taps_bwd"])
@pytest.mark.parametrize("kw", [dict(co0=-1), dict(co0=64), dict(co0=40, Cc=25), dict(Cc=65)])
def test_bad_chunk(name, kw):
    bad(name, args(ENTRY[name], **kw), "bad size")


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_null_pointers(name):
    for k in POINTERS[name]:
        if name == "ffb6d_upconv_taps_fwd" and k in OPTIONAL:
            continue
        bad(name, args(ENTRY[name], **{k: None}), "null pointer")


def test_scale_and_shift_come_together():
    bad("ffb6d_upconv_taps_fwd", args(TAPS_FWD, scale=None), "scale and shift come together")
    bad("ffb6d_upconv_taps_fwd", args(TAPS_FWD, shift=None), "scale and shift come together")


@pytest.mark.parametrize("name", sorted(ENTRY))
def test_misaligned_pointers(name):
    for k in POINTERS[name]:
        bad(name, args(ENTRY[name], **{k: P + 2}), "aligned")


@pytest.mark.parametrize("k", ["stats", "grad_alpha_part"])
def test_bn_prelu_bwd_wide_alignment(k):
    bad("ffb6d_bn_prelu_bwd", args(BN_PRELU, **{k: P + 4}), "aligned")


@pytest.mark.parametrize("name", ["ffb6d_upconv_taps_fwd", "ffb6d_upconv_taps_bwd"])
@pytest.mark.parametrize("kw", [dict(Hi=1 << 23), dict(Wi=1 << 23), dict(B=1 << 16, Co=1 << 15, Cc=1 << 15),
                                dict(B=1 << 12, Co=1 << 12, Cc=1 << 12, Hi=1 << 12, Wi=1 << 12)])
def test_taps_too_large(name, kw):
    bad(name, args(ENTRY[name], **kw), "too large")


def test_prelu_too_large():
    bad("ffb6d_prelu_fwd", args(PRELU, n=1 << 50), "too large")


@pytest.mark.parametrize("kw", [dict(B=1 << 16, C=1 << 15), dict(P=1 << 40)])
def test_bn_prelu_bwd_too_large(kw):
    bad("ffb6d_bn_prelu_bwd", args(BN_PRELU, **kw), "too large")


def test_ops_have_no_cpu_path():
    x = torch.zeros(1, 8, 3, 4)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.upconv_pack(torch.zeros(4, 8, 3, 3))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.upconv_taps_fwd(torch.zeros(1, 9, 3, 4), torch.zeros(1, 1, 6, 8), 0)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.upconv_taps_bwd(torch.zeros(1, 1, 6, 8), 0, 1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.upsample_conv3x3(x, None)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.prelu_(x, torch.zeros(1))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.bn_prelu_bwd(x, x, torch.zeros(8, 4), torch.zeros(1))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        cnn.PSPUpsample(8, 4).forward_restructured(x)


@pytest.mark.parametrize("change", ["scale", "align", "kernel", "padding", "stride", "prelu"])
def test_forward_restructured_rejects_other_modules(change):
    m = cnn.PSPUpsample(8, 4)
    up, conv = m.conv[0], m.conv[1]
    if change == "scale":
        up.scale_factor = 3.0
    elif change == "align":
        up.align_corners = False
    elif change == "kernel":
        m.conv[1] = nn.Conv2d(8, 4, 5, padding=1)
    elif change == "padding":
        conv.padding = (0, 0)
    elif change == "stride":
        conv.stride = (2, 2)
    else:
        m.conv[3] = nn.PReLU(4)
    with pytest.raises(ValueError, match="forward_restructured"):
        m.forward_restructured(torch.zeros(1, 8, 3, 4))
