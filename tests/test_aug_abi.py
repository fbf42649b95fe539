"""CPU: the augmentation entry points reject bad arguments before any launch, and the ops reject wrong dtypes and
shapes before touching a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from ffb6d_b200 import _lib, augment as A

B, H, W = 2, 32, 40
_buf = (C.c_double * (1 << 14))()
P = C.addressof(_buf)


def plans(**slots):
    p = np.stack([A.identity_record("ycb")] * B)
    for k, v in slots.items():
        p[:, getattr(A, k)] = v
    return p


def noise_call(plan=None, **kw):
    plan = plans() if plan is None else plan
    a = dict(rgb=P, B=B, H=H, W=W, host=plan.ctypes.data, dev=P, noise=None, out=P + 8, work=P + 16)
    a.update(kw)
    return _lib.lib.ffb6d_rgb_add_noise(a["rgb"], a["B"], a["H"], a["W"], a["host"], a["dev"], 1, a["noise"], a["out"],
                                        a["work"], None)


@pytest.mark.parametrize("kw", [dict(B=-1), dict(B=65536), dict(H=31), dict(W=31), dict(H=1 << 16, W=1 << 15),
                                dict(H=1 << 40, W=1 << 40), dict(H=3 << 61, W=4), dict(H=65535 * 8 + 1, W=32),
                                dict(H=600000, W=32)])
def test_bad_sizes(kw):
    assert noise_call(**kw) == _lib.ERR_INVALID and "bad size" in _lib.last_error()
    if kw.get("H", H) > 65535 * 8 and kw.get("W", W) == 32:     # rows the filters' grid.y cannot hold
        assert "H <= 524280" in _lib.last_error()
    assert _lib.lib.ffb6d_aug_noise_field(1, kw.get("B", B), kw.get("H", H), kw.get("W", W), 0, P, None) \
        == _lib.ERR_INVALID


@pytest.mark.parametrize("name", ["rgb", "host", "dev", "out", "work"])
def test_null_pointers(name):
    assert noise_call(**{name: None}) == _lib.ERR_INVALID and "null pointer" in _lib.last_error()


@pytest.mark.parametrize("name", ["dev", "noise"])
def test_misaligned_doubles(name):
    assert noise_call(**{name: P + 4}) == _lib.ERR_INVALID and "misaligned" in _lib.last_error()


def test_misaligned_host_plan():
    raw = np.zeros(B * A.REC_LEN + 1)
    raw[1:] = plans().ravel()
    assert noise_call(host=raw.ctypes.data + 4) == _lib.ERR_INVALID and "misaligned" in _lib.last_error()


def test_work_must_not_alias():
    assert noise_call(work=P) == _lib.ERR_INVALID and "alias" in _lib.last_error()


@pytest.mark.parametrize("slots,what", [
    (dict(I_VERSION=2), "version"), (dict(I_MOTION_A=31), "motion kernel size"), (dict(I_MOTION_A=2.5), "motion"),
    (dict(I_GAUSS_K=4), "Gaussian kernel size"), (dict(I_GAUSS_K=3), "sum"), (dict(I_HSV=2), "flag"),
    (dict(I_NOISE_SIGMA=-1), "sigma"), (dict(I_S_FACTOR=np.nan), "HSV"), (dict(I_PASS=2), "pass"),
    (dict(I_SHARPEN_K=np.inf), "sharpen")])
def test_bad_records(slots, what):
    assert noise_call(plans(**slots)) == _lib.ERR_INVALID and what in _lib.last_error()


def test_empty_batch_is_a_no_op():
    assert noise_call(B=0, rgb=None, host=None, dev=None, out=None, work=None) == _lib.OK


def back_call(**kw):
    a = dict(ch=1, ds=0, B=B, dpt=P)
    a.update(kw)
    return _lib.lib.ffb6d_add_real_back(P, P, a["dpt"], P, P, a["ch"], P, P, a["ds"], a["B"], H, W, P, P, None)


@pytest.mark.parametrize("kw,what", [(dict(ch=2), "channels"), (dict(ds=2), "dataset"), (dict(B=-1), "bad size"),
                                     (dict(dpt=None), "null"), (dict(dpt=P + 1), "misaligned")])
def test_add_real_back_rejects(kw, what):
    assert back_call(**kw) == _lib.ERR_INVALID and what in _lib.last_error()


def test_noise_field_stage_range():
    assert _lib.lib.ffb6d_aug_noise_field(1, B, H, W, 4, P, None) == _lib.ERR_INVALID


def test_ops_reject_before_the_gpu():
    import ffb6d_b200 as F
    rgb = torch.zeros(B, H, W, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        F.rgb_add_noise(rgb, plans(), 0)
    with pytest.raises(TypeError):
        F.rgb_add_noise(rgb.numpy(), plans(), 0)
    with pytest.raises(ValueError):
        F.add_real_back(rgb, None, None, None, None, None, dataset="coco")
