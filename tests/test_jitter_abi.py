"""CPU: ffb6d_color_jitter rejects bad arguments before any launch, and ops.color_jitter rejects host tensors."""
import ctypes as C

import numpy as np
import pytest
import torch

from ffb6d_b200 import _lib, augment as A

B, H, W = 2, 5, 7
_buf = (C.c_double * (1 << 14))()
P = C.addressof(_buf)                 # a fake "device" address; no call below reaches a launch
FAR = P + 8 * 8192                    # a second fake address, far from P's B*H*W*3 bytes


def plans(order=(0, 1, 2, 3), factors=(1.1, 0.9, 1.0, 0.01)):
    return np.tile(np.array(list(order) + list(factors), np.float64), (B, 1))


def call(plan=None, **kw):
    plan = plans() if plan is None else plan
    a = dict(rgb=P, B=B, H=H, W=W, host=plan.ctypes.data, dev=FAR, active=FAR + 256, out=P, work=FAR + 512)
    a.update(kw)
    n0 = _lib.launch_count()
    rc = _lib.lib.ffb6d_color_jitter(a["rgb"], a["B"], a["H"], a["W"], a["host"], a["dev"], a["active"], a["out"],
                                     a["work"], None)
    assert _lib.launch_count() == n0
    return rc


@pytest.mark.parametrize("kw", [dict(B=0), dict(B=-1), dict(B=65536), dict(H=0), dict(W=0), dict(H=-3),
                                dict(H=1 << 20), dict(W=1 << 20), dict(H=1 << 16, W=1 << 15),
                                dict(H=1 << 40, W=1 << 40), dict(H=3 << 61, W=4)])
def test_bad_sizes(kw):
    assert call(**kw) == _lib.ERR_INVALID and "bad size" in _lib.last_error()


@pytest.mark.parametrize("name", ["rgb", "host", "dev", "active", "out", "work"])
def test_null_pointers(name):
    assert call(**{name: None}) == _lib.ERR_INVALID and "null pointer" in _lib.last_error()


@pytest.mark.parametrize("name", ["dev", "work"])
def test_misaligned(name):
    assert call(**{name: {"dev": FAR, "work": FAR + 512}[name] + 4}) == _lib.ERR_INVALID
    assert "misaligned" in _lib.last_error()


def test_misaligned_host_plan():
    raw = np.zeros(B * A.JITTER_PLAN_LEN + 1)
    raw[1:] = plans().ravel()
    assert call(host=raw.ctypes.data + 4) == _lib.ERR_INVALID and "misaligned" in _lib.last_error()


def test_work_must_not_alias_the_images():
    assert call(work=P + 8) == _lib.ERR_INVALID and "alias" in _lib.last_error()
    assert call(out=FAR, work=FAR + 16) == _lib.ERR_INVALID and "alias" in _lib.last_error()


def test_out_overlapping_rgb_partially():
    assert call(out=P + 3) == _lib.ERR_INVALID and "overlap" in _lib.last_error()


@pytest.mark.parametrize("order", [(0, 1, 2, 2), (0, 0, 0, 0), (1, 2, 3, 4), (-1, 1, 2, 3), (0.5, 1, 2, 3),
                                   (np.nan, 1, 2, 3), (3, 2, 1, np.inf)])
def test_order_must_be_a_permutation(order):
    assert call(plans(order=order)) == _lib.ERR_INVALID and "order" in _lib.last_error()


@pytest.mark.parametrize("factors,what", [
    ((np.nan, 1, 1, 0), "finite"), ((1, np.inf, 1, 0), "finite"), ((1, 1, -1e-9, 0), ">= 0"),
    ((1e39, 1, 1, 0), "finite"), ((1, 1, 1, 0.5000001), "hue"), ((1, 1, 1, -0.51), "hue"), ((1, 1, 1, np.nan), "hue")])
def test_bad_factors(factors, what):
    assert call(plans(factors=factors)) == _lib.ERR_INVALID and what in _lib.last_error()


def test_bad_plan_in_a_later_frame_names_it():
    p = plans()
    p[1, 7] = 0.7
    assert call(p) == _lib.ERR_INVALID and "frame 1" in _lib.last_error()


def test_ops_reject_before_the_gpu():
    import ffb6d_b200 as F
    rgb = torch.zeros(B, H, W, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA"):
        F.color_jitter(rgb, plans())
    with pytest.raises(TypeError):
        F.color_jitter(rgb.numpy(), plans())
