"""CPU: the loss entry points reject bad arguments before any launch, and the Python layer rejects what it cannot
run (host tensors, unsupported alpha, normalize=False)."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib

B, Cn, N, K = 2, 22, 300, 8
_buf = (C.c_double * (1 << 14))()
P = C.addressof(_buf)                 # fake "device" addresses 16-byte aligned; no call below reaches a launch
WS = _lib.lib.ffb6d_loss_workspace_bytes(B, N, K)


def focal_fwd(**kw):
    a = dict(logits=P, layout=0, labels=P, is64=0, valid=None, B=B, C=Cn, N=N, gamma=2.0, alpha=None, avg=1,
             loss=P, acc=P + 4, count=P + 8, lse=P, ws=P, ws_bytes=WS)
    a.update(kw)
    n0 = _lib.launch_count()
    rc = _lib.lib.ffb6d_focal_loss_fwd(a["logits"], a["layout"], a["labels"], a["is64"], a["valid"], a["B"], a["C"],
                                       a["N"], a["gamma"], a["alpha"], a["avg"], a["loss"], a["acc"], a["count"],
                                       a["lse"], a["ws"], a["ws_bytes"], None)
    assert _lib.launch_count() == n0
    return rc


def focal_bwd(**kw):
    a = dict(logits=P, layout=0, labels=P, is64=0, valid=None, B=B, C=Cn, N=N, gamma=2.0, alpha=None, avg=1,
             lse=P, count=P + 8, g=P, grad=P)
    a.update(kw)
    n0 = _lib.launch_count()
    rc = _lib.lib.ffb6d_focal_loss_bwd(a["logits"], a["layout"], a["labels"], a["is64"], a["valid"], a["B"], a["C"],
                                       a["N"], a["gamma"], a["alpha"], a["avg"], a["lse"], a["count"], a["g"],
                                       a["grad"], None)
    assert _lib.launch_count() == n0
    return rc


def of_fwd(**kw):
    a = dict(pred=P, targ=P, labels=P, is64=0, valid=None, B=B, K=K, N=N, out=P, count=P, ws=P, ws_bytes=WS)
    a.update(kw)
    n0 = _lib.launch_count()
    rc = _lib.lib.ffb6d_of_l1_loss_fwd(a["pred"], a["targ"], a["labels"], a["is64"], a["valid"], a["B"], a["K"],
                                       a["N"], a["out"], a["count"], a["ws"], a["ws_bytes"], None)
    assert _lib.launch_count() == n0
    return rc


def of_bwd(**kw):
    a = dict(pred=P, targ=P, labels=P, is64=0, valid=None, B=B, K=K, N=N, count=P, g=P, grad=P)
    a.update(kw)
    n0 = _lib.launch_count()
    rc = _lib.lib.ffb6d_of_l1_loss_bwd(a["pred"], a["targ"], a["labels"], a["is64"], a["valid"], a["B"], a["K"],
                                       a["N"], a["count"], a["g"], a["grad"], None)
    assert _lib.launch_count() == n0
    return rc


FOCAL = (focal_fwd, focal_bwd)
OF = (of_fwd, of_bwd)


def bad(call, kw, text):
    assert call(**kw) == _lib.ERR_INVALID, kw
    assert text in _lib.last_error(), _lib.last_error()


def test_workspace_bytes():
    assert WS >= B * 3 * 16 and WS % 16 == 0
    assert _lib.lib.ffb6d_loss_workspace_bytes(B, N, 32) > WS
    for args in ((0, N, K), (65536, N, K), (B, 0, K), (B, N, 0), (B, N, 33), (B, 1 << 31, K)):
        assert _lib.lib.ffb6d_loss_workspace_bytes(*args) == 0, args


@pytest.mark.parametrize("kw", [dict(B=0), dict(B=65536), dict(N=0), dict(N=-1), dict(N=1 << 31), dict(C=0),
                                dict(C=257), dict(C=-3)])
@pytest.mark.parametrize("call", FOCAL)
def test_focal_bad_sizes(call, kw):
    bad(call, kw, "bad size")


@pytest.mark.parametrize("kw,text", [(dict(layout=2), "layout"), (dict(layout=-1), "layout"),
                                     (dict(is64=2), "labels_is_i64"), (dict(gamma=float("nan")), "gamma"),
                                     (dict(gamma=float("inf")), "gamma"), (dict(gamma=-0.5), "gamma")])
@pytest.mark.parametrize("call", FOCAL)
def test_focal_bad_arguments(call, kw, text):
    bad(call, kw, text)


@pytest.mark.parametrize("name", ["logits", "labels", "loss", "acc", "count", "lse", "ws"])
def test_focal_fwd_null_pointers(name):
    bad(focal_fwd, {name: None}, "null pointer")


@pytest.mark.parametrize("name", ["logits", "labels", "lse", "count", "g", "grad"])
def test_focal_bwd_null_pointers(name):
    bad(focal_bwd, {name: None}, "null pointer")


@pytest.mark.parametrize("kw", [dict(logits=P + 2), dict(labels=P + 2), dict(labels=P + 4, is64=1), dict(alpha=P + 1),
                                dict(loss=P + 2), dict(count=P + 4), dict(lse=P + 1), dict(ws=P + 8)])
def test_focal_fwd_misaligned(kw):
    bad(focal_fwd, kw, "misaligned")


@pytest.mark.parametrize("kw", [dict(logits=P + 1), dict(count=P + 4), dict(g=P + 2), dict(grad=P + 2),
                                dict(lse=P + 3)])
def test_focal_bwd_misaligned(kw):
    bad(focal_bwd, kw, "misaligned")


def test_focal_short_workspace():
    assert focal_fwd(ws_bytes=16) == _lib.ERR_WORKSPACE and "workspace" in _lib.last_error()


@pytest.mark.parametrize("kw", [dict(B=0), dict(B=65536), dict(N=0), dict(N=1 << 31), dict(K=0), dict(K=33),
                                dict(K=-1)])
@pytest.mark.parametrize("call", OF)
def test_of_bad_sizes(call, kw):
    bad(call, kw, "bad size")


@pytest.mark.parametrize("call", OF)
def test_of_bad_label_type(call):
    bad(call, dict(is64=3), "labels_is_i64")


@pytest.mark.parametrize("name", ["pred", "targ", "labels", "out", "count", "ws"])
def test_of_fwd_null_pointers(name):
    bad(of_fwd, {name: None}, "null pointer")


@pytest.mark.parametrize("name", ["pred", "targ", "labels", "count", "g", "grad"])
def test_of_bwd_null_pointers(name):
    bad(of_bwd, {name: None}, "null pointer")


@pytest.mark.parametrize("kw", [dict(pred=P + 2), dict(targ=P + 1), dict(labels=P + 4, is64=1), dict(out=P + 2),
                                dict(count=P + 1), dict(ws=P + 4)])
def test_of_fwd_misaligned(kw):
    bad(of_fwd, kw, "misaligned")


@pytest.mark.parametrize("kw", [dict(pred=P + 2), dict(targ=P + 1), dict(labels=P + 2), dict(count=P + 1),
                                dict(g=P + 2), dict(grad=P + 3)])
def test_of_bwd_misaligned(kw):
    bad(of_bwd, kw, "misaligned")


def test_of_short_workspace():
    assert of_fwd(ws_bytes=WS // 4) == _lib.ERR_WORKSPACE and "workspace" in _lib.last_error()


def test_python_layer_rejects_before_the_gpu():
    from ffb6d_b200 import loss as L
    x = torch.zeros(2, 22, 10)
    lab = torch.zeros(2, 10, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        L.FocalLoss(gamma=2)(x, lab)
    with pytest.raises(RuntimeError, match="CUDA"):
        L.OFLoss()(torch.zeros(2, 8, 10, 3), torch.zeros(2, 10, 8, 3), lab)
    for alpha in (torch.ones(22), (0.5, 0.5), "0.5", True):
        with pytest.raises(TypeError):
            L.FocalLoss(alpha=alpha)
    assert L.FocalLoss(alpha=0.25).alpha == [0.25, 0.75]
    assert L.FocalLoss(alpha=[1, 2]).alpha == [1.0, 2.0]
    with pytest.raises(NotImplementedError):
        L.of_l1_loss(torch.zeros(2, 8, 10, 3), torch.zeros(2, 10, 8, 3), lab, normalize=False)
