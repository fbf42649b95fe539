"""CPU: the batched voting entry point (``ffb6d_vote_poses``) refuses bad arguments before any launch, its limits
are the header's, and its workspace depends on the sizes only; ``VoteTable`` builds the reference's refinement
thresholds."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from ffb6d_b200 import _lib
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, last_error

MAX_POINTS, MAX_CLASSES, MAX_KPS, MAX_SETS, MAX_SLOTS = (1 << 24) - 1, 1024, 64, 1 << 24, 2 ** 31 - 1


def test_header_limits():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()
    got = {k: eval(v) for k, v in re.findall(r"#define FFB6D_VOTE_(\w+) (.+)", text)}
    assert got == dict(MAX_POINTS=MAX_POINTS, MAX_CLASSES=MAX_CLASSES, MAX_KPS=MAX_KPS, MAX_SETS=MAX_SETS,
                       MAX_SLOTS=MAX_SLOTS)
    assert (_lib.VOTE_MAX_POINTS, _lib.VOTE_MAX_CLASSES, _lib.VOTE_MAX_KPS, _lib.VOTE_MAX_SETS,
            _lib.VOTE_MAX_SLOTS) == (MAX_POINTS, MAX_CLASSES, MAX_KPS, MAX_SETS, MAX_SLOTS)


def test_workspace_bytes():
    ws = lib.ffb6d_vote_poses_workspace_bytes
    big = ws(8, 12288, 22, 8)
    # the packed points (two float4 buffers and their source indices) of n_kps * B * N slots dominate
    assert 8 * 8 * 12288 * 36 < big < 8 * 8 * 12288 * 36 + (4 << 20)
    assert ws(8, 12288, 22, 8) == big and ws(1, 2000, 5, 8) > 0
    assert ws(0, 100, 5, 8) == 0
    for args in ((1, 0, 5, 8), (1, MAX_POINTS + 1, 5, 8), (1, 10, 1, 8), (1, 10, MAX_CLASSES + 1, 8),
                 (1, 10, 5, 0), (1, 10, 5, MAX_KPS + 1), (MAX_SETS // 64 // 64 + 1, 1, 64, 64),
                 (MAX_SLOTS // 8 + 1, 1, 2, 8), (-1, 10, 5, 8)):
        assert ws(*args) == 0, args
    # at the edges the size is computed, without overflow
    assert ws(1, MAX_POINTS, 2, 1) > MAX_POINTS * 36
    assert ws(MAX_SETS // 64 // 64, 1, 64, 64) > MAX_SETS * 32
    assert ws(MAX_SLOTS // 8 // 1024, 1024, 2, 8) > (MAX_SLOTS // 1024) * 1024 * 36


def test_entry_point_checks():
    buf = (C.c_double * 4096)()
    p = C.addressof(buf)
    p = (p + 255) // 256 * 256
    need = lib.ffb6d_vote_poses_workspace_bytes(2, 100, 5, 8)

    def call(pcld=p, mask=p, ctr=p, kp=p, mesh=p, has=p, thr=p, B=2, N=100, C_=5, K=8, use_ctr=1, flt=1, bw=0.04,
             it=300, present=p, count=p, kps=p, poses=p, ws=p, wsb=need):
        return lib.ffb6d_vote_poses(pcld, mask, ctr, kp, mesh, has, thr, B, N, C_, K, use_ctr, flt, bw, it, present,
                                    count, kps, poses, ws, wsb, None)

    cases = [(dict(B=-1), ERR_INVALID, "B >= 0"), (dict(N=0), ERR_INVALID, "N"),
             (dict(N=MAX_POINTS + 1), ERR_INVALID, "N"), (dict(C_=1), ERR_INVALID, "n_cls"),
             (dict(C_=MAX_CLASSES + 1), ERR_INVALID, "n_cls"), (dict(K=0), ERR_INVALID, "n_kps"),
             (dict(K=MAX_KPS + 1), ERR_INVALID, "n_kps"),
             (dict(B=MAX_SETS // 64 // 64 + 1, N=1, C_=64, K=64), ERR_INVALID, "sets"),
             (dict(B=MAX_SLOTS // 8 // 1024 + 1, N=1024, C_=2, K=8), ERR_INVALID, "packed points"),
             (dict(use_ctr=2), ERR_INVALID, "use_ctr"), (dict(flt=-1), ERR_INVALID, "ctr_filter"),
             (dict(bw=0.0), ERR_INVALID, "bandwidth"), (dict(bw=float("inf")), ERR_INVALID, "bandwidth"),
             (dict(bw=float("nan")), ERR_INVALID, "bandwidth"), (dict(it=-1), ERR_INVALID, "max_iter"),
             (dict(ws=p + 16), ERR_INVALID, "256-byte"), (dict(mask=p + 4), ERR_INVALID, "aligned"),
             (dict(poses=p + 4), ERR_INVALID, "aligned"), (dict(pcld=p + 2), ERR_INVALID, "aligned"),
             (dict(ws=None), ERR_WORKSPACE, "workspace"), (dict(wsb=need - 1), ERR_WORKSPACE, "workspace")]
    for name in ("pcld", "mask", "ctr", "kp", "mesh", "has", "present", "count", "kps", "poses"):
        cases.append((dict(**{name: None}), ERR_INVALID, "null"))
    for kw, rc, text in cases:
        assert call(**kw) == rc, kw
        assert text in last_error(), (kw, last_error())
    # B = 0 is a successful no-op, whatever the pointers
    assert call(B=0, pcld=None, mask=None, ctr=None, kp=None, mesh=None, has=None, thr=None, present=None,
                count=None, kps=None, poses=None, ws=None, wsb=0) == 0


def test_vote_table_thresholds():
    """The refinement distance is float32(float64(r) * 0.8), the reference's rounding (not float32(r) * 0.8f)."""
    torch = pytest.importorskip("torch")
    from ffb6d_b200 import pose
    radius = [0.08, 0.12, 0.10, 0.07, 0.06]
    t = pose.VoteTable({1: np.ones((9, 3)), 3: np.zeros((9, 3))}, 5, radius, device="cpu")
    want = np.zeros(5, np.float32)
    want[1:] = (np.asarray(radius[:4], np.float64) * 0.8).astype(np.float32)
    assert np.array_equal(t.refine_thr.numpy(), want)
    assert t.has_mesh.tolist() == [0, 1, 0, 1, 0] and tuple(t.kps.shape) == (5, 9, 3)
    assert tuple(t.rows(8).shape) == (5, 8, 3)
    with pytest.raises(ValueError):
        t.rows(10)
    with pytest.raises(ValueError):
        pose.VoteTable({5: np.ones((9, 3))}, 5, device="cpu")
    with pytest.raises(ValueError):
        pose.VoteTable({1: np.ones((9, 3))}, 5, radius[:3], device="cpu")
    with pytest.raises(ValueError):
        pose.VoteTable({1: np.ones((9, 3)), 2: np.ones((8, 3))}, 5, device="cpu")
    assert pose.VoteTable({1: np.ones((9, 3))}, 5, device="cpu").refine_thr is None
    assert not hasattr(pose, "_vote_object")
