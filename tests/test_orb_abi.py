"""CPU: the ORB entry points (DESIGN.md §4.32) are declared and exported, the header's FFB6D_ORB_* limits equal
``_lib``'s, the capacity and workspace answers follow the layout, and bad arguments are refused before any launch
(by the entry points, and by the Python wrappers with ``ValueError`` before any CUDA work)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import ROOT
from ffb6d_b200 import _lib, objinfo, ops
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, OK
from oracle import orb_oracle as O
from test_abi import declared_symbols

_buf = (C.c_double * 4096)()
P = (C.addressof(_buf) + 15) // 16 * 16       # a fake "device" address; no call below reaches a launch


def test_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    for s in ("ffb6d_orb_capacity", "ffb6d_orb_workspace_bytes", "ffb6d_orb_detect", "ffb6d_orb_lift"):
        assert s in declared_symbols() and s in _lib.SYMBOLS and hasattr(raw, s), s
    assert F.orb_detect is ops.orb_detect and F.orb_lift is ops.orb_lift


def test_limits_match_header():
    with open(os.path.join(ROOT, "include", "ffb6d_b200.h")) as fh:
        text = fh.read()
    for name in ("MAX_FRAMES", "MIN_SIDE", "MAX_SIDE", "LEVELS", "MAX_OBJECTS"):
        m = re.search(r"#define FFB6D_ORB_%s (\S+)" % name, text)
        assert m and int(m.group(1)) == getattr(_lib, "ORB_" + name), name


def caps(H, W):
    return sum(((max(w - 62, 0) + 1) // 2) * ((max(h - 62, 0) + 1) // 2) for h, w in O.level_sizes(H, W))


@pytest.mark.parametrize("hw", [(2, 2), (63, 64), (480, 640), (141, 391), (8192, 8192), (8192, 2)])
def test_capacity_and_workspace(hw):
    H, W = hw
    assert lib.ffb6d_orb_capacity(H, W) == caps(H, W)
    frame = -(-sum(h * w for h, w in O.level_sizes(H, W)) // 16) * 16
    for B in (1, 3, 65535):
        n = lib.ffb6d_orb_workspace_bytes(B, H, W)
        assert n == 3 * B * frame and n % 16 == 0


@pytest.mark.parametrize("B,H,W", [(-1, 8, 8), (65536, 8, 8), (1, 1, 8), (1, 8, 1), (1, 8193, 8), (1, 8, 8193)])
def test_sizes_refused(B, H, W):
    assert lib.ffb6d_orb_workspace_bytes(B, H, W) == 0
    rc = lib.ffb6d_orb_detect(P, B, H, W, P, P, P, P, max(int(lib.ffb6d_orb_capacity(H, W)), 0), P, 1 << 20, None)
    assert rc == ERR_INVALID


def test_detect_refusals():
    cap = lib.ffb6d_orb_capacity(480, 640)
    assert lib.ffb6d_orb_detect(P, 0, 480, 640, None, None, None, None, cap, None, 0, None) == OK
    assert lib.ffb6d_orb_detect(P, 1, 480, 640, P, P, P, P, cap + 1, P, 1 << 30, None) == ERR_INVALID
    assert lib.ffb6d_orb_detect(None, 1, 480, 640, P, P, P, P, cap, P, 1 << 30, None) == ERR_INVALID
    assert lib.ffb6d_orb_detect(P, 1, 480, 640, P + 1, P, P, P, cap, P, 1 << 30, None) == ERR_INVALID
    assert lib.ffb6d_orb_detect(P, 1, 480, 640, P, P, P, P, cap, P + 8, 1 << 30, None) == ERR_INVALID
    need = lib.ffb6d_orb_workspace_bytes(1, 480, 640)
    assert lib.ffb6d_orb_detect(P, 1, 480, 640, P, P, P, P, cap, P, need - 1, None) == ERR_WORKSPACE


def test_lift_refusals():
    cap = lib.ffb6d_orb_capacity(48, 64)
    ok = (P, P, cap, P, 6, 48, 64, P, 0, P, 3, P, P, None)
    assert lib.ffb6d_orb_lift(*ok[:4], 0, *ok[5:]) == OK
    for i, v in ((2, cap + 1), (10, 4), (10, 0), (8, 2), (0, None), (9, P + 4), (1, P + 2)):
        a = list(ok)
        a[i] = v
        assert lib.ffb6d_orb_lift(*a) == ERR_INVALID, (i, v)


def test_python_refusals():
    with pytest.raises(ValueError):
        ops.orb_detect(torch.zeros((1, 8, 8, 3), dtype=torch.float32))
    with pytest.raises(ValueError):
        ops.orb_detect(np.zeros((1, 8, 8, 3), np.uint8))
    with pytest.raises(ValueError):
        objinfo.textured_kp3ds(object(), 0)
