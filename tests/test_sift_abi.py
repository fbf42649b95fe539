"""CPU: the SIFT entry points (DESIGN.md §4.33) are declared and exported, the header's FFB6D_SIFT_* limits equal
``_lib``'s, the capacity and workspace answers follow their formulas, and bad arguments are refused before any launch
(by the entry points with FFB6D_ERR_INVALID, and by the Python wrappers with ``ValueError`` before any CUDA work)."""
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
from oracle import sift_oracle as S
from test_abi import declared_symbols

_buf = (C.c_double * 4096)()
P = (C.addressof(_buf) + 15) // 16 * 16       # a fake "device" address; no call below reaches a launch


def test_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    for s in ("ffb6d_sift_capacity", "ffb6d_sift_workspace_bytes", "ffb6d_sift_detect", "ffb6d_sift_lift"):
        assert s in declared_symbols() and s in _lib.SYMBOLS and hasattr(raw, s), s
    assert F.sift_detect is ops.sift_detect and F.sift_lift is ops.sift_lift


def test_limits_match_header():
    with open(os.path.join(ROOT, "include", "ffb6d_b200.h")) as fh:
        text = fh.read()
    for name in ("MAX_FRAMES", "MIN_SIDE", "MAX_SIDE", "MAX_CAP", "CHUNK", "MAX_COPIES"):
        m = re.search(r"#define FFB6D_SIFT_%s (.+)" % name, text)
        assert m and eval(m.group(1)) == getattr(_lib, "SIFT_" + name), name
    assert _lib.SIFT_MAX_COPIES == S.MAX_COPIES


def frame_bytes(H, W):
    """One frame's workspace: 6 Gaussian, 5 DoG and 1 row-pass layers, two 3-layer int arrays, the row counts and
    16 bytes of state, each part on a 16-byte boundary."""
    up = lambda n: -(-n // 16) * 16                               # noqa: E731
    P = 4 * H * W
    return up(12 * P * 4) + 2 * up(3 * P * 4) + up((3 * 2 * H + 1) * 4) + 16


@pytest.mark.parametrize("hw", [(4, 4), (63, 64), (480, 640), (141, 391), (2048, 2048), (2048, 4)])
def test_capacity_and_workspace(hw):
    H, W = hw
    assert lib.ffb6d_sift_capacity(H, W) == max(H * W // 16, 256)
    for B in (1, 3, 16, 17, 65535):
        n = lib.ffb6d_sift_workspace_bytes(B, H, W)
        assert n == min(B, _lib.SIFT_CHUNK) * frame_bytes(H, W) and n % 16 == 0
    assert lib.ffb6d_sift_workspace_bytes(0, H, W) == 0


@pytest.mark.parametrize("B,H,W", [(-1, 8, 8), (65536, 8, 8), (1, 3, 8), (1, 8, 3), (1, 2049, 8), (1, 8, 2049)])
def test_sizes_refused(B, H, W):
    assert lib.ffb6d_sift_workspace_bytes(B, H, W) == 0
    assert lib.ffb6d_sift_detect(P, B, H, W, P, P, P, P, P, P, 256, P, 1 << 30, None) == ERR_INVALID
    assert lib.ffb6d_sift_lift(P, P, 256, P, B, H, W, P, 0, P, 1, P, P, None) == ERR_INVALID


def test_detect_refusals():
    ok = [P, 1, 48, 64, P, P, P, P, P, P, 256, P, 1 << 30, None]
    assert lib.ffb6d_sift_detect(P, 0, 48, 64, None, None, None, None, None, None, 256, None, 0, None) == OK
    for i, v in ((10, -1), (10, _lib.SIFT_MAX_CAP + 1), (0, None), (4, None), (5, None), (9, None), (4, P + 1),
                 (5, P + 2), (6, P + 1), (7, P + 3), (8, P + 1), (9, P + 2), (11, P + 8)):
        a = list(ok)
        a[i] = v
        assert lib.ffb6d_sift_detect(*a) == ERR_INVALID, (i, v)
    need = lib.ffb6d_sift_workspace_bytes(1, 48, 64)
    a = list(ok)
    a[12] = need - 1
    assert lib.ffb6d_sift_detect(*a) == ERR_WORKSPACE
    a[11] = None
    a[12] = need
    assert lib.ffb6d_sift_detect(*a) == ERR_WORKSPACE


def test_lift_refusals():
    ok = (P, P, 300, P, 6, 48, 64, P, 0, P, 3, P, P, None)
    assert lib.ffb6d_sift_lift(*ok[:4], 0, *ok[5:]) == OK
    for i, v in ((2, -1), (2, _lib.SIFT_MAX_CAP + 1), (10, 4), (10, 0), (8, 2), (0, None), (9, P + 4), (1, P + 2),
                 (3, P + 1), (11, P + 2), (12, P + 1)):
        a = list(ok)
        a[i] = v
        assert lib.ffb6d_sift_lift(*a) == ERR_INVALID, (i, v)


def test_python_refusals():
    with pytest.raises(ValueError):
        ops.sift_detect(torch.zeros((1, 8, 8, 3), dtype=torch.float32))
    with pytest.raises(ValueError):
        ops.sift_detect(np.zeros((1, 8, 8, 3), np.uint8))
    with pytest.raises(ValueError):
        objinfo.textured_kp3ds(object(), 0, extractor="SIFT")
    with pytest.raises(ValueError):
        objinfo.gen_obj_info(np.zeros((4, 3)), 2, start=0, extractor="SURF")


def test_write_obj_info_names_the_extractor(tmp_path):
    info = dict(corners=np.zeros((8, 3)), radius=1.0, center=np.zeros(3), fps=np.zeros((8, 3)),
                textured_fps=np.ones((8, 3), np.float32), extractor="SIFT")
    paths = objinfo.write_obj_info(info, str(tmp_path), "ape")
    assert os.path.basename(paths["SIFT_fps"]) == "ape_SIFT_fps.txt" and "ORB_fps" not in paths
    assert np.array_equal(np.loadtxt(paths["SIFT_fps"], dtype=np.float32), np.ones((8, 3), np.float32))
    del info["extractor"]
    assert os.path.basename(objinfo.write_obj_info(info, str(tmp_path), "ape")["ORB_fps"]) == "ape_ORB_fps.txt"
