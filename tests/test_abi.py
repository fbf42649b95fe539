"""CPU: libffb6d_b200.so loads, exports every symbol include/*.h declares, validates its
arguments without touching a GPU, and fails loudly (no CPU fallback) when no device exists."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT
from ffb6d_b200 import _lib

HAS_GPU = torch.cuda.is_available()


def declared_symbols():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        text = re.sub(r"/\*.*?\*/", "", open(h).read(), flags=re.S)
        names |= set(re.findall(r"\b(ffb6d_[a-z0-9_]+)\s*\(", text))
    return sorted(names)


def test_header_symbols_exported():
    syms = declared_symbols()
    assert len(syms) >= 14
    raw = C.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(raw, s), "include/ declares %s but the library does not export it" % s
    # and the Python binding covers exactly the header
    assert sorted(_lib.SYMBOLS) == syms


def test_abi_version_and_error_text():
    assert _lib.lib.ffb6d_version() == 3
    assert isinstance(_lib.last_error(), str)


def test_argument_validation_needs_no_gpu():
    lib = _lib.lib
    one = (C.c_float * 3)(0, 0, 0)
    out = (C.c_int64 * 64)()
    p, o = C.addressof(one), C.addressof(out)
    assert lib.ffb6d_knn_batch(p, p, 1, 1, 1, 0, o, 1, None, 0, None) == _lib.ERR_INVALID
    assert "K=0" in _lib.last_error()
    assert lib.ffb6d_knn_batch(p, p, 1, 1, 1, 65, o, 1, None, 0, None) == _lib.ERR_INVALID
    assert lib.ffb6d_knn_batch(p, p, -1, 1, 1, 1, o, 1, None, 0, None) == _lib.ERR_INVALID
    assert lib.ffb6d_knn_batch(None, p, 1, 1, 1, 1, o, 1, None, 0, None) == _lib.ERR_INVALID
    assert lib.ffb6d_knn_batch(p, p, 0, 1, 1, 1, o, 1, None, 0, None) == _lib.OK      # empty batch
    assert lib.ffb6d_knn_batch_host(p, 1, 1, 2, p, 1, 1, o) == _lib.ERR_INVALID        # dim != 3
    assert lib.ffb6d_gather_max_fwd(p, o, 1, 1, 1, 1, 1, 0, 0, p, None) == _lib.ERR_INVALID
    assert lib.ffb6d_gather_max_fwd(p, o, 1, 1, 1, 1, 1, 1, 7, p, None) == _lib.ERR_INVALID  # layout
    assert lib.ffb6d_gather_max_fwd(p, o, 1, 1, 1, 0, 1, 1, 0, p, None) == _lib.ERR_INVALID  # S == 0
    assert lib.ffb6d_gather_max_fwd(p, o, 1, 0, 1, 1, 1, 1, 0, p, None) == _lib.OK          # B == 0
    # channels-last: 8 queries per block in grid.x, so B*Q <= 8 * (2^31 - 1); NCS has no such bound
    q = (1 << 31) - 1
    assert lib.ffb6d_gather_max_fwd(p, o, 1, 9, 1, 1, q, 1, 1, p, None) == _lib.ERR_INVALID
    assert "too large for the channels-last layout" in _lib.last_error()
    assert lib.ffb6d_gather_max_fwd(p, o, 1, 0, 1, 1, q, 1, 1, p, None) == _lib.OK          # B*Q == 0
    assert lib.ffb6d_gather_neighbour_fwd(None, o, 1, 1, 1, 1, 1, 1, p, None) == _lib.ERR_INVALID
    assert lib.ffb6d_knn_workspace_bytes(1, 0, 1, 1) == 0


def test_train_argument_validation_needs_no_gpu():
    """The training entry points reject bad sizes, activations, null and misaligned pointers before any launch."""
    lib = _lib.lib
    buf = (C.c_float * 64)()
    p = (C.addressof(buf) + 15) & ~15           # 16-byte aligned
    BIG = 1 << 40                               # a workspace size that passes its check

    def fwd(z=p, B=2, Cc=3, P=5, act=1, stats=p, y=p, ws=p, nbytes=BIG):
        return lib.ffb6d_bn_train_fwd(z, B, Cc, P, p, p, 1e-5, 0.1, p, p, act, 0.0, stats, y, ws, nbytes, None)

    def bwd(z=p, gy=p, stats=p, B=2, Cc=3, P=5, act=1, gz=p, ws=p, nbytes=BIG):
        return lib.ffb6d_bn_train_bwd(z, gy, stats, B, Cc, P, act, 0.0, p, p, gz, ws, nbytes, None)

    for call, name in ((fwd, "bn_train_fwd"), (bwd, "bn_train_bwd")):
        for size in (dict(B=0), dict(Cc=0), dict(P=0), dict(B=-1), dict(B=65536), dict(Cc=65536), dict(P=1 << 31),
                     dict(B=40000, Cc=60000)):
            assert call(**size) == _lib.ERR_INVALID, (name, size)
            assert name + ": bad size" in _lib.last_error()
        for act in (-1, 3):
            assert call(act=act) == _lib.ERR_INVALID, (name, act)
            assert "act=%d" % act in _lib.last_error()
        assert call(stats=p + 4) == _lib.ERR_INVALID, name
        assert "16-byte aligned" in _lib.last_error()
        assert call(nbytes=0) == _lib.ERR_INVALID, name
        assert "workspace too small" in _lib.last_error()
    for ptr in ("z", "stats", "y", "ws"):
        assert fwd(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    for ptr in ("z", "gy", "stats", "gz", "ws"):
        assert bwd(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    assert lib.ffb6d_bn_workspace_bytes(0, 5) == 0 and lib.ffb6d_bn_workspace_bytes(3, 0) == 0

    assert lib.ffb6d_act_bwd(p, p, -1, 1, 0.0, p, None) == _lib.ERR_INVALID
    assert lib.ffb6d_act_bwd(p, p, 8, 3, 0.0, p, None) == _lib.ERR_INVALID
    assert lib.ffb6d_act_bwd(p, p, 8, -1, 0.0, p, None) == _lib.ERR_INVALID
    for i in range(3):
        ptrs = [p, p, p]
        ptrs[i] = None
        assert lib.ffb6d_act_bwd(ptrs[0], ptrs[1], 8, 1, 0.0, ptrs[2], None) == _lib.ERR_INVALID
        assert "null pointer" in _lib.last_error()
    assert lib.ffb6d_act_bwd(None, None, 0, 1, 0.0, None, None) == _lib.OK      # nothing to do

    assert lib.ffb6d_att_pool_bwd(p, 0, None, 0, p, p, 1, 4, 16, p, None, p, None) == _lib.ERR_INVALID   # C1 = 0
    assert lib.ffb6d_att_pool_bwd(p, 2, None, 0, p, p, 1, 4, 0, p, None, p, None) == _lib.ERR_INVALID    # K = 0
    assert lib.ffb6d_att_pool_bwd(p, 2, None, 0, p, p, 1, 4, 65, p, None, p, None) == _lib.ERR_INVALID   # K > 64
    assert lib.ffb6d_att_pool_bwd(p, 2, None, 3, p, p, 1, 4, 16, p, None, p, None) == _lib.ERR_INVALID   # f2 missing
    assert "null pointer" in _lib.last_error()
    assert lib.ffb6d_att_pool_bwd(p, 2, None, 0, p, p, 0, 4, 16, p, None, p, None) == _lib.OK            # B == 0


@pytest.mark.skipif(HAS_GPU, reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback():
    """Without a device the product must fail loudly, never compute on the CPU."""
    import ffb6d_b200 as F
    assert _lib.lib.ffb6d_device_count() == 0
    pts = np.random.RandomState(0).rand(1, 32, 3).astype(np.float32)
    with pytest.raises(_lib.FFB6DError) as e:
        F.knn_search(pts, pts, 4)
    assert e.value.code == _lib.ERR_NO_DEVICE
    with pytest.raises(RuntimeError, match="no CPU path"):
        F.random_sample(torch.zeros(1, 4, 8, 1), torch.zeros(1, 2, 16, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="no CPU path"):
        F.gather_neighbour(torch.zeros(1, 8, 3), torch.zeros(1, 8, 4, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="no CPU path"):
        F.knn_search(torch.zeros(1, 8, 3), torch.zeros(1, 8, 3), 2)


def test_product_does_not_import_oracle():
    """The product package must not reference oracle/ anywhere."""
    pkg = os.path.join(ROOT, "ffb6d_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f
                assert "liboracle" not in text and "_ref/" not in text, f


def test_schedule_and_mlp_planning_need_no_gpu():
    """Host-side arithmetic of the one-call schedule and the packed-weight layout; argument errors are
    reported before any CUDA call."""
    lib = _lib.lib
    # 32 KB ([A_hi | A_lo], 128 rows x 32 k) per (row tile, k-tile)
    assert lib.ffb6d_fusion_mlp_pack_bytes(1024, 2048) == 8 * 64 * 32768
    assert lib.ffb6d_fusion_mlp_pack_bytes(70, 44) == 1 * 2 * 32768          # ragged sizes round up
    assert lib.ffb6d_fusion_mlp_pack_bytes(0, 16) == 0
    w1 = lib.ffb6d_build_indices_workspace_bytes(1, 12288, 480, 640, 16)
    w4 = lib.ffb6d_build_indices_workspace_bytes(4, 12288, 480, 640, 16)
    assert 0 < w1 < w4 <= 4 * w1 + 4096
    assert lib.ffb6d_build_indices_workspace_bytes(1, 100, 480, 640, 16) == 0     # N0 too small
    assert lib.ffb6d_build_indices_workspace_bytes(1, 12288, 480, 640, 65) == 0   # K too large
    one = (C.c_float * 3)(0, 0, 0)
    p = C.addressof(one)
    outs = (C.c_void_p * 22)(*([p] * 22))
    args = (p, p, p, p)
    assert lib.ffb6d_build_indices(*args, 1, 1000, 480, 640, 16, outs, 0, p, 1 << 30, None) == _lib.ERR_INVALID
    assert "multiple of 256" in _lib.last_error()
    assert lib.ffb6d_build_indices(*args, 1, 12288, 481, 640, 16, outs, 0, p, 1 << 30, None) == _lib.ERR_INVALID
    assert lib.ffb6d_build_indices(*args, 1, 12288, 480, 640, 16, outs, 0, p, 16, None) == _lib.ERR_WORKSPACE
    assert lib.ffb6d_build_indices(*args, 0, 12288, 480, 640, 16, outs, 0, p, 0, None) == _lib.OK   # empty batch
    outs[5] = None
    assert lib.ffb6d_build_indices(*args, 1, 12288, 480, 640, 16, outs, 0, p, 1 << 30, None) == _lib.ERR_INVALID
    assert "out[5]" in _lib.last_error()
    assert lib.ffb6d_fusion_mlp_pack(None, 64, 64, p, 1 << 20, None) == _lib.ERR_INVALID
    assert lib.ffb6d_fusion_mlp_pack(p, 64, 64, p, 16, None) == _lib.ERR_WORKSPACE
