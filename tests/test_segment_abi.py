"""CPU: the segment sum (the backward of the restructured fusion stage's gathered addend) checks its arguments
before any launch -- sizes, null pointers, plan bytes, alignment -- and reports them through ffb6d_last_error;
ops.segment_plan / ops.segment_sum reject wrong dtypes, shapes and devices."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib, ops


def frame_words(P, NA):
    """int32 words of one frame's plan: offsets [NA+1], pixels [P], counts per (segment, 1024-pixel tile)."""
    t = -(-P // 1024)
    return (NA + 1 + P + NA * t + 3) // 4 * 4


def test_segment_plan_bytes():
    lib = _lib.lib
    assert lib.ffb6d_segment_plan_bytes(1, 1, 1) == 16
    assert lib.ffb6d_segment_plan_bytes(8, 19200, 3072) == 8 * 4 * frame_words(19200, 3072)     # ds0 at 480x640
    assert lib.ffb6d_segment_plan_bytes(3, 7 * 13, 5) == 3 * 4 * frame_words(91, 5)
    for bad in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (-1, 1, 1), (1, -5, 1), (65536, 1, 1), (1, 1 << 31, 1),
                (1, 1 << 30, 1 << 20)):          # the last one: a frame's plan past 2^31 words
        assert lib.ffb6d_segment_plan_bytes(*bad) == 0, bad


def test_segment_entry_points_reject_bad_arguments():
    lib = _lib.lib
    buf = (C.c_int64 * 64)()
    p = (C.addressof(buf) + 15) & ~15           # 16-byte aligned
    BIG = 1 << 40                               # a plan size that passes its check

    def plan(idx=p, i64=0, B=2, P=5, NA=3, out=p, nbytes=BIG):
        return lib.ffb6d_segment_plan(idx, i64, B, P, NA, out, nbytes, None)

    def ssum(grad=p, pl=p, nbytes=BIG, B=2, Cc=4, P=5, NA=3, out=p):
        return lib.ffb6d_segment_sum(grad, pl, nbytes, B, Cc, P, NA, out, None)

    for call, name in ((plan, "segment_plan"), (ssum, "segment_sum")):
        for size in (dict(B=0), dict(P=0), dict(NA=0), dict(B=-1), dict(P=-1), dict(NA=-2), dict(B=65536),
                     dict(P=1 << 31), dict(NA=1 << 31)):
            assert call(**size) == _lib.ERR_INVALID, (name, size)
            assert name + ": bad size" in _lib.last_error()
        assert call(nbytes=0) == _lib.ERR_INVALID, name
        assert "plan too small" in _lib.last_error()
        assert call(nbytes=lib.ffb6d_segment_plan_bytes(2, 5, 3) - 1) == _lib.ERR_INVALID, name
        assert "plan too small" in _lib.last_error()
    for size in (dict(Cc=0), dict(Cc=-1), dict(Cc=32 * 65535 + 1)):
        assert ssum(**size) == _lib.ERR_INVALID, size
        assert "segment_sum: bad size" in _lib.last_error()
    for ptr in ("idx", "out"):
        assert plan(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    for ptr in ("grad", "pl", "out"):
        assert ssum(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    assert plan(i64=2) == _lib.ERR_INVALID
    assert "idx_is_i64=2" in _lib.last_error()
    assert plan(idx=p + 2) == _lib.ERR_INVALID                   # int32 indices on a 2-byte boundary
    assert "idx misaligned" in _lib.last_error()
    assert plan(idx=p + 4, i64=1) == _lib.ERR_INVALID            # int64 indices on a 4-byte boundary
    assert "idx misaligned" in _lib.last_error()
    assert plan(out=p + 4) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    assert ssum(pl=p + 8) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    for ptr in ("grad", "out"):
        assert ssum(**{ptr: p + 2}) == _lib.ERR_INVALID, ptr
        assert "4-byte aligned" in _lib.last_error()


def test_segment_ops_reject_bad_inputs():
    idx = torch.zeros(2, 12, dtype=torch.int32)
    with pytest.raises(TypeError, match="int32 or int64"):
        ops.segment_plan(idx.float(), 4)
    with pytest.raises(TypeError, match="torch.Tensor"):
        ops.segment_plan(idx.numpy(), 4)
    for shape in ((24,), (2, 12, 2), (2, 3, 4, 1), (2, 0)):
        with pytest.raises(ValueError, match="idx must be"):
            ops.segment_plan(torch.zeros(shape, dtype=torch.int64), 4)
    with pytest.raises(ValueError, match="n_segments"):
        ops.segment_plan(idx, 0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.segment_plan(idx, 4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.segment_plan(idx.unsqueeze(2).long(), 4)
    grad = torch.zeros(2, 3, 12)
    with pytest.raises(TypeError, match="float32"):
        ops.segment_sum(grad.double(), idx, 4)
    for shape in ((2, 12), (2, 3, 3, 4, 1), (2, 0, 12)):
        with pytest.raises(ValueError, match="grad must be"):
            ops.segment_sum(torch.zeros(shape), idx, 4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.segment_sum(grad, idx, 4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.segment_sum(grad.view(2, 3, 3, 4), idx, 4)
