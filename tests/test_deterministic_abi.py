"""CPU: the deterministic backward entry points (segment CSR, gather + max, neighbour gather, layer weight gradient)
check their arguments before any launch -- sizes, null and misaligned pointers, short workspaces, idx_is_i64 -- and
report them through ffb6d_last_error; the CSR plan's size is linear in P + NA; ops.deterministic_backward follows
torch's switches."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib, ops

BIG = 1 << 40                                   # a byte count that passes every workspace check


@pytest.fixture
def buf():
    b = (C.c_int64 * 64)()
    return (C.addressof(b) + 15) & ~15, b       # 16-byte aligned address (the array keeps it alive)


def test_segment_csr_bytes_linear_in_p_plus_na():
    lib = _lib.lib
    assert lib.ffb6d_segment_csr_bytes(1, 1, 1) == 32
    for B, P, NA in ((8, 12288, 307200), (2, 12288 * 16, 12288), (2, 3072 * 16, 76800), (2, 19200, 3072), (1, 1, 1 << 20),
                     (1, 1 << 24, 1)):
        n = lib.ffb6d_segment_csr_bytes(B, P, NA)
        assert n % 16 == 0 and n == B * lib.ffb6d_segment_csr_bytes(1, P, NA), (B, P, NA)
        assert 4 * B * (NA + 1 + P) <= n <= B * 4 * (2 * NA + 2 * P) + B * 4 * (NA // 4096 + 8), (B, P, NA, n)
    # the issue's example: choose at 480x640, 8 frames
    assert lib.ffb6d_segment_csr_bytes(8, 12288, 307200) < 8 * 4 * (2 * 307200 + 2 * 12288) + 4096
    # the counter plan grows with NA x ceil(P / 1024); the CSR does not
    assert lib.ffb6d_segment_plan_bytes(8, 12288, 307200) > 5 * lib.ffb6d_segment_csr_bytes(8, 12288, 307200)
    for bad in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (-1, 1, 1), (65536, 1, 1), (1, 1 << 31, 1), (1, 1, 1 << 31),
                (1, 1 << 30, 1 << 30)):
        assert lib.ffb6d_segment_csr_bytes(*bad) == 0, bad


def test_segment_csr_entry_points_reject_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf

    def plan(idx=p, i64=0, B=2, P=5, NA=3, out=p, nbytes=BIG):
        return lib.ffb6d_segment_csr(idx, i64, B, P, NA, out, nbytes, None)

    def ssum(grad=p, pl=p, nbytes=BIG, B=2, Cc=4, P=5, NA=3, out=p):
        return lib.ffb6d_segment_sum_csr(grad, pl, nbytes, B, Cc, P, NA, out, None)

    for call, name in ((plan, "segment_csr"), (ssum, "segment_sum_csr")):
        for size in (dict(B=0), dict(P=0), dict(NA=0), dict(B=-1), dict(P=-1), dict(NA=-2), dict(B=65536),
                     dict(P=1 << 31), dict(NA=1 << 31)):
            assert call(**size) == _lib.ERR_INVALID, (name, size)
            assert name + ": bad size" in _lib.last_error()
        assert call(nbytes=lib.ffb6d_segment_csr_bytes(2, 5, 3) - 1) == _lib.ERR_INVALID, name
        assert "plan too small" in _lib.last_error()
    for size in (dict(Cc=0), dict(Cc=-1), dict(Cc=32 * 65535 + 1)):
        assert ssum(**size) == _lib.ERR_INVALID, size
        assert "segment_sum_csr: bad size" in _lib.last_error()
    for ptr in ("idx", "out"):
        assert plan(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    for ptr in ("grad", "pl", "out"):
        assert ssum(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    for v in (2, -1):
        assert plan(i64=v) == _lib.ERR_INVALID
        assert "idx_is_i64=%d" % v in _lib.last_error()
    assert plan(idx=p + 2) == _lib.ERR_INVALID
    assert "idx misaligned" in _lib.last_error()
    assert plan(idx=p + 4, i64=1) == _lib.ERR_INVALID
    assert "idx misaligned" in _lib.last_error()
    assert plan(out=p + 4) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    assert ssum(pl=p + 8) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    for ptr in ("grad", "out"):
        assert ssum(**{ptr: p + 2}) == _lib.ERR_INVALID, ptr
        assert "4-byte aligned" in _lib.last_error()


def test_gather_max_bwd_det_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf
    need = lib.ffb6d_gather_max_bwd_det_workspace_bytes(2, 4, 7, 5, 3)
    # the CSR of [B, Q*K] over S segments, then a uint8 arg-max map [B, C, Q] rounded up to 16 bytes
    assert need == lib.ffb6d_segment_csr_bytes(2, 15, 7) + 48
    assert lib.ffb6d_gather_max_bwd_det_workspace_bytes(2, 4, 7, 5, 1) == lib.ffb6d_segment_csr_bytes(2, 5, 7)
    for bad in ((0, 4, 7, 5, 3), (2, 0, 7, 5, 3), (2, 4, 0, 5, 3), (2, 4, 7, 0, 3), (2, 4, 7, 5, 0), (2, 4, 7, 5, 65),
                (2, 4, 7, 1 << 27, 16)):
        assert lib.ffb6d_gather_max_bwd_det_workspace_bytes(*bad) == 0, bad

    def call(feat=p, idx=p, i64=0, g=p, B=2, Cc=4, S=7, Q=5, K=3, layout=_lib.LAYOUT_NCS, ws=p, nbytes=BIG, out=p):
        return lib.ffb6d_gather_max_bwd_det(feat, idx, i64, g, B, Cc, S, Q, K, layout, ws, nbytes, out, None)

    for size in (dict(B=-1), dict(Cc=-1), dict(S=-1), dict(Q=-1)):
        assert call(**size) == _lib.ERR_INVALID, size
        assert "negative size" in _lib.last_error()
    for k in (0, 65):
        assert call(K=k) == _lib.ERR_INVALID
        assert "K=%d" % k in _lib.last_error()
    assert call(layout=2) == _lib.ERR_INVALID
    assert "unknown layout" in _lib.last_error()
    assert call(i64=2) == _lib.ERR_INVALID
    assert "idx_is_i64=2" in _lib.last_error()
    for size in (dict(S=0), dict(Cc=32 * 65535 + 1), dict(S=1 << 31), dict(Q=1 << 27, K=16)):
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bad size" in _lib.last_error()
    for ptr in ("feat", "idx", "g", "ws", "out"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    assert call(idx=p + 2) == _lib.ERR_INVALID
    assert "idx misaligned" in _lib.last_error()
    assert call(idx=p + 4, i64=1) == _lib.ERR_INVALID
    assert "idx misaligned" in _lib.last_error()
    for ptr in ("feat", "g", "out"):
        assert call(**{ptr: p + 2}) == _lib.ERR_INVALID, ptr
        assert "4-byte aligned" in _lib.last_error()
    assert call(ws=p + 8) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    assert call(nbytes=need - 1) == _lib.ERR_INVALID
    assert "workspace too small" in _lib.last_error()


def test_gather_neighbour_bwd_det_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf
    need = lib.ffb6d_gather_neighbour_bwd_det_workspace_bytes(2, 7, 5, 3)
    assert need == lib.ffb6d_segment_csr_bytes(2, 15, 7)
    for bad in ((0, 7, 5, 3), (2, 0, 5, 3), (2, 7, 0, 3), (2, 7, 5, 0), (2, 7, 1 << 27, 16)):
        assert lib.ffb6d_gather_neighbour_bwd_det_workspace_bytes(*bad) == 0, bad

    def call(g=p, idx=p, i64=0, B=2, S=7, D=4, N=5, K=3, ws=p, nbytes=BIG, out=p):
        return lib.ffb6d_gather_neighbour_bwd_det(g, idx, i64, B, S, D, N, K, ws, nbytes, out, None)

    for size in (dict(B=-1), dict(S=-1), dict(D=-1), dict(N=-1), dict(K=-1)):
        assert call(**size) == _lib.ERR_INVALID, size
        assert "negative size" in _lib.last_error()
    assert call(i64=2) == _lib.ERR_INVALID
    assert "idx_is_i64=2" in _lib.last_error()
    for size in (dict(S=0), dict(D=32 * 65535 + 1), dict(S=1 << 31), dict(N=1 << 27, K=16)):
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bad size" in _lib.last_error()
    for ptr in ("g", "idx", "ws", "out"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    assert call(idx=p + 2) == _lib.ERR_INVALID
    assert "idx misaligned" in _lib.last_error()
    for ptr in ("g", "out"):
        assert call(**{ptr: p + 2}) == _lib.ERR_INVALID, ptr
        assert "4-byte aligned" in _lib.last_error()
    assert call(ws=p + 4) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    assert call(nbytes=need - 1) == _lib.ERR_INVALID
    assert "workspace too small" in _lib.last_error()


def test_wgrad_det_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf
    for shape in ((64, 64, 2, 64, 3072), (10, 0, 4, 16, 196608), (1024, 1024, 2, 1024, 4800), (131, 125, 2, 200, 4097)):
        n = lib.ffb6d_fusion_mlp_wgrad_det_workspace_bytes(*shape)
        C1, C2, B, Co, P = shape
        # one [Co, Ci] fp32 partial per split
        assert n > 0 and n % 16 == 0 and (n // 4) >= Co * (C1 + C2), shape
    for bad in ((0, 0, 2, 4, 5), (3, -1, 2, 4, 5), (3, 0, 0, 4, 5), (3, 0, 2, 0, 5), (3, 0, 2, 4, 0), (3, 0, 65536, 4, 5),
                (3, 0, 2, 4, 1 << 31)):
        assert lib.ffb6d_fusion_mlp_wgrad_det_workspace_bytes(*bad) == 0, bad

    def call(dz=p, x1=p, C1=3, x2=p, C2=2, B=2, Co=4, P=5, ws=p, nbytes=BIG, out=p):
        return lib.ffb6d_fusion_mlp_wgrad_det(dz, x1, C1, x2, C2, B, Co, P, ws, nbytes, out, None)

    for size in (dict(B=-1), dict(C1=0), dict(C2=-1), dict(Co=0), dict(P=-1)):
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bad size" in _lib.last_error()
    for size in (dict(B=65536), dict(P=1 << 31), dict(Co=65535 * 128 + 1)):
        assert call(**size) == _lib.ERR_INVALID, size
        assert "size too large" in _lib.last_error()
    assert call(out=None) == _lib.ERR_INVALID
    assert "null grad_w" in _lib.last_error()
    for ptr in ("dz", "x1", "x2", "ws"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "null pointer" in _lib.last_error()
    for ptr in ("dz", "x1", "x2", "out"):
        assert call(**{ptr: p + 2}) == _lib.ERR_INVALID, ptr
        assert "4-byte aligned" in _lib.last_error()
    assert call(ws=p + 4) == _lib.ERR_INVALID
    assert "16-byte aligned" in _lib.last_error()
    assert call(nbytes=lib.ffb6d_fusion_mlp_wgrad_det_workspace_bytes(3, 2, 2, 4, 5) - 1) == _lib.ERR_INVALID
    assert "workspace too small" in _lib.last_error()


def test_deterministic_backward_follows_torch_switches():
    algo, cudnn = torch.are_deterministic_algorithms_enabled(), torch.backends.cudnn.deterministic
    try:
        torch.use_deterministic_algorithms(False)
        torch.backends.cudnn.deterministic = False
        assert not ops.deterministic_backward() and not ops.deterministic_backward(weight_grad=True)
        torch.backends.cudnn.deterministic = True          # the reference's --deterministic: the layers only
        assert not ops.deterministic_backward() and ops.deterministic_backward(weight_grad=True)
        torch.backends.cudnn.deterministic = False
        torch.use_deterministic_algorithms(True)
        assert ops.deterministic_backward() and ops.deterministic_backward(weight_grad=True)
        torch.use_deterministic_algorithms(True, warn_only=True)
        assert ops.deterministic_backward() and ops.deterministic_backward(weight_grad=True)
    finally:
        torch.use_deterministic_algorithms(algo)
        torch.backends.cudnn.deterministic = cudnn


def test_segment_csr_op_rejects_bad_inputs():
    idx = torch.zeros(2, 12, dtype=torch.int32)
    with pytest.raises(TypeError, match="int32 or int64"):
        ops.segment_csr(idx.float(), 4)
    for shape in ((24,), (2, 12, 2), (2, 0)):
        with pytest.raises(ValueError, match="idx must be"):
            ops.segment_csr(torch.zeros(shape, dtype=torch.int64), 4)
    with pytest.raises(ValueError, match="n_segments"):
        ops.segment_csr(idx, 0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.segment_csr(idx, 4)
