"""CPU: the argument checks of the attentive pooling's training kernels (ffb6d_lfa_train_fwd / _bwd and the
workspace query) and of their Python wrappers.  Every case here is rejected before anything touches a device."""
import ctypes as C

import pytest
import torch

from ffb6d_b200 import _lib, ops

lib = _lib.lib
INVALID = _lib.ERR_INVALID


@pytest.fixture
def bufs():
    mem = (C.c_float * 64)()
    return C.addressof(mem), mem


def fwd(p, B=1, N=1, K=16, Dh=16, i64=0, feature=True, idx=True, f_xyz=True, w=True, out=True):
    return lib.ffb6d_lfa_train_fwd(p if feature else None, p if idx else None, i64, p if f_xyz else None,
                                   p if w else None, B, N, K, Dh, p if out else None, None)


def bwd(p, B=1, N=1, K=16, Dh=16, i64=0, null=(), edge=None, gx=None):
    a = {k: (None if k in null else p) for k in ("feature", "idx", "f_xyz", "w", "g", "gw")}
    return lib.ffb6d_lfa_train_bwd(a["feature"], a["idx"], i64, a["f_xyz"], a["w"], a["g"], B, N, K, Dh,
                                   None if "edge" in null else (edge or p), None if "gx" in null else (gx or p),
                                   a["gw"], p, 1 << 20, None)


@pytest.mark.parametrize("K", [0, 1, 8, 15, 17, 32, 64])
def test_neighbour_count_other_than_16_is_rejected(bufs, K):
    p, _ = bufs
    assert fwd(p, K=K) == INVALID
    assert "only K = 16" in _lib.last_error()
    assert bwd(p, K=K) == INVALID
    assert "only K = 16" in _lib.last_error()
    assert lib.ffb6d_lfa_train_bwd_workspace_bytes(8, 12288, K, 16) == 0


@pytest.mark.parametrize("Dh", [0, 8, 24, 48, 128, 256, -16])
def test_unsupported_width_is_rejected(bufs, Dh):
    p, _ = bufs
    assert fwd(p, Dh=Dh) == INVALID
    assert "fused for 16, 32, 64" in _lib.last_error()
    assert bwd(p, Dh=Dh) == INVALID
    assert "fused for 16, 32, 64" in _lib.last_error()
    assert lib.ffb6d_lfa_train_bwd_workspace_bytes(8, 12288, 16, Dh) == 0


@pytest.mark.parametrize("B,N", [(-1, 1), (1, -1), (65536, 1), (1, 1 << 31), (1 << 40, 1)])
def test_sizes_past_the_limits_are_rejected(bufs, B, N):
    p, _ = bufs
    assert fwd(p, B=B, N=N) == INVALID
    assert "bad size" in _lib.last_error()
    assert bwd(p, B=B, N=N) == INVALID
    assert "bad size" in _lib.last_error()
    assert lib.ffb6d_lfa_train_bwd_workspace_bytes(B, N, 16, 16) == 0


def test_index_type_flag_is_checked(bufs):
    p, _ = bufs
    assert fwd(p, i64=2) == INVALID
    assert bwd(p, i64=-1) == INVALID
    assert "idx_is_i64" in _lib.last_error()


@pytest.mark.parametrize("which", ["feature", "idx", "f_xyz", "w", "out"])
def test_forward_null_pointers_are_rejected(bufs, which):
    p, _ = bufs
    assert fwd(p, **{which: False}) == INVALID
    assert "null pointer" in _lib.last_error()


@pytest.mark.parametrize("which", ["feature", "idx", "f_xyz", "w", "g", "edge", "gx", "gw"])
def test_backward_null_pointers_are_rejected(bufs, which):
    p, _ = bufs
    assert bwd(p, null=(which,)) == INVALID
    assert "null pointer" in _lib.last_error()


def test_empty_forward_is_a_no_op(bufs):
    p, _ = bufs
    assert fwd(p, B=0) == _lib.OK
    assert fwd(p, N=0, feature=False, idx=False, f_xyz=False, w=False, out=False) == _lib.OK


@pytest.mark.parametrize("which", ["edge", "gx"])
def test_misaligned_gradient_rows_are_rejected(bufs, which):
    """The backward stores a point's 16 positions with 128-bit stores."""
    p, _ = bufs
    assert bwd(p, **{which: p + 4}) == INVALID
    assert "16-byte aligned" in _lib.last_error()


def _args(B=2, Dh=16, N=5, K=16, idx_dtype=torch.int32):
    return (torch.zeros(B, Dh, N, 1), torch.zeros(B, N, K, dtype=idx_dtype), torch.zeros(B, Dh, N, K),
            torch.zeros(2 * Dh, 2 * Dh, 1, 1))


@pytest.mark.parametrize("case", ["feature_rank", "idx_batch", "idx_points", "f_xyz_width", "f_xyz_points",
                                  "f_xyz_k", "w_fc_width", "w_fc_square"])
def test_wrappers_reject_mismatched_shapes(case):
    f, idx, fx, w = _args()
    if case == "feature_rank":
        f = f.reshape(2, 16, 5, 1, 1)
    elif case == "idx_batch":
        idx = idx[:1]
    elif case == "idx_points":
        idx = idx[:, :4]
    elif case == "f_xyz_width":
        fx = torch.zeros(2, 32, 5, 16)
    elif case == "f_xyz_points":
        fx = fx[:, :, :4]
    elif case == "f_xyz_k":
        fx = fx[..., :8]
    elif case == "w_fc_width":
        w = torch.zeros(64, 64, 1, 1)
    else:
        w = torch.zeros(32, 16, 1, 1)
    with pytest.raises(ValueError):
        ops.lfa_train_fwd(f, idx, fx, w)
    with pytest.raises(ValueError):
        ops.lfa_train_bwd(f, idx, fx, w, torch.zeros(2, 32, 5, 1))


def test_wrappers_need_cuda_tensors():
    f, idx, fx, w = _args()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.lfa_train_fwd(f, idx, fx, w)


def test_fusable_range_matches_the_kernels():
    assert [d for d in (8, 16, 24, 32, 64, 128) if ops.lfa_fusable(d, 16)] == [16, 32, 64]
    assert not any(ops.lfa_fusable(16, k) for k in (1, 8, 15, 17, 32))
