"""CPU: the numpy restatement of the YCB depth completion (oracle/fill_oracle.py) reproduces the reference's
``fill_missing`` outputs and stages stored in tests/golden/fill_cases.npz, and ``ops.fill_missing`` /
``ffb6d_fill_depth`` reject what they do not implement before touching a GPU."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, _npz_groups
from oracle import fill_oracle as O
from ffb6d_b200.synthetic import fill_test_frames, FILL_CAM_SCALE

EXACT = ("s1_inverted_depths", "s2_dilated_depths", "s3_closed_depths", "s4_blurred_depths", "s5_combined_depths",
         "s6_extended_depths")
TOL_M = 2e-6          # metres, on the pixels the bilateral blur writes; every other pixel is bitwise


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def assert_fill_contract(got, want, blurred, scale=1.0):
    """Bitwise (uint32, signed zeros included) outside ``blurred``; within TOL_M * scale inside."""
    assert got.dtype == np.float32 and got.shape == want.shape
    assert np.array_equal(got[~blurred].view(np.uint32), want[~blurred].view(np.uint32))
    if blurred.any():
        err = np.abs(got[blurred].astype(np.float64) - want[blurred]).max()
        assert err <= TOL_M * scale, err


def assert_matches_golden(out, blurred, g, scale=1.0):
    """``out`` (the final map, raw units) against one frame of fill_cases.npz under the contract.  Small frames
    store the reference's output; the full frames store sha256s of the blurred-pixel mask, of the output with
    those pixels zeroed and of ``msk_dp``, plus the reference's value at a seeded sample of the blurred pixels."""
    if "out" in g:
        assert_fill_contract(out, g["out"], blurred, scale)
        assert np.array_equal(out > np.float32(1e-6), g["out"] > np.float32(1e-6))      # msk_dp
        return
    assert sha(blurred) == str(g["sha256_blurred"])
    unblurred = out.copy()
    unblurred[blurred] = 0
    assert sha(unblurred) == str(g["sha256_out_unblurred"])
    assert sha(out > np.float32(1e-6)) == str(g["sha256_msk_dp"])                        # msk_dp
    idx = g["sample_idx"]
    assert blurred.reshape(-1)[idx].all()
    err = np.abs(out.reshape(-1)[idx].astype(np.float64) - g["sample_out"]).max()
    assert err <= TOL_M * scale, err


@pytest.fixture(scope="module")
def golden():
    return _npz_groups(os.path.join(GOLDEN, "fill_cases.npz"))


@pytest.fixture(scope="module")
def frames():
    return fill_test_frames()


@pytest.mark.parametrize("name", sorted(fill_test_frames()))
def test_oracle_reproduces_reference(golden, frames, name):
    g, raw = golden[name], frames[name]
    assert sha(raw) == str(g["sha256_raw"]), "input generator changed"
    out, st = O.fill_missing(raw, FILL_CAM_SCALE, return_stages=True)
    for k in EXACT:
        if "sha256_" + k in g:
            assert sha(st[k]) == str(g["sha256_" + k]), k
        else:
            assert np.array_equal(st[k].view(np.uint32), g[k].view(np.uint32)), k
    blurred = st["bilateral_mask"]
    for k in ("s7_blurred_depths", "s8_inverted_depths"):
        if k in g:
            assert_fill_contract(st[k], g[k], blurred)
    assert_matches_golden(out, blurred, g, FILL_CAM_SCALE)


def test_golden_cases_cover_the_edges(golden, frames):
    """The small cases exercise what they are named after."""
    st = {n: O.fill_missing(frames[n], FILL_CAM_SCALE, return_stages=True)[1] for n in frames}
    assert not (golden["all_holes"]["out"] != 0).any()
    assert not st["constant"]["bilateral_mask"].any() or \
        np.array_equal(st["constant"]["s7_blurred_depths"], st["constant"]["s7_median_depths"])
    assert (frames["no_holes"] > 0).all() and st["no_holes"]["bilateral_mask"].any()
    sv = frames["special_values"]
    for v in (10000, 20000, 30001, 65535, 1, 100):
        assert (sv == v).any(), v
    assert (golden["special_values"]["out"] < 0).any()          # beyond 3 m: inverted to < 0, never inverted back
    et = frames["empty_top"]
    assert not et[:5].any() and not et[:, 40].any()
    assert min(frames["tiny"].shape) < 9


def _cpu_raw(shape=(8, 9)):
    return torch.zeros(shape, dtype=torch.uint16)


@pytest.mark.parametrize("kw", [dict(fill_type="fast"), dict(extrapolate=True), dict(blur_type="gaussian"),
                                dict(scale_2_80m=2), dict(scale_2_80m=0.5)])
def test_fill_missing_rejects_unsupported_options(kw):
    import ffb6d_b200 as F
    with pytest.raises(ValueError):
        F.fill_missing(_cpu_raw(), 10000.0, **kw)


@pytest.mark.parametrize("bad", [torch.zeros((8, 9), dtype=torch.float32), torch.zeros((8, 9), dtype=torch.int32),
                                 torch.zeros((72,), dtype=torch.uint16), torch.zeros((1, 1, 8, 9), dtype=torch.uint16),
                                 torch.zeros((0, 8, 9), dtype=torch.uint16)])
def test_fill_missing_rejects_dtype_and_shape(bad):
    import ffb6d_b200 as F
    with pytest.raises(ValueError):
        F.fill_missing(bad, 10000.0)


@pytest.mark.parametrize("cs", [0.0, -1.0, float("nan"), float("inf")])
def test_fill_missing_rejects_cam_scale(cs):
    import ffb6d_b200 as F
    with pytest.raises(ValueError):
        F.fill_missing(_cpu_raw(), cs)


def test_fill_depth_abi_validation_needs_no_gpu():
    from ffb6d_b200 import _lib
    lib = _lib.lib
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    ws = lib.ffb6d_fill_depth_workspace_bytes(2, 480, 640)
    assert ws >= 2 * 2 * 480 * 640 * 4 and ws < 2 * 2 * 480 * 640 * 4 + 8192
    assert lib.ffb6d_fill_depth_workspace_bytes(0, 480, 640) == 0
    assert lib.ffb6d_fill_depth_workspace_bytes(1, 0, 640) == 0
    assert lib.ffb6d_fill_depth(p, 1, 4, 4, 10000.0, None, None, p, 1 << 20, None) == _lib.ERR_INVALID   # no output
    assert "both outputs" in _lib.last_error()
    assert lib.ffb6d_fill_depth(p, 1, 4, 4, 0.0, p, None, p, 1 << 20, None) == _lib.ERR_INVALID        # cam_scale
    assert lib.ffb6d_fill_depth(p, 1, 4, 4, -2.0, p, None, p, 1 << 20, None) == _lib.ERR_INVALID
    assert lib.ffb6d_fill_depth(p, 1, 0, 4, 1.0, p, None, p, 1 << 20, None) == _lib.ERR_INVALID         # H = 0
    assert lib.ffb6d_fill_depth(p, -1, 4, 4, 1.0, p, None, p, 1 << 20, None) == _lib.ERR_INVALID
    assert lib.ffb6d_fill_depth(p, 1, 4, 4, 1.0, p, None, p, 16, None) == _lib.ERR_WORKSPACE
    assert lib.ffb6d_fill_depth(p, 1, 4, 4, 1.0, p, None, None, 0, None) == _lib.ERR_WORKSPACE
    assert lib.ffb6d_fill_depth(None, 0, 4, 4, 1.0, p, None, None, 0, None) == _lib.OK                # empty batch
