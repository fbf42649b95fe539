"""GPU: depth completion (ffb6d_fill_depth / ops.fill_missing) against the reference's outputs in
tests/golden/fill_cases.npz and against the numpy oracle on seeded frames of odd sizes; the raw-depth index
build against its explicit composition, eagerly and through a captured CUDA graph."""
import os

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import GOLDEN, _npz_groups
from oracle import fill_oracle as O
from ffb6d_b200.synthetic import FILL_CAM_SCALE, INTRINSICS, fill_test_frames, make_raw_depth
from test_fill_oracle import assert_fill_contract, assert_matches_golden, sha

pytestmark = pytest.mark.gpu
CS = np.float32(FILL_CAM_SCALE)
MSK_DP = np.float32(1e-6)


def dev_raw(raw, cuda):
    return torch.from_numpy(np.ascontiguousarray(raw, dtype=np.uint16)).to(cuda)


def blurred_mask(raw):
    return O.fill_missing(raw, CS, return_stages=True)[1]["bilateral_mask"]


@pytest.fixture(scope="module")
def golden():
    return _npz_groups(os.path.join(GOLDEN, "fill_cases.npz"))


@pytest.mark.parametrize("name", sorted(fill_test_frames()))
def test_golden_frames_meet_contract(cuda, golden, name):
    raw = fill_test_frames()[name]
    got = F.fill_missing(dev_raw(raw, cuda), CS).cpu().numpy()
    assert got.shape == raw.shape
    assert_matches_golden(got, blurred_mask(raw), golden[name], FILL_CAM_SCALE)


@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (3, 7, 5), (2, 37, 91), (1, 480, 640), (8, 45, 61)])
def test_random_frames_match_oracle(cuda, B, H, W):
    raws = np.stack([make_raw_depth(1000 + 17 * b + H, h=H, w=W) for b in range(B)])
    got = F.fill_missing(dev_raw(raws, cuda), CS).cpu().numpy()
    for b in range(B):
        want, st = O.fill_missing(raws[b], CS, return_stages=True)
        assert_fill_contract(got[b], want, st["bilateral_mask"], FILL_CAM_SCALE)
        one = F.fill_missing(dev_raw(raws[b], cuda), CS).cpu().numpy()          # [H,W] input, one frame
        assert np.array_equal(one.view(np.uint32), got[b].view(np.uint32)), b


def test_batch_determinism_and_metres(cuda):
    from ffb6d_b200.ops import _fill_depth
    raws = dev_raw(np.stack([make_raw_depth(s) for s in range(4)]), cuda)
    a = F.fill_missing(raws, CS)
    b = F.fill_missing(raws, CS)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    filled, depth_m = _fill_depth(raws, CS)
    assert torch.equal(filled.view(torch.int32), a.view(torch.int32))
    ref_m = filled / torch.tensor(CS, dtype=torch.float32, device=cuda)        # IEEE division on the device
    assert torch.equal(depth_m.view(torch.int32), ref_m.view(torch.int32))
    only_m = _fill_depth(raws, CS, want_raw=False)[1]
    assert torch.equal(only_m.view(torch.int32), depth_m.view(torch.int32))


def _composition(raw, K, n, seed):
    filled = F.fill_missing(raw, CS)
    depth_m = filled / torch.tensor(CS, dtype=torch.float32, device=raw.device)
    choose = F.sample_valid_pixels(filled, n, seed=seed, min_depth=1e-6)
    out = F.build_ffb6d_indices_from_depth(depth_m, K, choose)
    out["choose"], out["dpt_map_m"] = choose, depth_m
    return out


def test_indices_from_raw_depth_equal_composition(cuda, golden):
    frames = fill_test_frames()
    raw = dev_raw(np.stack([frames["full0"], frames["full1"]]), cuda)
    K = INTRINSICS["ycb_K1"]
    got = F.build_ffb6d_indices_from_raw_depth(raw, CS, K, 12288, seed=3)
    want = _composition(raw, K, 12288, 3)
    assert set(got) == set(want)
    for key, w in want.items():
        assert got[key].dtype == w.dtype and torch.equal(got[key], w), key
    filled = F.fill_missing(raw, CS).cpu().numpy()
    for b, name in enumerate(("full0", "full1")):
        msk_dp = filled[b] > MSK_DP
        assert sha(msk_dp) == str(golden[name]["sha256_msk_dp"]), name                 # the reference's msk_dp
        assert msk_dp.reshape(-1)[got["choose"][b, 0].cpu().numpy()].all(), name


def test_indices_from_raw_depth_graph_replay(cuda):
    from ffb6d_b200.ops import intrinsics_to_device
    raw = dev_raw(np.stack([make_raw_depth(s) for s in (5, 6)]), cuda)
    intr = intrinsics_to_device(INTRINSICS["ycb_K1"], cuda)
    want = F.build_ffb6d_indices_from_raw_depth(raw, CS, intr, 12288, seed=9)
    torch.cuda.synchronize()
    side = torch.cuda.Stream(device=cuda)
    side.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(side):
        F.build_ffb6d_indices_from_raw_depth(raw, CS, intr, 12288, seed=9)
    torch.cuda.current_stream(cuda).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = F.build_ffb6d_indices_from_raw_depth(raw, CS, intr, 12288, seed=9)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for key, w in want.items():
            assert torch.equal(got[key], w), key
