"""GPU: farthest point sampling (ffb6d_farthest_point_sampling, ops.farthest_point_sampling) against the indices the
reference's compiled farthest_point_sampling.cpp selects (tests/golden/fps_cases.npz, cases in tests/fps_cases.py).

Bitwise parity of every index: with init_center the run is deterministic; from a random start the device is given
the reference's own start (its first index), which pins every later round."""
import os

import numpy as np
import pytest
import torch

import fps_cases as FC
from conftest import GOLDEN
from ffb6d_b200 import ops
from ffb6d_b200._lib import lib, check, FPS_MAX_CLOUDS, FPS_MAX_POINTS, FPS_MAX_SAMPLES
from ffb6d_b200.ops import _stream

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "fps_cases.npz"))
    return {k: z[k] for k in z.files}


def _run(pts, S, init_center, start=None, counts=None):
    """The C entry point on a [G,P,3] tensor; returns idx [G,S] on the host."""
    G, P, _ = pts.shape
    idx = torch.full((G, S), -7, dtype=torch.int32, device=pts.device)
    st = None if start is None else torch.as_tensor(np.asarray(start, np.int32), device=pts.device)
    cn = None if counts is None else torch.as_tensor(np.asarray(counts, np.int32), device=pts.device)
    check(lib.ffb6d_farthest_point_sampling(pts.data_ptr(), cn.data_ptr() if cn is not None else None, G, P, S,
                                            st.data_ptr() if st is not None else None, int(init_center),
                                            idx.data_ptr(), None, 0, _stream(pts.device)))
    return idx.cpu().numpy()


@pytest.mark.parametrize("name", list(FC.CASES))
def test_cases_match_reference(cuda, golden, name):
    make, S = FC.CASES[name]
    pts = make()
    want_ic, want_rs = golden[name + ":ic"], golden[name + ":rs"]
    got, idx = ops.farthest_point_sampling(pts, S, init_center=True, return_index=True)
    assert np.array_equal(idx, want_ic)
    assert np.array_equal(got, pts[want_ic])                                   # fps_utils returns pts[idxs]
    idx = ops.farthest_point_sampling(torch.from_numpy(pts).to(cuda), S, start=int(want_rs[0]), return_index=True)[1]
    assert np.array_equal(idx.cpu().numpy(), want_rs)


def test_batch_equals_single_calls(cuda, golden):
    clouds = torch.from_numpy(FC.batch_clouds()).to(cuda)
    S = golden["batch:ic"].shape[1]
    assert np.array_equal(_run(clouds, S, True), golden["batch:ic"])
    start = golden["batch:rs"][:, 0]
    got = ops.farthest_point_sampling(clouds, S, start=torch.from_numpy(start).to(cuda), return_index=True)[1]
    assert np.array_equal(got.cpu().numpy(), golden["batch:rs"])
    for g in range(FC.BATCH_G):
        assert np.array_equal(_run(clouds[g:g + 1], S, True)[0], golden["batch:ic"][g])
        assert np.array_equal(_run(clouds[g:g + 1], S, False, start=start[g:g + 1])[0], golden["batch:rs"][g])


def test_ragged_batch(cuda, golden):
    clouds = torch.from_numpy(FC.batch_clouds()).to(cuda)
    S = golden["ragged:ic"].shape[1]
    assert np.array_equal(_run(clouds, S, True, counts=FC.BATCH_N), golden["ragged:ic"])
    got = ops.farthest_point_sampling(clouds, S, init_center=True, n_points=list(FC.BATCH_N), return_index=True)[1]
    assert np.array_equal(got.cpu().numpy(), golden["ragged:ic"])


def test_device_side_out_of_range_rows(cuda, golden):
    """A start or count the host did not check gives its cloud a row of -1; the other clouds are unaffected."""
    clouds = torch.from_numpy(FC.batch_clouds()).to(cuda)
    S = golden["batch:rs"].shape[1]
    start = golden["batch:rs"][:, 0].copy()
    start[1], start[3] = FC.BATCH_P, -1
    got = _run(clouds, S, False, start=start)
    for g in range(FC.BATCH_G):
        assert np.array_equal(got[g], np.full(S, -1) if g in (1, 3) else golden["batch:rs"][g])
    counts = list(FC.BATCH_N)
    counts[0], counts[2] = 0, FC.BATCH_P + 1
    got = _run(clouds, S, True, counts=counts)
    for g in range(FC.BATCH_G):
        assert np.array_equal(got[g], np.full(S, -1) if g in (0, 2) else golden["ragged:ic"][g])


def test_random_start_is_a_farthest_point_run(cuda, golden):
    """start=None draws the first index on the device; the rest is the reference's run from that index."""
    pts = FC.CASES["n1025"][0]()
    torch.manual_seed(5)
    idx = ops.farthest_point_sampling(torch.from_numpy(pts).to(cuda), 24, return_index=True)[1].cpu().numpy()
    again = ops.farthest_point_sampling(pts, 24, start=int(idx[0]), return_index=True)[1]
    assert 0 <= idx[0] < len(pts) and np.array_equal(idx, again) and len(set(idx.tolist())) == 24


def test_captures_in_cuda_graph(cuda, golden):
    clouds = torch.from_numpy(FC.batch_clouds()).to(cuda)
    S = golden["batch:ic"].shape[1]
    start = torch.from_numpy(golden["batch:rs"][:, 0].copy()).to(cuda)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.farthest_point_sampling(clouds, S, init_center=True)               # warm-up: smem opt-in, module load
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ic = ops.farthest_point_sampling(clouds, S, init_center=True, return_index=True)[1]
        rs = ops.farthest_point_sampling(clouds, S, start=start, return_index=True)[1]
    for _ in range(2):
        ic.fill_(-5)
        rs.fill_(-5)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(ic.cpu().numpy(), golden["batch:ic"])
        assert np.array_equal(rs.cpu().numpy(), golden["batch:rs"])


# ------------------------------------------------------------------ size limits
def test_limits_match_header():
    assert FC.MAX_POINTS == FPS_MAX_POINTS and FC.MAX_SAMPLES == FPS_MAX_SAMPLES and FPS_MAX_CLOUDS == 65535


def test_largest_cloud_and_most_samples(cuda, golden):
    """P = FFB6D_FPS_MAX_POINTS (a cluster of 8 CTAs) and S = FFB6D_FPS_MAX_SAMPLES are in the cases above; one past
    either is refused before any launch."""
    assert FC.CASES["max_points"][0]().shape[0] == FPS_MAX_POINTS
    assert FC.CASES["max_samples"][1] == FPS_MAX_SAMPLES
    pts = torch.zeros((1, FPS_MAX_POINTS + 1, 3), device=cuda)
    with pytest.raises(ValueError):
        ops.farthest_point_sampling(pts, 8, init_center=True)
    with pytest.raises(ValueError):
        ops.farthest_point_sampling(pts[:, :10], FPS_MAX_SAMPLES + 1, init_center=True)


def test_most_clouds(cuda, golden):
    """G = FFB6D_FPS_MAX_CLOUDS (grid.y): the batch's clouds tiled over 65535 rows, each row its cloud's answer."""
    clouds = torch.from_numpy(FC.batch_clouds()).to(cuda)
    rows = torch.arange(FPS_MAX_CLOUDS, device=cuda) % FC.BATCH_G
    S = 8
    got = _run(clouds[rows].contiguous(), S, True)
    want = golden["batch:ic"][:, :S][rows.cpu().numpy()]
    assert np.array_equal(got, want)
    start = golden["batch:rs"][:, 0][rows.cpu().numpy()]
    got = _run(clouds[rows].contiguous(), S, False, start=start)
    assert np.array_equal(got, golden["batch:rs"][:, :S][rows.cpu().numpy()])
    with pytest.raises(ValueError):
        ops.farthest_point_sampling(torch.zeros((FPS_MAX_CLOUDS + 1, 2, 3), device=cuda), 1, init_center=True)
