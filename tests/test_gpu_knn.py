"""GPU: the CUDA KNN index build, through the C ABI, against (a) the committed outputs of
the reference (tests/golden), (b) the CPU oracle on fresh seeded inputs, (c) size-independent
properties at BASELINE.json's full sizes.  Neighbour indices must be bit-exact (rows holding
exact fp32 distance ties: same sorted distances, DESIGN.md "tie contract")."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import GOLDEN, frame_point_sets
from oracle import cpu_oracle as O

pytestmark = pytest.mark.gpu

ALGOS = [1, 2, 0]        # tiled scan, uniform grid, automatic


def gpu_knn(sup, qry, k, algo=0, dtype=torch.int32):
    s = torch.from_numpy(np.ascontiguousarray(sup)).cuda()
    q = torch.from_numpy(np.ascontiguousarray(qry)).cuda()
    out = F.knn_search(s, q, k, out_dtype=dtype, algo=algo)
    assert out.dtype == dtype and out.is_cuda
    return out.cpu().numpy()


GOLD = ["self_768_k16", "interp_192_768_k1", "r2p_4800_192_k16", "p2r_192_4800_k1", "self_48_k16",
        "uniform_1000_500_k1", "uniform_1000_500_k8", "uniform_1000_500_k32", "k_gt_s_10_k16",
        "batch3_768_k16"]


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("name", GOLD)
def test_knn_golden_bit_exact(cuda, knn_golden, name, algo):
    c = knn_golden[name]
    sup, qry, want = c["support"], c["query"], c["idx"]
    if sup.ndim == 2:
        sup, qry, want = sup[None], qry[None], want[None]
    got = gpu_knn(sup, qry, int(c["k"]), algo)
    assert np.array_equal(got, want), O.knn_matches(sup, qry, got, want)[3]


@pytest.mark.parametrize("algo", ALGOS)
def test_knn_ties_contract(cuda, knn_golden, algo):
    c = knn_golden["ties_256_k8"]
    sup, qry, want = c["support"][None], c["query"][None], c["idx"][None]
    got = gpu_knn(sup, qry, int(c["k"]), algo)
    ok, _, _, msg = O.knn_matches(sup, qry, got, want)
    assert ok, msg
    # our own tie order is deterministic: lowest support index first == the oracle
    assert np.array_equal(got, O.knn_search(sup, qry, int(c["k"])))


def test_knn_host_abi_matches_reference_signature(cuda, knn_golden):
    """numpy in / numpy int32 out through ffb6d_knn_batch_host (signature of cpp_knn_batch_omp)."""
    c = knn_golden["batch3_768_k16"]
    got = F.knn_search(c["support"], c["query"], 16)
    assert isinstance(got, np.ndarray) and got.dtype == np.int32
    assert np.array_equal(got, c["idx"])
    got = F.DataProcessing.knn_search(c["support"][:1], c["query"][:1], 16)
    assert np.array_equal(got, c["idx"][:1])
    # non-contiguous / float64 inputs are marshalled like the Cython shim (NN/knn.pyx:95-96)
    sup64 = c["support"].astype(np.float64)[:, ::-1][:, ::-1]
    assert np.array_equal(F.knn_search(sup64, c["query"], 16), c["idx"])


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("seed,B,S,Q,K", [
    (0, 2, 500, 300, 16), (1, 1, 2000, 100, 1), (2, 3, 64, 64, 32), (3, 1, 5, 9, 8),
    (4, 2, 3000, 700, 4), (5, 1, 1, 1, 1), (6, 1, 100, 1000, 64), (7, 2, 1025, 257, 2),
    (8, 1, 20000, 33, 16), (9, 4, 300, 300, 3),
])
def test_knn_vs_oracle_random(cuda, seed, B, S, Q, K, algo):
    rs = np.random.RandomState(seed)
    sup = rs.randn(B, S, 3).astype(np.float32)
    qry = rs.randn(B, Q, 3).astype(np.float32)
    want = O.knn_search(sup, qry, K)
    for dt in (torch.int32, torch.int64):
        got = gpu_knn(sup, qry, K, algo, dt)
        assert np.array_equal(got, want), O.knn_matches(sup, qry, got, want)[3]


@pytest.mark.parametrize("algo", ALGOS)
def test_knn_degenerate_geometry(cuda, algo):
    """All points identical / collinear / one far outlier / queries far outside the support."""
    rs = np.random.RandomState(3)
    same = np.ones((1, 200, 3), np.float32) * 0.25
    line = np.zeros((1, 300, 3), np.float32)
    line[0, :, 0] = np.linspace(0, 1, 300)
    out = rs.rand(1, 400, 3).astype(np.float32)
    out[0, 17] = (1e4, -1e4, 1e4)
    far_q = (rs.rand(1, 50, 3).astype(np.float32) + 100.0)
    for sup, qry, k in ((same, same, 8), (line, line, 16), (out, out, 16), (out, far_q, 4),
                        (line, far_q, 1)):
        got = gpu_knn(sup, qry, k, algo)
        want = O.knn_search(sup, qry, k)
        ok, _, _, msg = O.knn_matches(sup, qry, got, want)
        assert ok, msg
        assert np.array_equal(got, want)          # same tie-break as the oracle (lowest index)


@pytest.mark.parametrize("algo", ALGOS)
def test_knn_empty_and_tiny(cuda, algo):
    sup = np.zeros((2, 7, 3), np.float32)
    assert gpu_knn(sup, np.zeros((2, 0, 3), np.float32), 4, algo).shape == (2, 0, 4)
    got = gpu_knn(np.zeros((1, 0, 3), np.float32), np.zeros((1, 5, 3), np.float32), 3, algo)
    assert got.shape == (1, 5, 3) and (got == 0).all()


@pytest.mark.parametrize("frame", ["seed0_n12288", "seed1_n12288", "seed2_n3072"])
def test_schedule_digest_full_frame(cuda, frame):
    """build_ffb6d_indices on a full 480x640 / 12288-point frame == the reference's 22 arrays
    (sha256 of the int32 arrays produced by the reference's compiled KNN)."""
    from ffb6d_b200.synthetic import make_frame
    d = json.load(open(os.path.join(GOLDEN, "schedule_digest.json")))["frames"][frame]
    fr = make_frame(d["seed"], n_points=d["n_points"])
    cld = torch.from_numpy(fr["cld"])[None].cuda()
    xyz = torch.from_numpy(fr["dpt_xyz"])[None].cuda()
    inputs = F.build_ffb6d_indices(cld, xyz)
    for key, meta in d["keys"].items():
        got = inputs[key][0].cpu().numpy()
        assert got.dtype == np.int32 and list(got.shape) == meta["shape"], key
        assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == meta["sha256"], key
    for i in range(4):
        n = d["n_points"] // 4 ** i
        assert inputs["cld_xyz%d" % i].shape == (1, n, 3)
        assert torch.equal(inputs["cld_sub_idx%d" % i], inputs["cld_nei_idx%d" % i][:, : n // 4])


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_native_schedule_entry_point(cuda, dtype):
    """ffb6d_build_indices (one C call, caller-owned buffers and workspace) == the reference's 22 arrays
    for a full frame (golden sha256) and == the Python scheduler on a second, batched input."""
    from ffb6d_b200.schedule import image_pyramid
    from ffb6d_b200.synthetic import make_frame, make_batch
    d = json.load(open(os.path.join(GOLDEN, "schedule_digest.json")))["frames"]["seed0_n12288"]
    fr = make_frame(d["seed"], n_points=d["n_points"])
    cld = torch.from_numpy(fr["cld"])[None].cuda()
    xyz = torch.from_numpy(fr["dpt_xyz"])[None].cuda()
    pyr = image_pyramid(xyz, (2, 4, 8))
    got = F.build_ffb6d_indices_native(cld, pyr, xyz.shape[1:3], index_dtype=dtype)
    for key, meta in d["keys"].items():
        g = got[key][0].cpu().numpy()
        assert g.dtype == (np.int32 if dtype == torch.int32 else np.int64) and list(g.shape) == meta["shape"], key
        assert hashlib.sha256(np.ascontiguousarray(g.astype(np.int32)).tobytes()).hexdigest() == meta["sha256"], key
    batch = make_batch(range(40, 43), n_points=3072)
    cld = torch.from_numpy(batch["cld"]).cuda()
    xyz = torch.from_numpy(batch["dpt_xyz"]).cuda()
    want = F.build_ffb6d_indices(cld, xyz, index_dtype=dtype)
    got = F.build_ffb6d_indices_native(cld, image_pyramid(xyz, (2, 4, 8)), xyz.shape[1:3], index_dtype=dtype)
    assert set(got) == set(want)
    for key in want:
        assert torch.equal(got[key], want[key]), key
    # error behaviour: short workspace / bad sizes are reported, not executed
    from ffb6d_b200._lib import lib
    assert lib.ffb6d_build_indices_workspace_bytes(1, 100, 480, 640, 16) == 0
    with pytest.raises(Exception):
        F.build_ffb6d_indices_native(cld[:, :1000], image_pyramid(xyz, (2, 4, 8)), xyz.shape[1:3])


def test_schedule_properties_at_full_batch(cuda):
    """BASELINE config 2 sizes (B=32 is sharded here as 4 frames to bound memory/time of the
    CPU checks): size-independent properties of every one of the 22 index tensors."""
    from ffb6d_b200.synthetic import make_batch
    from ffb6d_b200.schedule import knn_schedule
    B = 4
    batch = make_batch(range(100, 100 + B))
    cld = torch.from_numpy(batch["cld"]).cuda()
    xyz = torch.from_numpy(batch["dpt_xyz"]).cuda()
    inputs = F.build_ffb6d_indices(cld, xyz)
    rs = np.random.RandomState(0)
    for b in range(B):
        ps = frame_point_sets({"cld": batch["cld"][b], "dpt_xyz": batch["dpt_xyz"][b]}, 12288)
        for key, s, q, k in knn_schedule():
            idx = inputs[key][b].cpu().numpy()
            S, Q = len(ps[s]), len(ps[q])
            assert idx.shape == (Q, k) and idx.min() >= 0 and idx.max() < S, key
            rows = rs.choice(Q, size=min(Q, 64), replace=False)
            d = O.sqdist_of_indices(ps[s][None], ps[q][None][:, rows], idx[None][:, rows])[0]
            assert (np.diff(d, axis=1) >= 0).all(), key                       # ascending
            # exact check of the sampled rows against the oracle
            want = O.knn_search(ps[s][None], ps[q][None][:, rows], k)[0]
            assert np.array_equal(idx[rows], want), key
            if s == q:                                                        # self is nearest
                assert (idx[:, 0] == np.arange(Q)).all(), key
    # batch items are independent: frame 0 alone gives the same indices
    solo = F.build_ffb6d_indices(cld[:1], xyz[:1])
    for key in solo:
        assert torch.equal(solo[key][0], inputs[key][0]), key


def test_knn_grid_build_once_query_many(cuda):
    """KnnGrid: one grid, several searches with different K and query sets == knn_search."""
    rs = np.random.RandomState(12)
    sup = rs.rand(2, 5000, 3).astype(np.float32) * np.array([1.0, 0.8, 0.2], np.float32)
    q1 = rs.rand(2, 700, 3).astype(np.float32)
    q2 = (rs.rand(2, 50, 3).astype(np.float32) - 3.0)          # far outside -> overflow path
    q2[:, 10:30] = 0.0                                          # equal far queries (+0.0 / -0.0)
    q2[:, 20:30, 0] = -0.0
    ts = torch.from_numpy(sup).cuda()
    grid = F.KnnGrid(ts, 16)
    for q, k in ((q1, 16), (q1, 1), (q2, 16), (q2, 1), (q1, 7), (q1, 33)):
        got = grid.query(torch.from_numpy(q).cuda(), k).cpu().numpy()
        assert np.array_equal(got, O.knn_search(sup, q, k)), (q.shape, k)
    got = grid.query(ts, 16, out_dtype=torch.int64).cpu().numpy()              # self search
    assert np.array_equal(got, O.knn_search(sup, sup, 16))


@pytest.mark.parametrize("k", [8, 16, 32])
@pytest.mark.parametrize("n_points", [4096, 12288, 40960, 131072])
def test_stress_sweep_sizes(cuda, n_points, k):
    """BASELINE configs[4]: all 12 cells of N in {4096, 12288, 40960, 131072} x K in {8, 16, 32} on one
    frame: every index tensor of the schedule against the oracle -- EVERY row for N <= 12288, 256 sampled
    rows above -- plus range / self-first properties."""
    from ffb6d_b200.synthetic import make_frame
    from ffb6d_b200.schedule import knn_schedule
    fr = make_frame(31, n_points=n_points)
    cld = torch.from_numpy(fr["cld"])[None].cuda()
    xyz = torch.from_numpy(fr["dpt_xyz"])[None].cuda()
    inputs = F.build_ffb6d_indices(cld, xyz, k=k)
    ps = frame_point_sets(fr, n_points)
    rs = np.random.RandomState(1)
    for key, s, q, kk in knn_schedule(n_points, k=k):
        idx = inputs[key][0].cpu().numpy()
        S, Q = len(ps[s]), len(ps[q])
        assert idx.shape == (Q, kk) and idx.min() >= 0 and idx.max() < S, key
        rows = np.arange(Q) if n_points <= 12288 else np.sort(rs.choice(Q, size=min(Q, 256), replace=False))
        want = O.knn_search(ps[s][None], ps[q][None][:, rows], kk)[0]
        ok, _, _, msg = O.knn_matches(ps[s][None], ps[q][None][:, rows], idx[None][:, rows], want[None])
        assert ok, "%s: %s" % (key, msg)
        if s == q:
            assert (idx[:, 0] == np.arange(Q)).all(), key


def test_knn_organised_queries_tile_path(cuda):
    """K = 1 with the `query_width` layout hint (one warp per 8x4 pixel tile sharing a candidate box) gives
    exactly the result of the plain search: image shapes that do not divide into tiles, hole pixels at the
    origin (+0.0 / -0.0), a depth discontinuity (box too large -> per-thread finish), NaN queries."""
    from ffb6d_b200.synthetic import make_frame, image_pyramid_np
    fr = make_frame(9, n_points=3072)
    pyr = image_pyramid_np(fr["dpt_xyz"])
    rs = np.random.RandomState(5)
    cases = []
    for sr, (hh, ww) in ((8, (60, 80)), (4, (120, 160))):
        q = pyr[sr].reshape(hh, ww, 3).copy()
        cases.append((q, ww))
        cut = q[: hh - 3, : ww - 6].copy()                      # 57 x 74 / 117 x 154: ragged tiles
        cut[5:9, 10:30, 2] += 0.6                                # a step in depth inside tiles
        cut[20, 20] = np.nan
        cut[21, 21:25] = -0.0
        cases.append((cut, ww - 6))
    sup = np.stack([fr["cld"][:3072], fr["cld"][:3072] * np.array([1.0, 1.0, 1.1], np.float32)])
    grid = F.KnnGrid(torch.from_numpy(sup).cuda(), 1)
    for img, ww in cases:
        q = np.stack([img.reshape(-1, 3), img[::-1].reshape(-1, 3)]).astype(np.float32)
        tq = torch.from_numpy(q).cuda()
        plain = grid.query(tq, 1).cpu().numpy()
        tiled = grid.query(tq, 1, query_width=ww).cpu().numpy()
        assert np.array_equal(plain, tiled), (img.shape, ww)
        ok = ~np.isnan(q).any(axis=2)
        want = O.knn_search(sup, np.nan_to_num(q), 1)
        assert np.array_equal(tiled[ok], want[ok])
        for dt in (torch.int64,):
            assert np.array_equal(grid.query(tq, 1, out_dtype=dt, query_width=ww).cpu().numpy(), tiled)


@pytest.mark.parametrize("k", [2, 31, 32, 33, 64])
def test_knn_all_k_paths(cuda, k):
    """warp-per-query (K <= 32) and thread-per-query (K > 32) searches, overflow paths included."""
    rs = np.random.RandomState(k)
    sup = (rs.rand(2, 6000, 3) * np.array([1.0, 1.0, 0.05])).astype(np.float32)
    qry = np.concatenate([rs.rand(2, 500, 3).astype(np.float32), rs.rand(2, 40, 3).astype(np.float32) + 5.0], 1)
    qry[:, 520:530] = 0.0
    for algo in (2, 1):
        got = gpu_knn(sup, qry, k, algo)
        assert np.array_equal(got, O.knn_search(sup, qry, k)), (k, algo)


def test_bench_cli_small(cuda):
    """bench.py end to end on a tiny configuration: one JSON line with the contract's keys."""
    import subprocess
    import sys
    from conftest import ROOT
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--batch", "2", "--n-points", "3072",
                          "--steps", "3", "--warmup", "3", "--no-cpu-baseline", "--no-mlp"],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, out.stdout[-2000:]
    d = json.loads(lines[0])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "clocks"):
        assert key in d, key
    assert d["value"] > 0 and d["gpu_launches"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0
    assert 0 < d["roofline"]["frac"] and d["roofline"]["bound"] == "hbm"
