"""CPU: the oracle against outputs of the reference's own code (its compiled KNN and grid
subsampling, its torch gathers) on seeded inputs, stored in tests/golden/refcheck_cases.npz by
tests/golden/make_golden.py; the inputs are regenerated here from the same seeds."""
import os
import sys

import numpy as np
import pytest

from oracle import cpu_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden as G  # noqa: E402


@pytest.fixture(scope="module")
def ref():
    from conftest import GOLDEN
    z = np.load(os.path.join(GOLDEN, "refcheck_cases.npz"))
    return {k: z[k] for k in z.files}


@pytest.mark.parametrize("seed,S,Q,K", G.KNN_RANDOM)
def test_knn_random(ref, seed, S, Q, K):
    rs = np.random.RandomState(seed)
    sup = rs.randn(2, S, 3).astype(np.float32)
    qry = rs.randn(2, Q, 3).astype(np.float32)
    want = ref["knn_random/%d" % seed].astype(np.int64)
    got = O.knn_batch(sup, qry, K)
    ok, ndiff, _, msg = O.knn_matches(sup, qry, got, want)
    assert ok and ndiff == 0, msg


def test_knn_surface_frame(ref):
    from ffb6d_b200.synthetic import make_frame
    fr = make_frame(9, n_points=3072)
    cld = fr["cld"][None]
    assert np.array_equal(O.knn_batch(cld, cld, 16), ref["surface_frame/idx"].astype(np.int64))


@pytest.mark.parametrize("n_points", G.STRESS_SIZES)
def test_knn_stress_sweep_sizes(ref, n_points):
    """BASELINE configs[4] sizes: the port still equals the reference's KD-tree on the big clouds
    (self search K = 16 on level 1, image -> cloud K = 1 and cloud -> image K = 32 on level 2), on a
    seeded sample of query rows."""
    # dense clouds do produce the odd exact fp32 distance tie (seen: one row of 10240 at N0 = 40960), and
    # the hole pixels of the image level are exact duplicates: rows may then differ in ORDER only
    for name, sup, qry, k in G.stress_searches(n_points):
        q = qry[:, G.stress_rows(qry.shape[1], n_points)]
        got, want = O.knn_batch(sup, q, k), ref["stress/%d_%s" % (n_points, name)].astype(np.int64)
        ok, ndiff, nties, msg = O.knn_matches(sup, q, got, want)
        assert ok and ndiff == nties, msg
        assert ndiff <= max(4, q.shape[1] // 1000) or name == "cld2img", msg


def test_torch_ops_random(ref):
    import torch
    g = torch.Generator().manual_seed(7)
    feat = torch.randn(3, 17, 211, 1, generator=g)
    idx = torch.randint(0, 211, (3, 50, 16), generator=g)
    assert np.array_equal(ref["torch/random_sample"], O.random_sample(feat.numpy(), idx.numpy()))
    idx1 = torch.randint(0, 211, (3, 400, 1), generator=g)
    assert np.array_equal(ref["torch/nearest_interpolation"], O.nearest_interpolation(feat.numpy(), idx1.numpy()))
    pc = torch.randn(2, 90, 6, generator=g)
    nidx = torch.randint(0, 90, (2, 90, 16), generator=g)
    assert np.array_equal(ref["torch/gather_neighbour"], O.gather_neighbour(pc.numpy(), nidx.numpy()))


def test_grid_random(ref):
    rs = np.random.RandomState(5)
    pts = (rs.randn(4000, 3) * 0.5).astype(np.float32)
    feats = rs.rand(4000, 3).astype(np.float32)
    op, of, _ = O.grid_sub_sampling(pts, feats, None, 0.07)
    o2 = np.lexsort((op[:, 2], op[:, 1], op[:, 0]))
    assert np.array_equal(ref["grid/points"], op[o2]) and np.array_equal(ref["grid/features"], of[o2])


def test_wrap_padded_frame_tie_order_differs_but_gathers_agree(ref):
    """A frame padded with repeated pixels (np.pad 'wrap', ycb_dataset.py:230): thousands of index rows differ
    between the reference's KD-tree order and the (distance, index) order -- within the tie contract -- yet every
    gather of the forward pass returns the same values, because tied points are duplicates with identical features."""
    from ffb6d_b200.tables import gather_schedule, knn_schedule
    n = 3072
    _, sets, rs = G.wrap_padded_frame(n)
    refi, ours, differing = {}, {}, 0
    for key, s, q, kk in knn_schedule(n):
        refi[key] = ref["wrap_padded/" + key]
        ours[key] = O.knn_search(sets[s][None], sets[q][None], kk)
        ok, _, _, msg = O.knn_matches(sets[s][None], sets[q][None], ours[key], refi[key])
        assert ok, (key, msg)
        differing += int((refi[key] != ours[key]).any(axis=2).sum())
    assert differing > 1000
    for d in (refi, ours):
        d.update({"cld_sub_idx%d" % i: d["cld_nei_idx%d" % i][:, : n // 4 ** (i + 1)] for i in range(4)})
    support_of = {key: s for key, s, q, kk in knn_schedule(n)}
    for op, key, C, S, Q, K in gather_schedule(n):
        if op == "choose":
            continue
        pts = sets[support_of[key.replace("cld_sub_idx", "cld_nei_idx")]]
        w = rs.normal(size=(min(C, 16), 3)).astype(np.float32)
        feat = np.sin(pts @ w.T * 7.0).T[None, :, :, None].astype(np.float32).copy()     # features = f(xyz)
        f = O.random_sample if op == "random_sample" else O.nearest_interpolation
        assert np.array_equal(f(feat, refi[key].astype(np.int64)), f(feat, ours[key].astype(np.int64))), key
