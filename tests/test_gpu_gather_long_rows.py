"""GPU: the gathers from rows too long to stage (the `choose` gather and the K-lane r2p gathers), bitwise against
torch.gather (+ max over K) on the same device, at the pass's shapes and at the edges of the kernels' tiling."""
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib

pytestmark = pytest.mark.gpu

H, W = 480, 640


def _want(feat, idx):
    """torch's expression: gather the K neighbours of every query, max over K (models/ffb6d.py:166-177)."""
    B, C, S = feat.shape
    Q, K = idx.shape[1], idx.shape[2]
    g = torch.gather(feat, 2, idx.long().reshape(B, 1, Q * K).expand(B, C, Q * K))
    return g.reshape(B, C, Q, K).max(dim=3)[0]


def _same(got, want):
    """Bitwise equal, NaN at the same places (a NaN's payload is not part of torch.max's contract)."""
    got = got.reshape(want.shape)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32))


def _kernel(B, C, S, Q, K):
    return _lib.lib.ffb6d_gather_kernel_name(B, C, S, Q, K, 0).decode()


def _feat(B, C, S, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    f = torch.randn(B, C, S, device="cuda", generator=g)
    f[:, ::7, ::101] = float("nan")
    f[:, 1::5, ::89] = float("-inf")
    return f


def _patch_idx(B, S, Q, K, seed):
    """K neighbours per query in a 5x5 window of the image level around a random centre, like the r2p searches."""
    w = {19200: 160, 76800: 320, 4800: 80}.get(S, 64)
    g = torch.Generator(device="cuda").manual_seed(seed)
    centre = torch.randint(0, S, (B, Q, 1), device="cuda", generator=g)
    off = torch.randint(-2, 3, (B, Q, K), device="cuda", generator=g) * w + \
        torch.randint(-2, 3, (B, Q, K), device="cuda", generator=g)
    return (centre + off).clamp_(0, S - 1)


# (C, S, Q) of the `choose` gather and of the K-lane r2p gathers of the pass (tables.gather_schedule)
CHOOSE = (64, H * W, 12288)
R2P = [(1024, 4800, 48), (256, 19200, 192), (64, 76800, 768), (64, 76800, 3072)]


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("B", [1, 32])
def test_choose_shape(cuda, B, idx_dtype):
    C, S, Q = CHOOSE
    assert _kernel(B, C, S, Q, 1) == "gather1_ncs_direct_kernel"
    feat = _feat(B, C, S, B)
    g = torch.Generator(device="cuda").manual_seed(7)
    idx = torch.stack([torch.randperm(S, device="cuda", generator=g)[:Q] for _ in range(B)]).to(idx_dtype)
    got = F.choose_gather(feat.reshape(B, C, H, W), idx.reshape(B, 1, Q))
    _same(got, _want(feat, idx.reshape(B, Q, 1)))


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("B", [1, 32])
@pytest.mark.parametrize("shape", R2P, ids=lambda s: "C%d-S%d-Q%d" % s)
def test_r2p_shapes(cuda, shape, B, idx_dtype):
    C, S, Q = shape
    assert _kernel(B, C, S, Q, 16) == "gather_max_ncs_klane_kernel"
    feat = _feat(B, C, S, C + Q)
    idx = _patch_idx(B, S, Q, 16, Q).to(idx_dtype)
    _same(F.random_sample(feat, idx), _want(feat, idx))


@pytest.mark.parametrize("K", [8, 16, 32])
@pytest.mark.parametrize("shape", [(37, 76800, 1001), (5, 40000, 1), (3, 76800, 7)], ids=lambda s: "C%d-S%d-Q%d" % s)
def test_klane_partial_tiles(cuda, shape, K):
    """C not a multiple of the channel group, Q not a multiple of the queries per CTA (and below one CTA)."""
    C, S, Q = shape
    assert _kernel(2, C, S, Q, K) == "gather_max_ncs_klane_kernel"
    feat = _feat(2, C, S, K)
    idx = _patch_idx(2, S, Q, K, C)
    for ii in (idx, idx.int()):
        _same(F.random_sample(feat, ii), _want(feat, ii))


@pytest.mark.parametrize("shape", [(3, 13, 1000), (2, 1, 5), (1, 3, 12288)], ids=lambda s: "B%d-C%d-Q%d" % s)
def test_choose_partial(cuda, shape):
    """Channel counts that are not a multiple of a thread's channels, Q not a multiple of the CTA."""
    B, C, Q = shape
    S = H * W
    assert _kernel(B, C, S, Q, 1) == "gather1_ncs_direct_kernel"
    feat = _feat(B, C, S, Q)
    idx = torch.randint(0, S, (B, Q, 1), device="cuda", generator=torch.Generator(device="cuda").manual_seed(Q))
    for ii in (idx, idx.int()):
        _same(F.nearest_interpolation(feat.unsqueeze(3), ii), _want(feat, ii))


def test_duplicates_one_row_and_last_pixel(cuda):
    """'wrap' padding (every pick repeated), all picks in one image row, the last pixel of the map."""
    B, C, S, Q = 2, 64, H * W, 12288
    feat = _feat(B, C, S, 3)
    g = torch.Generator(device="cuda").manual_seed(4)
    wrap = torch.randperm(S, device="cuda", generator=g)[:1000].repeat(13)[:Q]
    row = 211 * W + torch.randint(0, W, (Q,), device="cuda", generator=g)
    idx = torch.stack([wrap, row])[:, :, None]
    idx[1, -1, 0] = S - 1
    _same(F.nearest_interpolation(feat.unsqueeze(3), idx), _want(feat, idx))
    # K = 16 with every neighbour of every query in one image row, and all queries of a frame on the same patch
    C, S, Q = 64, 76800, 768
    feat = _feat(B, C, S, 5)
    idx = torch.randint(100 * 320, 101 * 320, (B, Q, 16), device="cuda", generator=g)
    idx[1] = idx[1, :1]
    idx[0, 0, 0] = S - 1
    _same(F.random_sample(feat, idx), _want(feat, idx))


def test_graph_replay(cuda):
    """Both kernels captured in a CUDA graph and replayed on new inputs written in place."""
    B = 2
    C1, S1, Q1 = CHOOSE
    C2, S2, Q2 = R2P[2]
    f1, f2 = _feat(B, C1, S1, 1), _feat(B, C2, S2, 2)
    i1 = torch.randint(0, S1, (B, Q1, 1), device="cuda")
    i2 = _patch_idx(B, S2, Q2, 16, 3)
    F.nearest_interpolation(f1.unsqueeze(3), i1)
    F.random_sample(f2, i2)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o1 = F.nearest_interpolation(f1.unsqueeze(3), i1)
        o2 = F.random_sample(f2, i2)
    for seed in (10, 11):
        f1.copy_(_feat(B, C1, S1, seed))
        f2.copy_(_feat(B, C2, S2, seed))
        i1.copy_(torch.randint(0, S1, (B, Q1, 1), device="cuda"))
        i2.copy_(_patch_idx(B, S2, Q2, 16, seed))
        graph.replay()
        torch.cuda.synchronize()
        _same(o1, _want(f1, i1))
        _same(o2, _want(f2, i2))
