"""GPU: the fused attentive pooling (``ops.lfa_att_pool_fused``, lfa_fused.cu) against the float64 oracle
(oracle/lfa_oracle.py, itself pinned to the reference's modules by tests/test_lfa_oracle.py) over every width the
kernel is built for, with and without the encoding's second MLP, output widths below, between and at the multiples
of the 32-lane loop, batches of several frames, more points than one pass of the persistent grid, degenerate
neighbourhoods and saturated or uniform attention.  Bound: tests/test_gpu_lfa.py's ``close`` (1e-5 of the output
scale, 1e-4 element-wise above 10 % of it), widened to 4x the error of the same composition in torch fp32 where
that is larger."""
import pytest
import torch

from ffb6d_b200 import ops
from oracle import lfa_oracle as L

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (1, 7), (3, 1), (3, 7), (1, 12288), (3, 12288)]     # (B, N)


def make_layers(Dh, Do, mlp2, seed):
    g = torch.Generator().manual_seed(seed)

    def layer(co, ci):
        return ((torch.randn(co, ci, generator=g) / ci ** 0.5).cuda(), (torch.rand(co, generator=g) + 0.5).cuda(),
                (torch.randn(co, generator=g) * 0.1).cuda())
    m1 = layer(Dh, 10)
    m2 = layer(Dh, Dh) if mlp2 else None
    fc = (torch.randn(2 * Dh, 2 * Dh, generator=g) / (2 * Dh) ** 0.5).cuda()
    return m1, m2, fc, layer(Do, 2 * Dh)


def make_points(B, N, Dh, pattern, seed):
    """xyz [B, N, 3], features [B, d/2, N, 1] and a neighbour pattern [B, N, 16] (int64): random neighbours, every
    neighbour the point itself (distance 0), all 16 one random point, or all 16 the last point N - 1."""
    g = torch.Generator().manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    feature = torch.randn(B, Dh, N, 1, generator=g)
    if pattern == "random":
        idx = torch.randint(0, N, (B, N, 16), generator=g)
    elif pattern == "self":
        idx = torch.arange(N).view(1, N, 1).expand(B, N, 16)
    elif pattern == "same":
        idx = torch.randint(0, N, (B, N, 1), generator=g).expand(B, N, 16)
    else:
        idx = torch.full((B, N, 16), N - 1)
    return xyz.cuda(), feature.cuda(), idx.contiguous().cuda()


def saturate(fc, xyz, idx, feature, m1, m2, slope):
    """fc scaled so that the median gap between a channel's largest and smallest score over the 16 neighbours is
    60: most softmaxes put all their weight on one neighbour, as the ``pm60`` logits of the training test."""
    f_cat = L.encode(xyz, idx, feature, m1, m2, slope)
    att = torch.einsum("oc,bcnk->bonk", fc.double(), f_cat)
    gap = (att.amax(dim=3) - att.amin(dim=3)).median().item()
    return fc * (60.0 / gap) if gap > 0 else fc


def close(got, want, want32, what):
    """test_gpu_lfa.close, each bound widened to 4x torch fp32's error where that is larger."""
    got, want, want32 = got.double(), want.double(), want32.double()
    scale = max(want.abs().max().item(), 1.0)
    d, d32 = (got - want).abs(), (want32 - want).abs()
    assert d.max().item() <= max(1e-5 * scale, 4 * d32.max().item()), "%s: max abs err %.3e, output scale %.3e, torch fp32 %.3e" % (
        what, d.max().item(), scale, d32.max().item())
    big = want.abs() > 0.1 * scale
    if big.any():
        rel, rel32 = (d[big] / want.abs()[big]).max().item(), (d32[big] / want.abs()[big]).max().item()
        assert rel <= max(1e-4, 4 * rel32), "%s: max element-wise relative err %.3e (torch fp32 %.3e)" % (what, rel, rel32)


def run_and_check(xyz, idx, feature, layers, slope, what):
    m1, m2, fc, mo = layers
    got = ops.lfa_att_pool_fused(xyz, idx, feature, m1, m2, fc, mo, negative_slope=slope)
    assert got.shape == (idx.shape[0], mo[0].shape[0], idx.shape[1], 1) and got.dtype == torch.float32
    got32 = ops.lfa_att_pool_fused(xyz, idx.int(), feature, m1, m2, fc, mo, negative_slope=slope)
    assert torch.equal(got, got32), what + ": int32 and int64 indices differ"
    want = L.lfa_att_pool(xyz, idx, feature, m1, m2, fc, mo, slope)
    want32 = L.lfa_att_pool(xyz, idx, feature, m1, m2, fc, mo, slope, dtype=torch.float32)
    close(got, want, want32, what)
    return got


def _do_values(Dh):
    return sorted({v for v in (1, 31, 33, Dh, 2 * Dh) if v <= 2 * Dh})


WIDTHS = [(Dh, mlp2, Do) for Dh in (16, 32, 64) for mlp2 in (False, True) for Do in _do_values(Dh)]


@pytest.mark.parametrize("slope", [0.2, 0.0])
@pytest.mark.parametrize("Dh,mlp2,Do", WIDTHS, ids=["d%d%s_out%d" % (2 * h, "_mlp2" if m else "", o) for h, m, o in WIDTHS])
def test_lfa_fused_widths_and_shapes(cuda, Dh, mlp2, Do, slope):
    """Random neighbours and ordinary attention at every (d/2, mlp2, d_out), one to three frames of 1, 7 and 12288
    points; at d/2 = 16 also 4 frames of 12288 points.  int32 and int64 indices give the same bits."""
    layers = make_layers(Dh, Do, mlp2, seed=Dh + Do)
    for B, N in SHAPES + ([(4, 12288)] if Dh == 16 else []):
        xyz, feature, idx = make_points(B, N, Dh, "random", seed=B * N + Dh)
        run_and_check(xyz, idx, feature, layers, slope, "d/2=%d mlp2=%s Do=%d slope=%g B=%d N=%d" % (Dh, mlp2, Do, slope, B, N))


@pytest.mark.parametrize("attention", ["ordinary", "saturated", "uniform"])
@pytest.mark.parametrize("pattern", ["random", "self", "same", "last"])
@pytest.mark.parametrize("Dh", [16, 32, 64])
def test_lfa_fused_neighbourhoods_and_attention(cuda, Dh, pattern, attention):
    """Degenerate neighbourhoods (distance 0, one repeated point, the row's last point) and attention that is
    ordinary, saturated (score gaps of about 60 between neighbours) or uniform (fc = 0: the mean over K)."""
    m1, m2, fc, mo = make_layers(Dh, 2 * Dh, True, seed=Dh)
    for B, N in ((3, 7), (2, 12288)):
        xyz, feature, idx = make_points(B, N, Dh, pattern, seed=N + Dh)
        fcx = fc
        if attention == "saturated":
            fcx = saturate(fc, xyz, idx, feature, m1, m2, 0.2)
        elif attention == "uniform":
            fcx = torch.zeros_like(fc)
        got = run_and_check(xyz, idx, feature, (m1, m2, fcx, mo), 0.2,
                            "d/2=%d %s neighbours, %s attention, B=%d N=%d" % (Dh, pattern, attention, B, N))
        if attention == "uniform":      # the pooled vector is the mean of the 16 neighbours
            f_cat = L.encode(xyz, idx, feature, m1, m2, 0.2)
            want = L.fusion_layer(f_cat.mean(dim=3, keepdim=True), None, *mo, L.ACT_LEAKY, 0.2)
            assert (got.double() - want).abs().max().item() <= 1e-5 * max(want.abs().max().item(), 1.0)


@pytest.mark.parametrize("Dh", [16, 32, 64])
def test_lfa_fused_nan_feature(cuda, Dh):
    """A NaN at feature[b, c, j]: exactly the points of frame b whose neighbour list holds j are NaN, in every
    output channel; every other output is bitwise the output without the NaN."""
    B, N = 2, 3000
    m1, m2, fc, mo = make_layers(Dh, 2 * Dh, True, seed=7)
    xyz, feature, idx = make_points(B, N, Dh, "random", seed=11)
    b, c, j = 1, Dh - 1, 1234
    idx[b, 5] = j                        # at least one point with j as every neighbour ...
    idx[b, 6, 3] = j                     # ... and one with j once
    bad = feature.clone()
    bad[b, c, j] = float("nan")
    for slope in (0.2, 0.0):
        clean = ops.lfa_att_pool_fused(xyz, idx, feature, m1, m2, fc, mo, negative_slope=slope)
        got = ops.lfa_att_pool_fused(xyz, idx, bad, m1, m2, fc, mo, negative_slope=slope)
        hit = torch.zeros(B, N, dtype=torch.bool, device=cuda)
        hit[b] = (idx[b] == j).any(dim=1)
        nan = torch.isnan(got[..., 0])                  # [B, Do, N]
        assert nan.any(dim=1).eq(hit).all(), "slope=%g: NaN points %s, expected %s" % (
            slope, nan.any(dim=1).nonzero().tolist()[:8], hit.nonzero().tolist()[:8])
        assert nan.all(dim=1).eq(hit).all(), "slope=%g: a point with the NaN neighbour has finite channels" % slope
        keep = ~hit.unsqueeze(1).expand_as(nan)
        assert torch.equal(got[..., 0][keep], clean[..., 0][keep]), "slope=%g: unaffected points changed" % slope
