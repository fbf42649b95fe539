"""GPU: the fused cat + 1x1 conv + BatchNorm(eval) + activation tensor-core kernel against a float64
evaluation of the reference layer (models/pytorch_utils.py:75-129: conv(bias=False) -> BatchNorm2d
-> ReLU, or RandLA's LeakyReLU) and against torch's own fp32 path.  Floating-point kernel: tolerance 1e-5 of
the output scale (BASELINE.json "fused features within 1e-5 fp32").  Also: the epilogue addend, and what a NaN or
an infinity in the input does to the output."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import ffb6d_b200 as F
from ffb6d_b200 import tables
from oracle import lfa_oracle

pytestmark = pytest.mark.gpu

# (act, negative_slope): ReLU (the fusion layers), none (the attention fc), LeakyReLU (RandLA's convs)
ACTS = [(1, 0.0), (0, 0.0), (2, 0.2)]


def _record(name, err_of_scale, rel, rel32):
    """Append the measured errors to gpurun_out/mlp_errors.jsonl (DESIGN.md quotes them)."""
    import json
    import os
    from conftest import ROOT
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", "mlp_errors.jsonl"), "a") as fh:
            fh.write(json.dumps({"layer": name, "max_abs_err_over_scale": err_of_scale, "max_rel_err_above_floor": rel,
                                 "torch_fp32_rel": rel32}) + "\n")
    except OSError:
        pass


def reference_layer(x1, x2, conv, bn, act=1, slope=0.0, dtype=torch.float64):
    x = torch.cat((x1, x2), dim=1) if x2 is not None else x1
    y = nn.functional.conv2d(x.to(dtype), conv.weight.to(dtype))
    y = nn.functional.batch_norm(y, bn.running_mean.to(dtype), bn.running_var.to(dtype), bn.weight.to(dtype),
                                 bn.bias.to(dtype), training=False, eps=bn.eps)
    return lfa_oracle.activation(y, act, slope)


def run_layer(x1, x2, weight, scale, shift, act, slope, **kw):
    return F.fusion_mlp(x1, x2, weight, scale, shift, relu=act == 1, negative_slope=slope if act == 2 else None, **kw)


def make_layer(cin, cout, seed, nonneg=False):
    g = torch.Generator().manual_seed(seed)
    conv = nn.Conv2d(cin, cout, (1, 1), bias=False)
    bn = nn.BatchNorm2d(cout)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / cin ** 0.5)
        if nonneg:
            conv.weight.abs_()
        bn.weight.copy_(torch.rand(cout, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(cout, generator=g) * 0.1)
        bn.running_mean.copy_(torch.randn(cout, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(cout, generator=g) + 0.3)
    return conv.cuda().eval(), bn.cuda().eval()


def make_inputs(B, C1, C2, tail, seed, post_relu=False):
    """N(0,1), or relu(N(0,1) + 0.3): the non-negative post-activation features real fusion layers see."""
    g = torch.Generator().manual_seed(seed)

    def one(C):
        x = torch.randn((B, C) + tail, generator=g)
        return (torch.relu(x + 0.3) if post_relu else x).cuda()
    return one(C1), (one(C2) if C2 else None)


def check_layer(x1, x2, conv, bn, what):
    """Every activation: within 1e-5 of the output scale of float64, no worse than 8x torch's fp32 path (TF32 off),
    and element-wise within max(1e-5, 4x torch fp32) relative above a floor of 10 % of the scale."""
    scale, shift = F.fold_batchnorm(bn)
    for act, slope in ACTS:
        got = run_layer(x1, x2, conv.weight, scale, shift, act, slope)
        want = reference_layer(x1, x2, conv, bn, act, slope)
        assert got.shape == want.shape and got.dtype == torch.float32
        ref_scale = want.abs().max().item()
        err = (got.double() - want).abs().max().item()
        assert err <= 1e-5 * max(ref_scale, 1.0), "%s act=%d: max abs err %.3e (output scale %.3e)" % (
            what, act, err, ref_scale)
        # no worse than torch's own fp32 path (TF32 disabled) by more than a small factor
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            fp32 = reference_layer(x1, x2, conv, bn, act, slope, dtype=torch.float32)
        finally:
            torch.backends.cudnn.allow_tf32 = prev
        err32 = (fp32.double() - want).abs().max().item()
        assert err <= max(8 * err32, 2e-6 * max(ref_scale, 1.0)), (what, act, err, err32)
        # element-wise relative error above an absolute floor of 10 % of the output scale (outputs near zero
        # are sums of K cancelling fp32 products: their error scales with the terms, not with the result);
        # 1e-5, or what torch's own fp32 path shows on the same elements if that is larger
        big = want.abs() > 0.1 * max(ref_scale, 1.0)
        if big.any():
            rel = ((got.double() - want).abs()[big] / want.abs()[big]).max().item()
            rel32 = ((fp32.double() - want).abs()[big] / want.abs()[big]).max().item()
            if act == 1:
                _record(what, err / max(ref_scale, 1.0), rel, rel32)
            assert rel <= max(1e-5, 4 * rel32), "%s act=%d: element-wise relative err %.3e (torch fp32: %.3e)" % (
                what, act, rel, rel32)


# (B, C1, C2, Co, trailing shape): fusion layers of models/ffb6d.py (SURVEY.md App. A.3) + ragged shapes
CASES = [
    (2, 64, 64, 64, (3072, 1)),        # ds0 r2p_fuse
    (2, 64, 64, 64, (120, 160)),       # ds0 p2r_fuse on the image map
    (1, 512, 512, 256, (192, 1)),      # ds2 r2p_fuse
    (1, 1024, 1024, 1024, (60, 80)),   # ds3 p2r_fuse (20 GFLOP / frame)
    (2, 256, 0, 256, (192, 1)),        # *_pre layers: no concat
    (1, 36, 8, 70, (50, 1)),           # ragged: Ci % 32 != 0, Co % 128 != 0, P % 128 != 0
    (1, 5, 0, 3, (7, 1)),              # nothing aligned (scalar path)
    (1, 6, 10, 64, (256, 1)),          # vector loads with the concat boundary inside a 4-row K chunk
    (2, 36, 8, 64, (3072, 1)),         # fast path (P % 128 == 0, C1 % 4 == 0) with a ragged last k-tile
    (2, 130, 2, 200, (1000, 1)),       # a partial second 128-row M tile
    (1, 64, 0, 129, (129, 1)),         # a one-row second M tile and a one-column last N tile
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_%d+%d->%d_%s" % (c[0], c[1], c[2], c[3], "x".join(map(str, c[4]))))
def test_fusion_mlp_matches_reference_layer(cuda, case):
    B, C1, C2, Co, tail = case
    x1, x2 = make_inputs(B, C1, C2, tail, seed=C1 + Co)
    conv, bn = make_layer(C1 + C2, Co, seed=Co)
    check_layer(x1, x2, conv, bn, "%d+%d->%d x%d" % (C1, C2, Co, int(np.prod(tail))))


SCHEDULE = sorted({(P, C1, C2, Co) for _, P, C1, C2, Co in tables.fusion_mlp_schedule()})


@pytest.mark.parametrize("P,C1,C2,Co", SCHEDULE, ids=["P%d_%d+%d->%d" % s for s in SCHEDULE])
def test_fusion_mlp_schedule_post_relu(cuda, P, C1, C2, Co):
    """Every layer shape FFB6D runs (480x640 frames, 12288 points), on the non-negative inputs a fusion layer gets
    from the ReLU before it: same-sign products are where a biased accumulation would show.  The layers with 1024
    or more input channels (ds3's, and ds2's p2r_fuse) also run with all-non-negative weights, so that no product
    cancels another."""
    x1, x2 = make_inputs(1, C1, C2, (P, 1), seed=P + C1 + Co, post_relu=True)
    for nonneg in (False, True) if C1 + C2 >= 1024 else (False,):
        conv, bn = make_layer(C1 + C2, Co, seed=Co + 1, nonneg=nonneg)
        check_layer(x1, x2, conv, bn, "%d+%d->%d x%d post-relu%s" % (C1, C2, Co, P, " w>=0" if nonneg else ""))


@pytest.mark.parametrize("which", ["x1", "x2"])
def test_fusion_mlp_misaligned_input(cuda, which):
    """An input that starts 4 bytes past a 16-byte boundary (a view at storage offset 1) with P % 4 == 0: the
    element-wise load path, at a real layer size."""
    B, C1, C2, Co, P = 1, 64, 64, 64, 3072
    x1, x2 = make_inputs(B, C1, C2, (P, 1), seed=5, post_relu=True)
    src = x1 if which == "x1" else x2
    view = torch.empty(src.numel() + 1, device=cuda)[1:].view(src.shape).copy_(src)
    assert view.data_ptr() % 16 == 4 and view.is_contiguous()
    x1, x2 = (view, x2) if which == "x1" else (x1, view)
    conv, bn = make_layer(C1 + C2, Co, seed=9)
    check_layer(x1, x2, conv, bn, "%d+%d->%d x%d %s misaligned" % (C1, C2, Co, P, which))


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["int32", "int64"])
@pytest.mark.parametrize("act,slope", ACTS, ids=["relu", "none", "leaky"])
def test_fusion_mlp_epilogue_addend(cuda, act, slope, idx_dtype):
    """``act(scale * (W x + add[b, add_idx[b, p], :]) + shift)`` at Co = 200 (a partial second M tile) against float64,
    with indices that include the addend's last row, in both output layouts (bitwise the same values)."""
    B, C1, Co, P, NA = 2, 64, 200, 1000, 300
    g = torch.Generator().manual_seed(17)
    x1 = torch.randn(B, C1, P, generator=g).cuda()
    add = torch.randn(B, NA, Co, generator=g).cuda()
    idx = torch.randint(0, NA, (B, P), generator=g)
    idx[:, ::97] = NA - 1
    idx[1, -1] = NA - 1
    idx = idx.to(idx_dtype).cuda()
    conv, bn = make_layer(C1, Co, seed=21)
    scale, shift = F.fold_batchnorm(bn)
    want = lfa_oracle.fusion_layer(x1, None, conv.weight, scale, shift, act, slope, add=add, add_idx=idx)
    ref_scale = max(want.abs().max().item(), 1.0)
    ncs = run_layer(x1, None, conv.weight, scale, shift, act, slope, add=add, add_idx=idx)
    nsc = run_layer(x1, None, conv.weight, scale, shift, act, slope, add=add, add_idx=idx, out_channels_last=True)
    assert ncs.shape == (B, Co, P) and nsc.shape == (B, P, Co)
    err = (ncs.double() - want).abs().max().item()
    assert err <= 1e-5 * ref_scale, "addend act=%d: max abs err %.3e (output scale %.3e)" % (act, err, ref_scale)
    assert torch.equal(nsc.permute(0, 2, 1), ncs)


NONFINITE_CASES = [(2, 64, 64, 64, (3072, 1)), (1, 36, 8, 200, (50, 1)), (1, 5, 0, 3, (7, 1))]


# bit patterns of the non-finite inputs: torch's NaN, the NaN the GPU's arithmetic produces (inf - inf, 0 / 0), its
# negative twin, and the two infinities
NONFINITE = {"nan": 0x7FC00000, "nan_7fffffff": 0x7FFFFFFF, "nan_ffffffff": -1, "inf": 0x7F800000, "-inf": -0x800000}


@pytest.mark.parametrize("bad", list(NONFINITE))
@pytest.mark.parametrize("case", NONFINITE_CASES, ids=["fast", "ragged", "scalar"])
def test_fusion_mlp_nonfinite_input(cuda, case, bad):
    """One NaN or infinity at x1[b, c, p]: every output channel at (b, p) is NaN for every activation --
    torch.relu(NaN) is NaN, a poisoned position must not come out as 0, and an infinity comes out NaN through the
    3xTF32 lo products (inf - inf) -- and every other position is bitwise the output without it."""
    B, C1, C2, Co, tail = case
    x1, x2 = make_inputs(B, C1, C2, tail, seed=3)
    conv, bn = make_layer(C1 + C2, Co, seed=4)
    scale, shift = F.fold_batchnorm(bn)
    P = int(np.prod(tail))
    b, c, p = B - 1, C1 // 2, P - 3
    xb = x1.clone().view(B, C1, P)
    xb.view(torch.int32)[b, c, p] = NONFINITE[bad]
    assert not torch.isfinite(xb[b, c, p])
    xb = xb.view(x1.shape)
    for act, slope in ACTS:
        clean = run_layer(x1, x2, conv.weight, scale, shift, act, slope).view(B, Co, P)
        got = run_layer(xb, x2, conv.weight, scale, shift, act, slope).view(B, Co, P)
        hit = got[b, :, p]
        assert torch.isnan(hit).all(), "act=%d: %d of %d channels at the %s position are not NaN: %s" % (
            act, int((~torch.isnan(hit)).sum()), Co, bad, hit[~torch.isnan(hit)][:8].tolist())
        got[b, :, p] = clean[b, :, p]
        assert torch.equal(got, clean), "act=%d: positions other than the non-finite input changed" % act


@pytest.mark.parametrize("case", [CASES[0], CASES[3], CASES[5]], ids=["ds0", "ds3", "ragged"])
def test_fusion_mlp_packed_weights_bit_identical(cuda, case):
    """Weights split once (ffb6d_fusion_mlp_pack) give the same bits as the per-call split, and the
    pack survives many calls."""
    B, C1, C2, Co, tail = case
    g = torch.Generator().manual_seed(7)
    x1 = torch.randn((B, C1) + tail, generator=g).cuda()
    x2 = torch.randn((B, C2) + tail, generator=g).cuda() if C2 else None
    conv, bn = make_layer(C1 + C2, Co, seed=3)
    scale, shift = F.fold_batchnorm(bn)
    packed = F.fusion_mlp_pack(conv.weight)
    assert packed.Co == Co and packed.Ci == C1 + C2
    want = F.fusion_mlp(x1, x2, conv.weight, scale, shift)
    for _ in range(3):
        got = F.fusion_mlp(x1, x2, packed, scale, shift)
        assert torch.equal(got, want)
    with pytest.raises(ValueError):
        F.fusion_mlp(x1[:, :-1], x2, packed, scale, shift)
