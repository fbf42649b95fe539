"""GPU: the 3xTF32 tensor-core GEMMs of ``fusion_mlp.cu`` across the float32 range.

Every operand of these GEMMs is split into ``hi = tf32(x)`` and ``lo = tf32(x - hi)``, and the products
``Ahi*Bhi + Alo*Bhi + Ahi*Blo`` are accumulated on the tensor core (DESIGN.md §4.4).  The rest of the suite feeds them
values of a few binades around 1.  Here:

* the split the pack kernel writes equals its numpy restatement (``oracle/tf32_oracle.py``) bit for bit, over every
  exponent with the mantissas at the rounding edges;
* scaling x by 2^a and W by 2^b is exact, so the outputs must be bitwise 2^(a+b) times the unscaled ones wherever
  nothing leaves the normal range (the comment above ``PAIRS`` derives that range); on every forward path, the PSP
  bottleneck, ``final``'s log-softmax (against float64) and both weight gradients;
* outside that range, against float64 with a condition-aware bound: finite operands up to FLT_MAX, subnormal
  operands and products, one dot product spanning 2^-40 .. 2^40, and zero-sum weight rows on offset features.
"""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200._lib import lib, check
from ffb6d_b200.ops import _stream
from oracle import tf32_oracle as T

pytestmark = pytest.mark.gpu

# ----------------------------------------------------------------------------------------- the split, bit for bit
EDGE_MANTISSAS = [0x000000, 0x000001, 0x000FFF, 0x001000, 0x001001, 0x001FFF, 0x002000, 0x003000, 0x7FEFFF, 0x7FF000,
                  0x7FE000, 0x7FFFFF, 0x400000, 0x555555]


def _edge_patterns():
    """Both signs x all 256 exponents x the rounding-edge mantissas (infinities and NaNs among them)."""
    sign = np.array([0, 1], np.uint32)[:, None, None] << np.uint32(31)
    expo = np.arange(256, dtype=np.uint32)[None, :, None] << np.uint32(23)
    mant = np.asarray(EDGE_MANTISSAS, np.uint32)[None, None, :]
    return (sign | expo | mant).ravel()


def _unpack(pk):
    """hi and lo planes [ceil(Co/128)*128, ceil(Ci/32)*32] (uint32 bits) from the blocks of ``ffb6d_fusion_mlp_pack``:
    one 32 KB block per (128-row tile, 32-column k-tile), [hi | lo], each 8 chunks (k = 4c .. 4c+3) x 128 rows x
    16 bytes (fusion_mlp_pack_kernel)."""
    nmt, nk = -(-pk.Co // 128), -(-pk.Ci // 32)
    a = pk.data.view(torch.int32).cpu().numpy().view(np.uint32).reshape(nmt, nk, 2, 8, 128, 4)
    a = a.transpose(2, 0, 4, 1, 3, 5).reshape(2, nmt * 128, nk * 32)   # [plane, row, k]
    return a[0], a[1]


@pytest.mark.parametrize("Co,Ci", [(130, 56), (7, 1030)], ids=["two_m_tiles", "one_row_tile"])
def test_pack_split_matches_restatement(cuda, Co, Ci):
    """``ffb6d_fusion_mlp_pack`` on weights made of every exponent with the rounding-edge mantissas (and finite
    fillers): for every finite weight, hi and lo bitwise equal to the restatement; for a NaN or an infinity, hi NaN;
    the padding of the last tiles +0."""
    u = _edge_patterns()
    rs = np.random.RandomState(Co + Ci)
    w = rs.randn(Co * Ci).astype(np.float32)
    assert u.size <= w.size
    w[rs.permutation(w.size)[:u.size]] = u.view(np.float32)
    w = w.reshape(Co, Ci)
    hi, lo = _unpack(F.fusion_mlp_pack(torch.from_numpy(w).cuda()))
    want_hi, want_lo = T.split(w)
    fin = np.isfinite(w)
    got_hi, got_lo = hi[:Co, :Ci], lo[:Co, :Ci]
    for name, got, want in (("hi", got_hi, want_hi), ("lo", got_lo, want_lo)):
        bad = fin & (got != want.view(np.uint32))
        assert not bad.any(), "%s differs at %d finite weights, e.g. %s: got %s, want %s" % (
            name, int(bad.sum()), hex(int(w.view(np.uint32)[bad][0])), hex(int(got[bad][0])),
            hex(int(want.view(np.uint32)[bad][0])))
    assert np.isnan(got_hi[~fin].view(np.float32)).all()
    assert fin.sum() < w.size and np.isfinite(got_hi[fin].view(np.float32)).all()
    pad = np.ones(hi.shape, bool)
    pad[:Co, :Ci] = False
    assert not hi[pad].any() and not lo[pad].any()


# --------------------------------------------------------------------------------- exact power-of-two invariance
# Operands are drawn with magnitudes in [2^-3, 2^3] (_operand).  Scaled by 2^a (x) and 2^b (W), the kernels' outputs
# are bitwise 2^(a+b) times the unscaled ones as long as every value they round stays normal and finite:
#   * operands: 2^(3+a) is below the top band (0x7F7FF000), so hi is rounded, not truncated: a, b <= 124;
#   * lo parts: a nonzero lo is a multiple of ulp(x) >= 2^(-26+a), normal for a, b >= -100;
#   * products and partial sums: multiples of ulp(lo) * ulp(hi) >= 2^(-26+a) * 2^(-13+b) = 2^(a+b-39), so every
#     nonzero one is normal for a + b >= -87; the largest is below sum_k |W_k||x_k| (1 + 2^-10)^2 * 1.5 (the
#     folded BatchNorm scale) < 2^20 * 2^(a+b) for K <= 10 000, finite for a + b <= 107.
# The sweep takes a, b in -100 .. 100 in steps of 20 with -80 <= a + b <= 100.
EXPS = range(-100, 101, 20)
PAIRS = [(a, b) for a in EXPS for b in EXPS if -80 <= a + b <= 100]


def _operand(g, shape, positive=False):
    e = torch.rand(shape, generator=g, dtype=torch.float64) * 6 - 3
    v = torch.exp2(e)
    if not positive:
        v = torch.where(torch.rand(shape, generator=g) < 0.5, -v, v)
    return v.float()


def _scaled(t, s):
    """``t * s``, 4 bytes past a 16-byte boundary where ``t`` is."""
    out = t * s
    if t.data_ptr() % 16:
        out = torch.empty(out.numel() + 1, device=t.device)[1:].view(out.shape).copy_(out)
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same_bits(got, want, what):
    if not torch.equal(_bits(got), _bits(want)):
        d = _bits(got) != _bits(want)
        i = int(d.flatten().nonzero()[0])
        raise AssertionError("%s: %d of %d outputs not bitwise 2^(a+b) times the unscaled ones, e.g. %r vs %r" % (
            what, int(d.sum()), d.numel(), got.flatten()[i].item(), want.flatten()[i].item()))


FWD_PATHS = {
    "scalar": (1, 5, 0, 3, (7, 1)),                 # nothing aligned: element-wise loads and stores
    "concat_in_chunk": (1, 6, 10, 64, (256, 1)),    # vector loads, the concat boundary inside a 4-row K chunk
    "fast_ragged_k": (2, 36, 8, 64, (3072, 1)),     # whole-tile fast path with a ragged last k-tile
    "ragged": (1, 36, 8, 70, (50, 1)),              # Ci % 32, Co % 128 and P % 128 all nonzero
    "two_m_tiles": (2, 130, 2, 200, (1000, 1)),     # a partial second 128-row tile
    "ds3": (1, 1024, 1024, 1024, (60, 80)),         # ds3 p2r_fuse: the largest K
}


@pytest.mark.parametrize("path", list(FWD_PATHS) + ["misaligned"])
def test_fusion_mlp_power_of_two_scaling_is_exact(cuda, path):
    """``fusion_mlp`` (shift 0, activation none and ReLU) on 2^a x and 2^b W is bitwise 2^(a+b) times its output on
    x and W, for every (a, b) of the sweep."""
    B, C1, C2, Co, tail = FWD_PATHS.get(path, FWD_PATHS["ragged"])
    g = torch.Generator().manual_seed(Co + C1)
    x1 = _operand(g, (B, C1) + tail).cuda()
    x2 = _operand(g, (B, C2) + tail).cuda() if C2 else None
    if path == "misaligned":     # x1 4 bytes past a 16-byte boundary: the element-wise load path at P % 4 == 0
        x1 = _operand(g, (1, 64, 3072, 1)).cuda()
        x2, Co = None, 64
        x1 = torch.empty(x1.numel() + 1, device=cuda)[1:].view(x1.shape).copy_(x1)
        assert x1.data_ptr() % 16 == 4
    w = _operand(g, (Co, x1.shape[1] + (x2.shape[1] if x2 is not None else 0))).cuda()
    scale = (torch.rand(Co, generator=g) + 0.5).cuda()
    zero = torch.zeros(Co, device=cuda)
    for relu in (False, True):
        base = F.fusion_mlp(x1, x2, w, scale, zero, relu=relu)
        assert torch.isfinite(base).all() and (base != 0).any()
        for b in EXPS:
            pk = F.fusion_mlp_pack(w * 2.0 ** b)
            for a in EXPS:
                if (a, b) not in PAIRS:
                    continue
                xs1 = _scaled(x1, 2.0 ** a)
                xs2 = _scaled(x2, 2.0 ** a) if x2 is not None else None
                got = F.fusion_mlp(xs1, xs2, pk, scale, zero, relu=relu)
                _same_bits(got, base * 2.0 ** (a + b), "%s relu=%d a=%d b=%d" % (path, relu, a, b))


@pytest.mark.parametrize("B,C,Co,H,W", [(2, 40, 70, 7, 9), (1, 64, 128, 30, 40)], ids=["ragged", "map"])
def test_psp_bottleneck_power_of_two_scaling_is_exact(cuda, B, C, Co, H, W):
    """``psp_bottleneck`` (the prior tables through ``ffb6d_fusion_mlp_fwd_ex``, the feature GEMM, the bilinear taps,
    the bias and the ReLU in ``ffb6d_psp_bottleneck_fwd``) on 2^a x, 2^b W and 2^(a+b) bias.  The stage convs are
    the identity, so the folded tables M_s = W_s; operands are positive, so no sum cancels below the normal range."""
    g = torch.Generator().manual_seed(C + H)
    x = _operand(g, (B, C, H, W), positive=True).cuda()
    wt = _operand(g, (Co, 5 * C, 1, 1), positive=True).cuda()
    bias = _operand(g, (Co,), positive=True).cuda()
    eye = [torch.eye(C, device=cuda).view(C, C, 1, 1)] * 4

    def run(x, wt, bias):
        return F.psp_bottleneck(x, F.psp_pool(x), F.psp_pack(eye, wt, bias))

    base = run(x, wt, bias)
    assert torch.isfinite(base).all() and (base > 0).all()
    for a, b in PAIRS:
        got = run(x * 2.0 ** a, wt * 2.0 ** b, bias * 2.0 ** (a + b))
        _same_bits(got, base * 2.0 ** (a + b), "psp_bottleneck a=%d b=%d" % (a, b))


@pytest.mark.parametrize("B,Ci,Co,H,W", [(2, 64, 22, 7, 33), (1, 40, 128, 5, 26)], ids=["ycb_classes", "co128"])
def test_conv1x1_log_softmax_scaled_logits_vs_float64(cuda, B, Ci, Co, H, W):
    """``conv1x1_log_softmax`` on 2^a x, 2^b W and 2^(a+b) bias: within 2^-22 relative + 1e-5 of the float64
    log-softmax of the kernel's own logits (``fusion_mlp`` on the same packed weights: bitwise 2^(a+b) times the
    unscaled ones, which this test checks too), and within the condition-aware bound of the float64 log-softmax of
    the exact logits.  A log-softmax moves by at most twice the largest logit error."""
    g = torch.Generator().manual_seed(Ci + Co)
    x = _operand(g, (B, Ci, H, W)).cuda()
    w = _operand(g, (Co, Ci)).cuda()
    bias = _operand(g, (Co,)).cuda()
    one = torch.ones(Co, device=cuda)
    base = F.fusion_mlp(x, None, w, one, bias, relu=False)
    for a, b in PAIRS:
        xs, pk, bs = x * 2.0 ** a, F.fusion_mlp_pack(w * 2.0 ** b), bias * 2.0 ** (a + b)
        logits = F.fusion_mlp(xs, None, pk, one, bs, relu=False)
        _same_bits(logits, base * 2.0 ** (a + b), "final logits a=%d b=%d" % (a, b))
        got = F.conv1x1_log_softmax(xs, pk, bs).double()
        what = "conv1x1_log_softmax a=%d b=%d" % (a, b)
        own = torch.log_softmax(logits.double(), dim=1)
        err = (got - own).abs()
        assert (err <= 2.0 ** -22 * own.abs() + 1e-5).all(), "%s: %.3e from the float64 log-softmax of its logits" % (
            what, err.max().item())
        exact = torch.einsum("oc,bchw->bohw", w.double() * 2.0 ** b, xs.double()) + bs.double().view(1, -1, 1, 1)
        cond = (torch.einsum("oc,bchw->bohw", w.double().abs() * 2.0 ** b, xs.double().abs())
                + bs.double().abs().view(1, -1, 1, 1))
        want = torch.log_softmax(exact, dim=1)
        bound = 2 * 8 * 2.0 ** -21 * cond.amax(dim=1, keepdim=True) + 2.0 ** -22 * want.abs() + 1e-5
        bad = (got - want).abs() > bound
        assert not bad.any(), "%s: %d outputs over the condition-aware bound" % (what, int(bad.sum()))


def _wgrad(dz, x1, x2, det):
    B, Co, P = dz.shape
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    gw = torch.full((Co, C1 + C2), float("nan"), device=dz.device)
    x2p = x2.data_ptr() if x2 is not None else None
    if det:
        nbytes = int(lib.ffb6d_fusion_mlp_wgrad_det_workspace_bytes(C1, C2, B, Co, P))
        ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dz.device)
        check(lib.ffb6d_fusion_mlp_wgrad_det(dz.data_ptr(), x1.data_ptr(), C1, x2p, C2, B, Co, P, ws.data_ptr(), nbytes,
                                             gw.data_ptr(), _stream(dz.device)))
    else:
        check(lib.ffb6d_fusion_mlp_wgrad(dz.data_ptr(), x1.data_ptr(), C1, x2p, C2, B, Co, P, gw.data_ptr(),
                                         _stream(dz.device)))
    return gw


# (B, C1, C2, Co, P, det).  The atomic kernel is only deterministic where every weight gets one partial: B * P of at
# most 8 k-tiles of 32 points is one split.  The deterministic kernel adds its splits in a fixed order in fp64.
WGRAD_PATHS = {"atomic_one_split": (1, 100, 40, 200, 256, False), "det_ragged": (2, 131, 125, 200, 4097, True),
               "det_ds3": (1, 1024, 1024, 1024, 600, True)}


@pytest.mark.parametrize("path", list(WGRAD_PATHS))
def test_wgrad_power_of_two_scaling_is_exact(cuda, path):
    """``ffb6d_fusion_mlp_wgrad`` / ``_det`` on 2^a dz and 2^b x: bitwise 2^(a+b) times the unscaled weight gradient."""
    B, C1, C2, Co, P, det = WGRAD_PATHS[path]
    g = torch.Generator().manual_seed(P)
    dz = _operand(g, (B, Co, P)).cuda()
    x1 = _operand(g, (B, C1, P)).cuda()
    x2 = _operand(g, (B, C2, P)).cuda() if C2 else None
    base = _wgrad(dz, x1, x2, det)
    assert torch.isfinite(base).all()
    assert torch.equal(_bits(_wgrad(dz, x1, x2, det)), _bits(base)), "not bitwise repeatable"
    for a, b in PAIRS:
        got = _wgrad(dz * 2.0 ** a, x1 * 2.0 ** b, x2 * 2.0 ** b if x2 is not None else None, det)
        _same_bits(got, base * 2.0 ** (a + b), "wgrad %s a=%d b=%d" % (path, a, b))


# ------------------------------------------------------------------------- outside the invariant range: float64
SUB = 2.0 ** -136     # the spacing of TF32's subnormals: hi and lo of any x are multiples of it


def _check_vs_float64(got, W, X, what, c=8):
    """``got [B, Co, P]`` = W [Co, K] . X [B, K, P] (act none, scale 1, shift 0) against float64, element-wise:
    ``|got - want| <= c 2^-21 sum_k |W_k||x_k| + 2^-136 sum_k (|W_k| + |x_k|) + K 2^-149`` (the split's 2^-22
    relative error on each operand, the dropped lo*lo, the accumulation; each operand's split loses at most 2^-137
    below the normal range, and each of the fewer than K additions at most 2^-149 where its sum is subnormal).  And
    no worse than 8x torch's fp32 product (TF32 off), or 2e-6 of the output scale, where larger."""
    W64, X64 = W.double(), X.double()
    want = torch.matmul(W64, X64)
    cond = torch.matmul(W64.abs(), X64.abs())
    floor = SUB * (W64.abs().sum(1).view(1, -1, 1) + X64.abs().sum(1, keepdim=True)) + W.shape[1] * 2.0 ** -149
    assert torch.isfinite(want).all(), "%s: the test's own product is not finite" % what
    assert torch.isfinite(got).all(), "%s: %d non-finite outputs" % (what, int((~torch.isfinite(got)).sum()))
    err = (got.double() - want).abs()
    bad = err > c * 2.0 ** -21 * cond + floor
    if bad.any():
        i = int((err - c * 2.0 ** -21 * cond - floor).flatten().argmax())
        raise AssertionError("%s: %d outputs over the bound; worst err %.3e, want %.3e, sum |W||x| %.3e" % (
            what, int(bad.sum()), err.flatten()[i].item(), want.flatten()[i].item(), cond.flatten()[i].item()))
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref32 = torch.matmul(W.float(), X.float())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    e32 = (ref32.double() - want).abs().max().item()
    scale = want.abs().max().item()
    e = err.max().item()
    assert e <= max(8 * e32, 2e-6 * scale, floor.max().item()), "%s: max err %.3e, torch fp32 %.3e, scale %.3e" % (
        what, e, e32, scale)
    return e, e32


def _layer(x1, x2, W):
    Co = W.shape[0]
    one, zero = torch.ones(Co, device=W.device), torch.zeros(Co, device=W.device)
    return F.fusion_mlp(x1, x2, W, one, zero, relu=False)


def _cat(x1, x2):
    return torch.cat((x1, x2), 1) if x2 is not None else x1


BAND = [0x7F7FF000, 0x7F7FF001, 0x7F7FF7FF, 0x7F7FF800, 0x7F7FFFFE, 0x7F7FFFFF]
RANGE_PATHS = {"scalar": (1, 5, 0, 3, 7), "ragged": (1, 36, 8, 70, 50), "fast": (2, 64, 64, 64, 3072)}


def _band_values(rs, n):
    u = np.array([BAND[i % len(BAND)] | (0x80000000 if rs.rand() < 0.5 else 0) for i in range(n)], np.uint32)
    return torch.from_numpy(u.view(np.float32))


@pytest.mark.parametrize("path", list(RANGE_PATHS))
@pytest.mark.parametrize("where", ["x", "W"])
def test_fusion_mlp_finite_operands_near_flt_max(cuda, path, where):
    """Single operands in the top band (0x7F7FF000 .. 0x7F7FFFFF, both signs), on both sides of the concat, with
    partners of 2^-12 so that every output is finite: finite outputs within the bound.  Round-to-nearest carried
    these operands into +-inf and the split made them NaN, with every output they entered."""
    B, C1, C2, Co, P = RANGE_PATHS[path]
    g = torch.Generator().manual_seed(P + Co)
    rs = np.random.RandomState(P)
    x = torch.randn(B, C1 + C2, P, generator=g)
    W = torch.randn(Co, C1 + C2, generator=g)
    if where == "x":
        W *= 2.0 ** -12
        n = min(P, 6 * (C1 + C2))
        b, c, p = rs.randint(0, B, n), rs.randint(0, C1 + C2, n), rs.permutation(P)[:n]   # at most one per column
        x[b, c, p] = _band_values(rs, n)
    else:
        x *= 2.0 ** -12
        n = min(Co, 12)
        W[np.arange(n), rs.randint(0, C1 + C2, n)] = _band_values(rs, n)
    x, W = x.cuda(), W.cuda()
    x1, x2 = x[:, :C1].contiguous(), (x[:, C1:].contiguous() if C2 else None)
    got = _layer(x1, x2, W)
    _check_vs_float64(got, W, x, "%s band in %s" % (path, where))


@pytest.mark.parametrize("where", ["dz", "x"])
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
def test_wgrad_finite_operands_near_flt_max(cuda, where, det):
    """The weight gradient with single top-band elements in dz or in x (partners of 2^-12): finite, within the
    bound of the forward (the gradient is the product dz [Co, B*P] . x^T)."""
    B, C1, C2, Co, P = 2, 100, 40, 200, 1000
    g = torch.Generator().manual_seed(7)
    rs = np.random.RandomState(8)
    dz, x = torch.randn(B, Co, P, generator=g), torch.randn(B, C1 + C2, P, generator=g)
    big, small = (dz, x) if where == "dz" else (x, dz)
    small *= 2.0 ** -12
    n = 12
    rows = rs.permutation(big.shape[1])[:n]          # one per row, so each weight sums at most one band product
    big[rs.randint(0, B, n), rows, rs.randint(0, P, n)] = _band_values(rs, n)
    dz, x = dz.cuda(), x.cuda()
    gw = _wgrad(dz, x[:, :C1].contiguous(), x[:, C1:].contiguous(), det)
    A = dz.permute(1, 0, 2).reshape(Co, B * P)
    X = x.permute(1, 0, 2).reshape(1, C1 + C2, B * P).transpose(1, 2)
    _check_vs_float64(gw[None], A, X, "wgrad%s band in %s" % (" det" * det, where))


@pytest.mark.parametrize("case", ["subnormal_x", "subnormal_W", "subnormal_products", "tiny_lo"])
def test_fusion_mlp_subnormal_range(cuda, case):
    """Operands and products below the normal range, against float64 within the bound with its subnormal floor:
    subnormal x (2^-149 .. 2^-127) with unit W; subnormal W with unit x; normal operands of 2^-80 .. 2^-60 whose
    products are subnormal; normal x of 2^-126 .. 2^-100 whose lo parts are subnormal."""
    B, C1, C2, Co, P = 1, 36, 8, 70, 50
    g = torch.Generator().manual_seed(11)
    mant = lambda *s: torch.where(torch.rand(s, generator=g) < 0.5, -1.0, 1.0) * (1 + torch.rand(s, generator=g))
    expo = lambda lo, hi, *s: torch.exp2(torch.randint(lo, hi + 1, s, generator=g).double())
    x = mant(B, C1 + C2, P).double() * expo(-2, 2, B, C1 + C2, P)
    W = mant(Co, C1 + C2).double() * expo(-2, 2, Co, C1 + C2)
    if case == "subnormal_x":
        x = mant(B, C1 + C2, P).double() * expo(-149, -128, B, C1 + C2, P)
    elif case == "subnormal_W":
        W = mant(Co, C1 + C2).double() * expo(-149, -128, Co, C1 + C2)
    elif case == "subnormal_products":
        x *= expo(-80, -60, B, C1 + C2, P)
        W *= expo(-80, -60, Co, C1 + C2)
    else:
        x *= expo(-126, -100, B, C1 + C2, P)
    x, W = x.float().cuda(), W.float().cuda()
    got = _layer(x[:, :C1].contiguous(), x[:, C1:].contiguous(), W)
    _check_vs_float64(got, W, x, case)


def test_subnormal_operands_and_products_are_not_flushed(cuda):
    """The tensor core keeps subnormal tf32 operands and subnormal products: one product per output, each operand a
    TF32 value (so its split is exact), gives the exact product, down to 2^-149.  What the layers lose below the
    normal range is the split's: hi and lo are multiples of 2^-136 (``tests/test_tf32_split.py``)."""
    xs = [2.0 ** -130, 1.5 * 2.0 ** -127, 2.0 ** -136, -(2.0 ** -128), 1.0, 2.0 ** -70, 2.0 ** -79, 2.0 ** 100]
    ws = [1.0, 2.0 ** -60, 2.0 ** -13, 2.0 ** -70, 2.0 ** -130, -(2.0 ** -149) * 2 ** 13]
    x = torch.zeros(1, 8, len(xs))
    x[0, 0] = torch.tensor(xs)
    W = torch.zeros(len(ws), 8)
    W[:, 0] = torch.tensor(ws)
    want = (W[:, :1].double() * x[0, :1].double())              # [Co, P]: every product of the two lists
    keep = (want.abs() >= 2.0 ** -149) & (want.abs() < 2.0 ** 127)
    got = _layer(x.cuda(), None, W.cuda())[0].cpu().double()
    assert keep.sum() > 20 and ((want.abs() < 2.0 ** -126) & keep).sum() > 8
    assert torch.equal(got[keep], want[keep]), (got[keep] - want[keep]).abs().max().item()


def test_fusion_mlp_dot_product_spanning_2e80(cuda):
    """One input column per position spanning 2^-40 .. 2^40 over its channels (every binade between), under
    random-sign weights: within the condition-aware bound, and no worse than 8x torch fp32."""
    B, C1, C2, Co, P = 2, 64, 17, 70, 300
    g = torch.Generator().manual_seed(5)
    e = torch.linspace(-40, 40, C1 + C2, dtype=torch.float64)[torch.randperm(C1 + C2, generator=g)]
    x = (torch.exp2(e).view(1, -1, 1) * (1 + torch.rand(B, C1 + C2, P, generator=g, dtype=torch.float64))).float()
    x = torch.where(torch.rand(x.shape, generator=g) < 0.5, -x, x)
    W = torch.randn(Co, C1 + C2, generator=g)
    x, W = x.cuda(), W.cuda()
    got = _layer(x[:, :C1].contiguous(), x[:, C1:].contiguous(), W)
    _check_vs_float64(got, W, x, "2^-40 .. 2^40")


@pytest.mark.parametrize("B,C1,C2,Co,P", [(1, 1024, 1024, 1024, 4800), (1, 36, 8, 70, 50)], ids=["ds3", "ragged"])
def test_fusion_mlp_forward_cancellation(cuda, B, C1, C2, Co, P):
    """Zero-sum weight rows (each row's float64 mean removed) applied to features 4 + N(0,1), the forward's analogue
    of the weight gradient's "centred" case: the output is a small fraction of sum |W||x|.  Within the bound, no worse
    than 8x torch fp32, and within 1e-5 of the output scale (BASELINE.json)."""
    g = torch.Generator().manual_seed(C1 + P)
    W = torch.randn(Co, C1 + C2, generator=g, dtype=torch.float64) / (C1 + C2) ** 0.5
    W = (W - W.mean(1, keepdim=True)).float()
    x = 4 + torch.randn(B, C1 + C2, P, generator=g)
    x, W = x.cuda(), W.cuda()
    got = _layer(x[:, :C1].contiguous(), x[:, C1:].contiguous(), W)
    e, _ = _check_vs_float64(got, W, x, "cancellation %d+%d->%d" % (C1, C2, Co))
    want = torch.matmul(W.double(), x.double())
    assert e <= 1e-5 * max(want.abs().max().item(), 1.0)
    assert want.abs().mean().item() < 0.1 * torch.matmul(W.double().abs(), x.double().abs()).mean().item()
