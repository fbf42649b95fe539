"""GPU: TRAINING mode of the 1x1 layers and RandLA blocks (batch-statistics BatchNorm, backward) against
the reference's own modules run in training mode with autograd (tests/golden/train_cases.npz, made by
tests/golden/make_golden.py from models/pytorch_utils.py and models/RandLA/RandLANet.py).  The modules are
loaded through ``load_state_dict(strict=True)`` with the reference's state dicts: parameter names are part
of the contract.  Floating point: 1e-5 of each tensor's scale.

At training shapes (seeded inputs, no fixtures) every kernel and module path is also held to float64 torch
on the GPU: 1e-5 of each tensor's scale, or -- where fp32 numerics are inherently worse -- no worse than a
small multiple of torch's own fp32 CUDA path on the same inputs; running statistics element-wise."""
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F_

import ffb6d_b200 as F
from ffb6d_b200 import modules as M
from ffb6d_b200._lib import lib, check
from ffb6d_b200.ops import _stream
from conftest import GOLDEN

pytestmark = pytest.mark.gpu


def load(name):
    z = np.load(os.path.join(GOLDEN, "train_cases.npz"))
    return {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "/")}


def close(got, want, what, tol=1e-5):
    got = got.detach().cpu().numpy().astype(np.float64) if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = max(np.abs(want).max(), 1e-3)
    err = np.abs(got - want).max()
    assert err <= tol * scale, "%s: max abs err %.3e at scale %.3e (%.2e relative)" % (what, err, scale, err / scale)


def sd_of(case, prefix="sd."):
    return {k[len(prefix):]: torch.from_numpy(v) for k, v in case.items() if k.startswith(prefix)}


def close_fp32(got, want, ref32, what, tol=1e-5, factor=4, inherent=0.0, why=""):
    """Device tensors: max |got - want| <= tol * scale(want), or <= factor * torch fp32's own error where
    that is larger (the numerics are inherently worse there), or <= ``inherent``, an error the fp32 result
    cannot avoid (``why``).  The message names the bound that applied."""
    want = want.detach().double()
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    if want.numel() == 0:
        return
    scale = max(want.abs().max().item(), 1e-3)
    err = (got.detach().double() - want).abs().max().item()
    e32 = (ref32.detach().double() - want).abs().max().item() if ref32 is not None else 0.0
    bound, which = max((tol * scale, "%g of scale" % tol), (factor * e32, "%gx torch fp32's error %.3e" % (factor, e32)),
                       (inherent, why), key=lambda b: b[0])
    assert err <= bound, "%s: max abs err %.3e at scale %.3e (%.2e relative), bound %s" % (
        what, err, scale, err / scale, which)


def close_elementwise(got, want, tol, what):
    """Device tensors: |got - want| <= tol element-wise (tol a tensor or a number)."""
    err = (got.detach().double() - want.detach().double()).abs()
    tol = torch.as_tensor(tol, dtype=torch.float64, device=err.device).expand_as(err)
    bad = err > tol
    if bad.any():
        i = int((err - tol).argmax())
        raise AssertionError("%s: %d elements out of bound, the worst has err %.3e where the bound is %.3e" % (
            what, int(bad.sum()), err.flatten()[i].item(), tol.flatten()[i].item()))


def act_fn(act, slope):
    return {0: lambda t: t, 1: torch.relu, 2: lambda t: F_.leaky_relu(t, slope)}[act]


def away_from_kink(g, pre64, act):
    """The upstream gradient with the elements whose float64 pre-activation lies within 1e-4 of its scale
    of the activation's kink set to zero.  fp32 puts a few of the millions of elements on the other side of
    zero there; the derivative's jump would then measure the rounding of the forward, not the backward."""
    if act == 0:
        return g
    p = pre64.detach().abs()
    return g * (p > 1e-4 * p.max()).to(g.dtype)


# ------------------------------------------------------------------ batch-statistics BatchNorm through the C ABI
def cdiv(a, b):
    return -(-a // b)


def bn_split_plan(C, P, num_sms):
    """train.cu's split_plan: about two CTAs per SM over (split, channel), chunks of whole 1024-position
    strides.  Returns (chunk, nsplit)."""
    want = max(1, cdiv(2 * num_sms, C))
    chunk = max(1024, cdiv(cdiv(P, want), 1024) * 1024)
    return chunk, cdiv(P, chunk)


def bn_workspace_bytes(C, nsplit):
    align = lambda n: cdiv(n, 256) * 256     # noqa: E731
    return align(C * nsplit * 2 * 8) + align(C * 8)


# (B, C, P): RandLA ds0 in training (12288 points x K=16), the fusion ds0 image map (120 x 160), ds3 (60 x 80,
# 1024 channels: more than one finalize block), a ragged P (scalar path) that still splits, one channel of 10
BN_SHAPES = [(4, 16, 196608), (8, 64, 19200), (8, 1024, 4800), (3, 7, 4099), (2, 1, 5)]
BN_DISTS = ["randn", "offset10", "offset100", "offset1000", "const"]


def test_bn_train_shapes_cover_split_reductions(cuda):
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    plans = {}
    for B, C, P in BN_SHAPES:
        chunk, nsplit = bn_split_plan(C, P, sms)
        assert lib.ffb6d_bn_workspace_bytes(C, P) == bn_workspace_bytes(C, nsplit), (C, P)
        plans[(C, P)] = nsplit
    assert plans[(16, 196608)] > 8                      # RandLA ds0: many chunks per channel
    assert plans[(64, 19200)] > 1
    assert plans[(7, 4099)] > 1 and 4099 % 4 != 0       # split reductions on the scalar path
    assert max(C for _, C, _ in BN_SHAPES) > 256        # bn_finalize_kernel over more than one block


@pytest.mark.parametrize("dist", BN_DISTS)
@pytest.mark.parametrize("eps,momentum", [(1e-5, 0.1), (1e-6, 0.99)], ids=["fusion", "randla"])
@pytest.mark.parametrize("act,slope", [(0, 0.0), (1, 0.0), (2, 0.2)], ids=["none", "relu", "leaky"])
@pytest.mark.parametrize("B,C,P", BN_SHAPES)
def test_bn_train_vs_float64(cuda, B, C, P, act, slope, eps, momentum, dist):
    """ffb6d_bn_train_fwd / _bwd against F.batch_norm(training=True) -> activation -> autograd in float64.
    ``offsetR``: every channel's |mean| is R times its std; ``const``: one channel is exactly constant, so
    its variance is 0 and its normalised value must be exactly 0."""
    g = torch.Generator(device=cuda).manual_seed(B * 7919 + C * 104729 + P + 31 * act + 1000 * BN_DISTS.index(dist))
    z = torch.randn(B, C, P, generator=g, device=cuda)
    if dist.startswith("offset"):
        std = torch.exp(torch.rand(C, generator=g, device=cuda) * 2 - 1)
        sign = torch.where(torch.rand(C, generator=g, device=cuda) < 0.5, -1.0, 1.0)
        z = z * std[:, None] + (sign * float(dist[6:]) * std)[:, None]
    cc = C - 1 if dist == "const" else None
    if cc is not None:
        z[:, cc] = 0.3
    gamma = 1 + 0.5 * torch.randn(C, generator=g, device=cuda)
    beta = 0.5 * torch.randn(C, generator=g, device=cuda)
    rm0 = torch.randn(C, generator=g, device=cuda)
    rv0 = torch.rand(C, generator=g, device=cuda) + 0.5
    gy = torch.randn(B, C, P, generator=g, device=cuda)
    f = act_fn(act, slope)

    # float64 reference; running statistics updated by F.batch_norm itself
    z64 = z.double().requires_grad_(True)
    gam64, bet64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm64, rv64 = rm0.double(), rv0.double()
    pre64 = F_.batch_norm(z64, rm64, rv64, gam64, bet64, True, momentum, eps)
    y64 = f(pre64)
    gy = away_from_kink(gy, pre64, act)
    del pre64
    gz64, gg64, gb64 = torch.autograd.grad(y64, (z64, gam64, bet64), gy.double())
    y64 = y64.detach()
    with torch.no_grad():
        mean64 = z64.mean(dim=(0, 2))
        var64 = z64.var(dim=(0, 2), unbiased=False)
    del z64

    # the kernels
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    nbytes = int(lib.ffb6d_bn_workspace_bytes(C, P))
    assert nbytes == bn_workspace_bytes(C, bn_split_plan(C, P, sms)[1])
    ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda)
    stats = torch.empty(C, 4, device=cuda)
    y, dz = torch.empty_like(z), torch.empty_like(z)
    ggam, gbet = torch.empty(C, device=cuda), torch.empty(C, device=cuda)
    rm, rv = rm0.clone(), rv0.clone()
    check(lib.ffb6d_bn_train_fwd(z.data_ptr(), B, C, P, gamma.data_ptr(), beta.data_ptr(), eps, momentum, rm.data_ptr(),
                                 rv.data_ptr(), act, slope, stats.data_ptr(), y.data_ptr(), ws.data_ptr(), nbytes,
                                 _stream(cuda)))
    check(lib.ffb6d_bn_train_bwd(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, C, P, act, slope, ggam.data_ptr(),
                                 gbet.data_ptr(), dz.data_ptr(), ws.data_ptr(), nbytes, _stream(cuda)))

    # torch's own fp32 path on the same inputs
    z32 = z.clone().requires_grad_(True)
    gam32, bet32 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    y32 = f(F_.batch_norm(z32, rm0.clone(), rv0.clone(), gam32, bet32, True, momentum, eps))
    gz32, gg32, gb32 = torch.autograd.grad(y32, (z32, gam32, bet32), gy)
    del z32

    what = "bn_train %s act=%d eps=%g %s" % ((B, C, P), act, eps, dist)
    rest = slice(0, C if cc is None else cc)       # the channels that are not constant
    std64 = (var64 + eps).sqrt()
    # The stats hold the mean in fp32.  Its one rounding moves xhat by up to 2^-24 |mean| / std: 6e-5 at
    # |mean| / std = 1000, a constant offset per channel that torch's fp32 path may or may not happen to
    # share.  Twice what that moves y, dz and grad_gamma by is the bound where it exceeds the others.
    dxhat = (2.0 ** -24 * mean64.abs() / std64)[rest]
    why = "2x what the fp32 mean's rounding moves it by"
    floor_y = 2 * (gamma.double()[rest].abs() * dxhat).max().item() if dxhat.numel() else 0.0
    floor_dz = 2 * (gamma.double()[rest].abs() / std64[rest] * dxhat * gg64[rest].abs() / (B * P)).max().item() if dxhat.numel() else 0.0
    floor_gg = 2 * (dxhat * gb64[rest].abs()).max().item() if dxhat.numel() else 0.0
    close_fp32(y[:, rest], y64[:, rest], y32[:, rest], what + " y", inherent=floor_y, why=why)
    # mean: 1e-5 of the channel's std plus the rounding of its fp32 store; the others relative, element-wise
    close_elementwise(stats[:, 0], mean64, 1e-5 * std64 + 2.0 ** -24 * mean64.abs(), what + " stats mean")
    close_elementwise(stats[:, 1], 1 / std64, 1e-5 / std64, what + " stats invstd")
    close_elementwise(stats[:, 2], gamma.double() / std64, 1e-5 * (gamma.double() / std64).abs(), what + " stats gamma*invstd")
    assert torch.equal(stats[:, 3], beta), what + " stats beta"
    m = momentum
    close_elementwise(rm, rm64, 1e-5 * ((1 - m) * rm0.double().abs() + m * (mean64.abs() + std64)), what + " running_mean")
    close_elementwise(rv, rv64, 1e-5 * rv64.abs(), what + " running_var")
    close_fp32(dz[:, rest], gz64[:, rest], gz32[:, rest], what + " dz", inherent=floor_dz, why=why)
    close_fp32(ggam, gg64, gg32, what + " grad_gamma", inherent=floor_gg, why=why)
    close_fp32(gbet, gb64, gb32, what + " grad_beta")
    if cc is not None:
        # var = 0: mean is the constant itself, xhat = 0 and y = act(beta) bit for bit
        assert stats[cc, 0].item() == z[0, cc, 0].item(), what + " constant channel mean"
        close_elementwise(stats[cc, 1], torch.tensor(eps, dtype=torch.float64).rsqrt(), 1e-6 / eps ** 0.5,
                          what + " constant channel invstd")
        assert torch.equal(y[:, cc], f(beta[cc].expand(B, P))), what + " constant channel y"
        close_fp32(dz[:, cc], gz64[:, cc], gz32[:, cc], what + " constant channel dz")


@pytest.mark.parametrize("name,C1,C2,Co", [("conv_cat", 24, 40, 48), ("conv_pre", 64, 0, 32), ("conv_wide", 256, 256, 128)])
def test_fusion_conv_train_matches_reference(cuda, name, C1, C2, Co):
    c = load(name)
    layer = M.Conv2d(C1 + C2, Co, kernel_size=(1, 1), bn=True)
    sd = sd_of(c)
    sd["normlayer.bn.num_batches_tracked"] = torch.tensor(0)
    layer.load_state_dict(sd, strict=True)
    layer.cuda().train()
    x1 = torch.from_numpy(c["x1"]).cuda().requires_grad_(True)
    x2 = torch.from_numpy(c["x2"]).cuda().requires_grad_(True) if C2 else None
    out = layer(x1, x2)
    close(out, c["out"], name + " out")
    out.backward(torch.from_numpy(c["gout"]).cuda())
    close(x1.grad, c["gx1"], name + " grad x1")
    if C2:
        close(x2.grad, c["gx2"], name + " grad x2")
    close(layer.conv.weight.grad, c["gw"], name + " grad W")
    close(layer.normlayer.bn.weight.grad, c["ggamma"], name + " grad gamma")
    close(layer.normlayer.bn.bias.grad, c["gbeta"], name + " grad beta")
    close(layer.normlayer.bn.running_mean, c["after.normlayer.bn.running_mean"], name + " running_mean")
    close(layer.normlayer.bn.running_var, c["after.normlayer.bn.running_var"], name + " running_var")
    assert int(layer.normlayer.bn.num_batches_tracked) == 1
    # the same layer on the materialised concat (one input tensor) gives the same bits
    layer.zero_grad()
    xa = torch.cat((x1.detach(), x2.detach()), 1) if C2 else x1.detach()
    assert torch.equal(layer(xa), out)
    # eval mode: the fused inference kernel == torch's eval-mode layer
    layer.eval()
    with torch.no_grad():
        got = layer(x1.detach(), x2.detach() if C2 else None)
        bn = layer.normlayer.bn
        ref = torch.relu(torch.nn.functional.batch_norm(
            torch.nn.functional.conv2d(xa.double(), layer.conv.weight.double()), bn.running_mean.double(),
            bn.running_var.double(), bn.weight.double(), bn.bias.double(), False, 0.0, bn.eps))
    close(got, ref.cpu().numpy(), name + " eval")


@pytest.mark.parametrize("name,d_in,d_out", [("blk_train_8_16", 8, 16), ("blk_train_64_64", 64, 64)])
def test_dilated_res_block_train_matches_reference(cuda, name, d_in, d_out):
    c = load(name)
    blk = M.Dilated_res_block(d_in, d_out)
    sd = sd_of(c)
    for k in list(blk.state_dict()):
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0)
    blk.load_state_dict(sd, strict=True)          # the reference's parameter names
    blk.cuda().train()
    feature = torch.from_numpy(c["feature"]).cuda().requires_grad_(True)
    xyz, idx = torch.from_numpy(c["xyz"]).cuda(), torch.from_numpy(c["idx"]).cuda()
    out = blk(feature, xyz, idx)
    close(out, c["out"], name + " out", tol=2e-5)
    out.backward(torch.from_numpy(c["gout"]).cuda())
    close(feature.grad, c["gfeature"], name + " grad feature", tol=5e-5)
    for k, prm in blk.named_parameters():
        close(prm.grad, c["grad." + k], name + " grad " + k, tol=5e-5)
    for k, v in blk.state_dict().items():
        if "running_" in k:
            close(v, c["after." + k], name + " " + k)
    # eval mode (frozen statistics, fused residual GEMM) agrees with the modules' own eval composition
    blk.eval()
    with torch.no_grad():
        got = blk(feature.detach(), xyz, idx)
        f_pc = blk.mlp2(blk.lfa(xyz, blk.mlp1(feature.detach()), idx))
        want = torch.nn.functional.leaky_relu(f_pc + blk.shortcut(feature.detach()), 0.2)
    close(got, want.cpu().numpy(), name + " eval", tol=2e-5)


def test_att_pool_backward_vs_autograd(cuda):
    """Against float64 autograd of sum_k f * softmax_k(att), frame by frame.  Cases: the vectorised K = 16
    kernel (also at a training size, B=4, C=32+32, N=12288), the generic kernel (K = 7, and K = 16 reached
    through a 4-byte storage offset of f1), and logits of +-60 where the softmax saturates."""
    g = torch.Generator().manual_seed(11)
    for (B, C1, C2, N, K, offset, logits) in ((2, 16, 16, 50, 16, 0, "randn"), (1, 5, 0, 33, 7, 0, "randn"),
                                              (4, 32, 32, 12288, 16, 0, "randn"), (2, 16, 16, 1000, 16, 1, "randn"),
                                              (2, 16, 16, 3000, 16, 0, "pm60")):
        n1 = B * C1 * N * K
        f1 = torch.randn(offset + n1, generator=g).cuda()[offset:].view(B, C1, N, K).requires_grad_(True)
        assert (f1.data_ptr() % 16 != 0) == bool(offset)
        f2 = torch.randn(B, C2, N, K, generator=g).cuda().requires_grad_(True) if C2 else None
        if logits == "randn":
            att = torch.randn(B, C1 + C2, N, K, generator=g) * 2
        else:
            sign = torch.where(torch.rand(B, C1 + C2, N, K, generator=g) < 0.5, -1.0, 1.0)
            att = 60 * sign + torch.randn(B, C1 + C2, N, K, generator=g)
        att = att.cuda().requires_grad_(True)
        go = torch.randn(B, C1 + C2, N, 1, generator=g).cuda()
        out = M._AttPool.apply(f1, f2, att)
        out.backward(go)
        what = "att_pool %s offset=%d %s" % ((B, C1, C2, N, K), offset, logits)
        err, scale = {}, {}
        for b in range(B):      # float64 reference one frame at a time (bounded memory)
            f1d, attd = f1[b:b + 1].detach().double().requires_grad_(True), att[b:b + 1].detach().double().requires_grad_(True)
            f2d = f2[b:b + 1].detach().double().requires_grad_(True) if C2 else None
            fs = torch.cat((f1d, f2d), 1) if C2 else f1d
            ref = torch.sum(fs * torch.softmax(attd, dim=3), dim=3, keepdim=True)
            ref.backward(go[b:b + 1].double())
            pairs = [("grad f1", f1.grad, f1d), ("grad att", att.grad, attd)] + ([("grad f2", f2.grad, f2d)] if C2 else [])
            for name, got, want in pairs:
                err[name] = max(err.get(name, 0.0), (got[b:b + 1].double() - want.grad).abs().max().item())
                scale[name] = max(scale.get(name, 1e-3), want.grad.abs().max().item())
        for name in err:
            assert err[name] <= 1e-5 * scale[name], "%s %s: max abs err %.3e at scale %.3e (%.2e relative), bound 1e-05 of scale" % (
                what, name, err[name], scale[name], err[name] / scale[name])


WGRAD_CASES = [(2, 64, 64, 64, 3072), (1, 36, 8, 70, 50), (3, 5, 0, 3, 7), (2, 1024, 1024, 1024, 600), (8, 64, 64, 64, 19200),
               (2, 10, 0, 16, 98304), (2, 32, 32, 64, 1001), (1, 16, 16, 32, 3072),
               # the narrow-layer kernel at RandLA's training size; a wgmma case whose concat boundary and ragged
               # edges cross the 128-tiles
               (4, 32, 32, 64, 196608), (4, 10, 0, 16, 196608), (2, 131, 125, 200, 4097)]
# "centred": dz has zero mean per channel, as BatchNorm's backward leaves it, and x a common offset of 4, as
# post-activation features have -- the sum over positions cancels to a small fraction of its terms
WGRAD_CENTRED = [(4, 32, 32, 64, 196608), (2, 131, 125, 200, 4097)]


@pytest.mark.parametrize("B,C1,C2,Co,P,centred", [pytest.param(*c, False, id="-".join(map(str, c))) for c in WGRAD_CASES]
                         + [pytest.param(*c, True, id="-".join(map(str, c)) + "-centred") for c in WGRAD_CENTRED])
def test_wgrad_vs_float64(cuda, B, C1, C2, Co, P, centred):
    g = torch.Generator().manual_seed(P)
    dz = torch.randn(B, Co, P, generator=g).cuda()
    x1 = torch.randn(B, C1, P, generator=g).cuda()
    x2 = torch.randn(B, C2, P, generator=g).cuda() if C2 else None
    if centred:
        dz = (dz.double() - dz.double().mean(dim=(0, 2), keepdim=True)).float()
        x1 += 4
        if C2:
            x2 += 4
    gw = torch.full((Co, C1 + C2), float("nan"), device="cuda")
    check(lib.ffb6d_fusion_mlp_wgrad(dz.data_ptr(), x1.data_ptr(), C1, x2.data_ptr() if C2 else None, C2, B, Co, P,
                                     gw.data_ptr(), _stream(dz.device)))
    x = torch.cat((x1, x2), 1) if C2 else x1
    want = sum(dz[b].double() @ x[b].double().t() for b in range(B))     # one frame at a time (bounded memory)
    ref32 = torch.einsum("bop,bcp->oc", dz, x)
    e_ours = (gw.double() - want).abs().max().item()
    e_32 = (ref32.double() - want).abs().max().item()
    scale = want.abs().max().item()
    if not centred:
        close_fp32(gw, want, None, "wgrad")
    assert e_ours <= max(8 * e_32, 1e-6 * scale), (
        "wgrad%s: max abs err %.3e at scale %.3e, bound max(8x torch fp32's error %.3e, 1e-6 of scale)"
        % (" centred" if centred else "", e_ours, scale, e_32))


# ------------------------------------------------------------------ module paths against the torch modules in float64
def torch_twin(layer, activation):
    """The plain torch layer with ``layer``'s state-dict keys: conv [-> <bn name>.bn] [-> activation]."""
    conv = layer._conv
    mods = OrderedDict(conv=type(conv)(conv.in_channels, conv.out_channels, 1, bias=conv.bias is not None))
    if layer.has_bn:
        bn = layer._bn
        mods[layer._bn_name] = nn.Sequential(OrderedDict(bn=type(bn)(bn.num_features, eps=bn.eps, momentum=bn.momentum)))
    if activation is not None:
        mods["activation"] = activation
    twin = nn.Sequential(mods)
    twin.load_state_dict(layer.state_dict(), strict=True)
    return twin


def randomise(layer, g):
    """Non-trivial parameters and running statistics (the modules initialise bias 0, gamma 1, beta 0)."""
    with torch.no_grad():
        if layer._conv.bias is not None:
            layer._conv.bias.copy_(torch.randn(layer._conv.bias.shape, generator=g))
        if layer.has_bn:
            bn = layer._bn
            bn.weight.copy_(1 + 0.5 * torch.randn(bn.num_features, generator=g))
            bn.bias.copy_(0.5 * torch.randn(bn.num_features, generator=g))
            bn.running_mean.copy_(torch.randn(bn.num_features, generator=g))
            bn.running_var.copy_(torch.rand(bn.num_features, generator=g) + 0.5)


def check_layer_vs_float64(layer, activation, x_shape, training, seed, what):
    """One forward + backward of ``layer`` (on this package's kernels) against its torch twin in float64, with
    torch's fp32 twin as the yardstick where fp32 is inherently worse: output, input / weight / bias / BN
    gradients, running statistics (element-wise) and num_batches_tracked."""
    g = torch.Generator().manual_seed(seed)
    randomise(layer, g)
    before = {k: v.double().cuda() for k, v in layer.state_dict().items() if "running_" in k}
    twin64 = torch_twin(layer, activation).double().cuda().train(training)
    twin32 = torch_twin(layer, activation).cuda().train(training)
    layer.cuda().train(training)
    x = torch.randn(x_shape, generator=g).cuda()
    gy = torch.randn((x_shape[0], layer._conv.out_channels) + tuple(x_shape[2:]), generator=g).cuda()

    x64 = x.double().requires_grad_(True)
    pre64 = twin64[:-1](x64) if activation is not None else twin64(x64)
    y64 = twin64[-1](pre64) if activation is not None else pre64
    gy = away_from_kink(gy, pre64, 1 if activation is not None else 0)
    names = [k for k, _ in twin64.named_parameters()]
    grads64 = torch.autograd.grad(y64, [x64] + [p for _, p in twin64.named_parameters()], gy.double())

    x32 = x.clone().requires_grad_(True)
    y32 = twin32(x32)
    grads32 = torch.autograd.grad(y32, [x32] + [p for _, p in twin32.named_parameters()], gy)

    xk = x.clone().requires_grad_(True)
    y = layer(xk)
    y.backward(gy)
    close_fp32(y, y64, y32, what + " out")
    ours = dict(layer.named_parameters())
    assert sorted(ours) == sorted(names), (sorted(ours), names)
    close_fp32(xk.grad, grads64[0], grads32[0], what + " grad x")
    for k, w64, w32 in zip(names, grads64[1:], grads32[1:]):
        close_fp32(ours[k].grad, w64, w32, what + " grad " + k)
    sd, sd64 = layer.state_dict(), twin64.state_dict()
    for k in sd:
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(sd64[k]), (what, k, int(sd[k]), int(sd64[k]))
        elif "running_" in k:     # relative to the update's terms: (1 - m) * before and m * batch statistic
            close_elementwise(sd[k], sd64[k], 1e-5 * (sd64[k].abs() + before[k].abs()), what + " " + k)


def test_layer_without_bn_train_vs_float64(cuda):
    """No BatchNorm, an activation and a conv bias: the bias is the GEMM's shift, its gradient dz.sum, and the
    activation's backward is ffb6d_act_bwd."""
    torch.manual_seed(0)
    check_layer_vs_float64(M.Conv1d(128, 64, bn=False, activation=nn.ReLU(), bias=True), nn.ReLU(),
                           (4, 128, 12288), True, 1, "Conv1d(bn=False, ReLU, bias)")
    check_layer_vs_float64(M.RandLAConv2d(10, 16, bn=False), nn.LeakyReLU(0.2), (4, 10, 12288, 16), True, 2,
                           "RandLAConv2d(bn=False, LeakyReLU)")


def test_eval_bn_under_autograd_vs_float64(cuda):
    """Frozen-BN fine-tuning: eval() with inputs and parameters that require grad."""
    torch.manual_seed(0)
    check_layer_vs_float64(M.Conv2d(128, 64, bn=True), nn.ReLU(), (2, 128, 120, 160), False, 3, "Conv2d(bn=True).eval()")


@pytest.mark.parametrize("kind,Ci,Co", [("Conv1d", 128, 64), ("RandLAConv1d", 9, 8)])
def test_conv1d_bn_train_vs_float64(cuda, kind, Ci, Co):
    torch.manual_seed(0)
    layer, act = (M.Conv1d(Ci, Co, bn=True), nn.ReLU()) if kind == "Conv1d" else (M.RandLAConv1d(Ci, Co, bn=True), nn.LeakyReLU(0.2))
    check_layer_vs_float64(layer, act, (8, Ci, 12288), True, 4, kind + "(bn=True).train()")


def test_bn_momentum_none_is_a_cumulative_average(cuda):
    """nn.BatchNorm2d(momentum=None) averages the batch statistics with factor 1/num_batches_tracked."""
    torch.manual_seed(0)
    layer = M.Conv2d(16, 8, bn=True)
    layer.normlayer.bn.momentum = None
    twin = torch_twin(layer, None).double().cuda().train()
    assert twin.normlayer.bn.momentum is None
    layer.cuda().train()
    g = torch.Generator().manual_seed(5)
    for step in range(3):
        x = (torch.randn(2, 16, 30, 40, generator=g) + 1 + step).cuda()
        with torch.no_grad():
            layer(x)
            twin(x.double())
        bn, bn64 = layer.normlayer.bn, twin.normlayer.bn
        assert int(bn.num_batches_tracked) == int(bn64.num_batches_tracked) == step + 1
        close_elementwise(bn.running_mean, bn64.running_mean, 1e-5 * bn64.running_mean.abs() + 1e-6,
                          "momentum=None step %d running_mean" % step)
        close_elementwise(bn.running_var, bn64.running_var, 1e-5 * bn64.running_var.abs(),
                          "momentum=None step %d running_var" % step)


def test_one_value_per_channel_is_rejected_in_training(cuda):
    """As torch's BatchNorm: training statistics over one value per channel raise ValueError."""
    torch.manual_seed(0)
    for layer, shape in ((M.Conv2d(4, 8, bn=True), (1, 4, 1, 1)), (M.RandLAConv1d(4, 8, bn=True), (1, 4, 1))):
        layer.cuda().train()
        twin = torch_twin(layer, None).cuda().train()
        x = torch.randn(shape, device=cuda)
        with pytest.raises(ValueError, match="more than 1 value per channel"):
            twin(x)
        before = {k: v.clone() for k, v in layer.state_dict().items()}
        with pytest.raises(ValueError, match="more than 1 value per channel"):
            layer(x)
        for k, v in layer.state_dict().items():
            assert torch.equal(v, before[k]), k      # a rejected batch leaves the statistics alone
        layer(torch.randn((2,) + shape[1:], device=cuda))      # two values per channel are fine
        layer.eval()
        with torch.no_grad():
            layer(x)                                           # and eval mode needs no batch statistics
