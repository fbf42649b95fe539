"""GPU: RandLA local feature aggregation (Att_pooling, Building_block, Dilated_res_block) assembled
from this package's kernels, against outputs of the reference's own classes (tests/golden/lfa_cases.npz,
made by tests/golden/make_golden.py).  Floating point: 1e-5 of the output scale."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import randla

pytestmark = pytest.mark.gpu


def load_case(path, name):
    z = np.load(path)
    case, sd = {}, {}
    for k in z.files:
        if not k.startswith(name + "/"):
            continue
        f = k[len(name) + 1:]
        if f.startswith("sd."):
            sd[f[3:]] = torch.from_numpy(z[k]).cuda()
        else:
            case[f] = z[k]
    return case, sd


def close(got, want, what):
    """1e-5 of the output scale for every element AND element-wise relative 1e-4 above an absolute
    floor of 10 % of the scale (a composition of six fp32 GEMM layers: the reference's own CPU/GPU
    paths differ by this much)."""
    scale = max(np.abs(want).max(), 1.0)
    d = np.abs(got.astype(np.float64) - want)
    assert d.max() <= 1e-5 * scale, "%s: max abs err %.3e, output scale %.3e" % (what, d.max(), scale)
    big = np.abs(want) > 0.1 * scale
    rel = (d[big] / np.abs(want[big])).max() if big.any() else 0.0
    assert rel <= 1e-4, "%s: max element-wise relative err %.3e" % (what, rel)


@pytest.mark.parametrize("name", ["blk_8_16", "blk_32_32", "ffb6d_ds0", "ffb6d_ds1", "ffb6d_ds2", "ffb6d_ds3"])
def test_dilated_res_block_matches_reference(cuda, name):
    import os
    from conftest import GOLDEN
    c, sd = load_case(os.path.join(GOLDEN, "lfa_cases.npz"), name)
    feature = torch.from_numpy(c["feature"]).cuda()
    xyz = torch.from_numpy(c["xyz"]).cuda()
    idx = torch.from_numpy(c["idx"]).cuda()
    # first conv
    w, scale, shift = randla._conv_bn(sd, "mlp1")
    f_pc = F.fusion_mlp(feature, None, w, scale, shift, negative_slope=0.2)
    close(f_pc.cpu().numpy(), c["mlp1_out"], "mlp1")
    # local feature aggregation (relative position encoding, 2 neighbour gathers, 2 attentive poolings)
    f1 = torch.from_numpy(c["mlp1_out"]).cuda()
    for fused in (True, False):      # one fused kernel per attentive pooling / the per-op kernels
        lfa = randla.building_block(sd, "lfa", xyz, f1, idx, fused=fused)
        close(lfa.cpu().numpy(), c["lfa_out"], "building_block fused=%s" % fused)
        out = randla.dilated_res_block(sd, "", feature, xyz, idx, fused=fused)
        assert out.shape == c["out"].shape
        close(out.cpu().numpy(), c["out"], "dilated_res_block fused=%s" % fused)
    # int32 indices (what the index build produces) == int64
    assert torch.equal(randla.building_block(sd, "lfa", xyz, f1, idx.int()), randla.building_block(sd, "lfa", xyz, f1, idx))


def test_att_pool_against_torch(cuda):
    """The kernels for K = 8, 16, 32 and the generic one (K = 1, 2, 7, 33, 64); at K = 16 also an f1 that starts
    4 bytes past a 16-byte boundary (the element-wise loads) and logits of +-60, where the softmax saturates."""
    g = torch.Generator().manual_seed(3)
    for (B, C1, C2, N, K, offset, logits) in ((2, 16, 16, 50, 16, 0, "randn"), (1, 5, 0, 33, 7, 0, "randn"),
                                              (1, 8, 8, 20, 32, 0, "randn"), (2, 6, 3, 40, 1, 0, "randn"),
                                              (2, 4, 4, 30, 2, 0, "randn"), (2, 8, 8, 50, 8, 0, "randn"),
                                              (1, 5, 3, 20, 33, 0, "randn"), (1, 8, 0, 25, 64, 0, "randn"),
                                              (2, 16, 16, 100, 16, 1, "randn"), (2, 16, 16, 300, 16, 0, "pm60"),
                                              (1, 8, 8, 40, 8, 0, "pm60"), (1, 4, 4, 20, 33, 0, "pm60")):
        f1 = torch.randn(offset + B * C1 * N * K, generator=g).cuda()[offset:].view(B, C1, N, K)
        assert (f1.data_ptr() % 16 != 0) == bool(offset)
        f2 = torch.randn(B, C2, N, K, generator=g).cuda() if C2 else None
        if logits == "randn":
            att = torch.randn(B, C1 + C2, N, K, generator=g) * 3
        else:
            sign = torch.where(torch.rand(B, C1 + C2, N, K, generator=g) < 0.5, -1.0, 1.0)
            att = 60 * sign + torch.randn(B, C1 + C2, N, K, generator=g)
        att = att.cuda()
        fs = torch.cat((f1, f2), 1) if f2 is not None else f1
        want = torch.sum(fs.double() * torch.softmax(att.double(), dim=3), dim=3, keepdim=True)   # RandLANet.py:245-248
        got = F.att_pool(f1, f2, att)
        close(got.cpu().numpy(), want.cpu().numpy(), "att_pool %s offset=%d %s" % ((B, C1, C2, N, K), offset, logits))


def test_relative_pos_encoding_channel_major(cuda):
    g = torch.Generator().manual_seed(4)
    xyz = torch.randn(2, 70, 3, generator=g).cuda()
    idx = torch.randint(0, 70, (2, 70, 16), generator=g).cuda()
    a = F.relative_pos_encoding(xyz, idx)
    b = F.relative_pos_encoding(xyz, idx, channel_major=True)
    assert torch.equal(a.permute(0, 3, 1, 2).contiguous(), b)
