"""CPU: the float64 LFA oracle (oracle/lfa_oracle.py) against the outputs of the reference's own RandLA modules
(tests/golden/lfa_cases.npz, made by tests/golden/make_golden.py), so that the GPU tests that compare the fused
attentive pooling with the oracle rest on the reference's composition.  The golden outputs are fp32: 1e-5 of scale."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import lfa_oracle as L

CASES = ["blk_8_16", "blk_32_32", "ffb6d_ds0", "ffb6d_ds1", "ffb6d_ds2", "ffb6d_ds3"]


def load_case(name):
    z = np.load(os.path.join(GOLDEN, "lfa_cases.npz"))
    case, sd = {}, {}
    for k in z.files:
        if k.startswith(name + "/"):
            f = k[len(name) + 1:]
            (sd if f.startswith("sd.") else case)[f[3:] if f.startswith("sd.") else f] = torch.from_numpy(z[k])
    return case, sd


def within(got, want, what):
    want = want.double()
    scale = max(want.abs().max().item(), 1.0)
    err = (got - want).abs().max().item()
    assert got.dtype == torch.float64 and got.shape == want.shape, what
    assert err <= 1e-5 * scale, "%s: max abs err %.3e at scale %.3e" % (what, err, scale)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_modules(name):
    c, sd = load_case(name)
    xyz, idx, feature = c["xyz"], c["idx"], c["feature"]
    within(L.fusion_layer(feature, None, *L.fold(sd, "mlp1"), L.ACT_LEAKY, 0.2), c["mlp1_out"], name + " mlp1")
    within(L.building_block(sd, "lfa", xyz, c["mlp1_out"], idx), c["lfa_out"], name + " building_block")
    within(L.dilated_res_block(sd, feature, xyz, idx), c["out"], name + " dilated_res_block")
    # int32 indices read the same neighbours
    assert torch.equal(L.building_block(sd, "lfa", xyz, c["mlp1_out"], idx.int()),
                       L.building_block(sd, "lfa", xyz, c["mlp1_out"], idx))


def test_fusion_layer_addend_and_activations():
    """The epilogue addend is a gather along the point axis added before the affine; the three activations."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 7, generator=g)
    w, sc, sh = torch.randn(3, 5, generator=g), torch.rand(3, generator=g) + 0.5, torch.randn(3, generator=g)
    add = torch.randn(2, 4, 3, generator=g)
    idx = torch.randint(0, 4, (2, 7), generator=g)
    z = torch.einsum("oc,bcp->bop", w.double(), x.double())
    z = z + torch.stack([add[b].double()[idx[b]].t() for b in range(2)])
    pre = z * sc.double()[:, None] + sh.double()[:, None]
    for act, slope, want in ((0, 0.0, pre), (1, 0.0, pre.clamp_min(0)), (2, 0.1, torch.where(pre > 0, pre, 0.1 * pre))):
        assert torch.allclose(L.fusion_layer(x, None, w, sc, sh, act, slope, add=add, add_idx=idx), want, rtol=1e-14, atol=0)
