"""CPU: both orders of PSPUpsample's upsampling + 3x3 conv in oracle/upconv_oracle.py, and their adjoints, against
torch's float64 autograd of ``nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True) -> nn.Conv2d(3x3,
padding=1)``, at maps of one row or column, odd and non-square sizes (DESIGN.md §4.23)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import upconv_oracle as U

SHAPES = [(1, 3, 2, 1, 1), (2, 4, 3, 1, 5), (1, 2, 5, 6, 1), (2, 5, 3, 3, 3), (1, 3, 4, 7, 4), (2, 6, 2, 4, 9)]


def torch64(x, w, b, dz):
    xt = torch.from_numpy(x).requires_grad_(True)
    wt = torch.from_numpy(w).requires_grad_(True)
    bt = torch.from_numpy(b).requires_grad_(True)
    z = F.conv2d(F.interpolate(xt, scale_factor=2, mode="bilinear", align_corners=True), wt, bt, padding=1)
    z.backward(torch.from_numpy(dz))
    return z.detach().numpy(), xt.grad.numpy(), wt.grad.numpy(), bt.grad.numpy()


@pytest.mark.parametrize("B,Ci,Co,Hi,Wi", SHAPES)
def test_both_orders_and_adjoints_match_torch_float64(B, Ci, Co, Hi, Wi):
    rs = np.random.RandomState(B * 1000 + Ci * 100 + Hi * 10 + Wi)
    x = rs.randn(B, Ci, Hi, Wi)
    w = rs.randn(Co, Ci, 3, 3)
    b = rs.randn(Co)
    dz = rs.randn(B, Co, 2 * Hi, 2 * Wi)
    z, dx, dw, db = torch64(x, w, b, dz)
    for fwd, bwd in ((U.forward_reference, U.backward_reference), (U.forward_restructured, U.backward_restructured)):
        for got, want in zip((fwd(x, w, b),) + bwd(x, w, dz), (z, dx, dw, db)):
            assert got.shape == want.shape
            assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_tap_adjoint_is_the_transpose_of_the_tap_sum():
    """<sum_t S_t up(T_t), dz> == sum_t <T_t, G_t> for random T and dz, on an odd, non-square map."""
    rs = np.random.RandomState(7)
    Hi, Wi = 3, 5
    t = rs.randn(2, 9, 4, Hi, Wi)
    dz = rs.randn(2, 4, 2 * Hi, 2 * Wi)
    uy, ux = U.up_matrix(Hi, 2 * Hi), U.up_matrix(Wi, 2 * Wi)
    z = sum(U._plane(U._plane(t[:, k], uy, ux), U.shift_matrix(2 * Hi, k // 3 - 1), U.shift_matrix(2 * Wi, k % 3 - 1))
            for k in range(9))
    lhs = (z * dz).sum()
    rhs = (t * U.taps_adjoint(dz, Hi, Wi)).sum()
    assert abs(lhs - rhs) <= 1e-12 * abs(lhs)
