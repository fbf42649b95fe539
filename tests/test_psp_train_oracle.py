"""CPU: the float64 restatement of the PSP head's restructured backward (oracle/psp_train_oracle.py, explicit pool and
tap matrices) equals torch.autograd of ``cnn.PSPModule.double()`` and of ``F.interpolate(align_corners=True)``, at
shapes whose bins overlap or repeat (H, W not divisible by 3 or 6, maps smaller than 6, 1x1 maps) and with Hi = 1
for the x2 upsampling.  This pins the bin and tap conventions the kernels share."""
import pytest
import torch
import torch.nn.functional as Fn

from ffb6d_b200 import cnn
from oracle import psp_train_oracle as O

TOL = 1e-12


def close(got, want, what):
    scale = max(want.abs().max().item(), 1e-300)
    err = (got - want).abs().max().item()
    assert err <= TOL * scale, "%s: %.3e of scale %.3e" % (what, err / scale, scale)


SHAPES = [(2, 5, 7, 11, 9), (1, 4, 13, 17, 6), (3, 3, 5, 4, 7), (2, 3, 1, 1, 4), (1, 6, 2, 5, 3), (1, 2, 6, 1, 5),
          (2, 4, 12, 18, 8)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_psp_backward_matches_autograd(shape):
    B, C, H, W, Co = shape
    torch.manual_seed(sum(shape))
    m = cnn.PSPModule(C, Co).double()
    with torch.no_grad():
        m.bottleneck.bias.normal_(0, 0.5)
    x = torch.randn(B, C, H, W, dtype=torch.float64, requires_grad=True)
    out = m(x)
    grad = torch.randn_like(out)
    out.backward(grad)
    stage_w = [st[1].weight.detach() for st in m.stages]
    close(O.psp_forward(x.detach(), stage_w, m.bottleneck.weight.detach(), m.bottleneck.bias.detach()), out.detach(),
          "forward")
    dx, dcs, dw, db = O.psp_backward(x.detach(), stage_w, m.bottleneck.weight.detach(), m.bottleneck.bias.detach(),
                                     grad)
    close(dx, x.grad, "dx")
    for s, dc, st in zip(O.PSP_SIZES, dcs, m.stages):
        close(dc, st[1].weight.grad, "stage conv %d" % s)
    C5 = C * 5
    for i in range(5):
        close(dw.reshape(Co, C5)[:, i * C:(i + 1) * C], m.bottleneck.weight.grad.reshape(Co, C5)[:, i * C:(i + 1) * C],
              "bottleneck block %d" % i)
    close(db, m.bottleneck.bias.grad, "bias")


def test_psp_relu_mask_is_torchs():
    """torch's ReLU backward on its result masks where out <= 0 and passes the gradient where out is NaN."""
    out = torch.tensor([[[[float("nan"), 0.0, -0.0, 1.0]]]], dtype=torch.float64)
    x = out.clone().requires_grad_(True)
    torch.relu(x).backward(torch.ones_like(x))
    assert x.grad.flatten().tolist() == [1.0, 0.0, 0.0, 1.0]


@pytest.mark.parametrize("shape", [(2, 3, 5, 7), (1, 2, 1, 4), (1, 1, 1, 1), (2, 2, 3, 1), (1, 3, 60, 80)],
                         ids=lambda s: "x".join(map(str, s)))
def test_upsample_backward_matches_autograd(shape):
    torch.manual_seed(sum(shape))
    x = torch.randn(shape, dtype=torch.float64, requires_grad=True)
    y = Fn.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
    g = torch.randn_like(y)
    y.backward(g)
    close(O.upsample_ac_backward(g, shape[2:]), x.grad, "upsample backward %s" % (shape,))


@pytest.mark.parametrize("n_in,n_out", [(1, 2), (5, 10), (7, 3), (4, 1), (60, 120)])
def test_tap_matrix_rows_sum_to_one(n_in, n_out):
    for ac in (False, True):
        u = O.tap_matrix(n_out, n_in, ac)
        assert torch.allclose(u.sum(1), torch.ones(n_out, dtype=torch.float64), atol=1e-15, rtol=0)
