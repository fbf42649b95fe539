"""Float64 restatement of the PSP head's restructured training path (DESIGN.md §4.17, §4.18) with explicit matrices,
so that its bin and tap conventions are pinned on the CPU against torch's own modules:

* ``pool_matrix(n, s)`` [s, n]: torch's adaptive-average bins along an axis (bin i covers
  [floor(i n / s), ceil((i + 1) n / s)), overlapping where s does not divide n); ``A_s = kron(P_H, P_W)`` [s², HW].
* ``tap_matrix(n_out, n_in, align_corners)`` [n_out, n_in]: torch's bilinear taps along an axis (both taps added,
  weight 0 included); ``U_s = kron(U_H, U_W)`` [HW, s²].

With ``M_s = W_s C_s``, ``p_s = x A_s^T``, ``T_s = M_s p_s`` the forward is ``out = relu(W_f x + b + sum_s T_s U_s^T)``,
and the backward the adjoints: ``gz = threshold_backward(grad, out, 0)``, ``dT_s = gz U_s``,
``dM_s = sum_b dT_s p_s^T``, ``dW_s = dM_s C_s^T``, ``dC_s = W_s^T dM_s``, ``dp_s = M_s^T dT_s``,
``dW_f = sum_b gz x^T``, ``db = sum gz``, ``dx = W_f^T gz + sum_s dp_s A_s``."""
import torch

PSP_SIZES = (1, 2, 3, 6)


def pool_matrix(n, s):
    p = torch.zeros(s, n, dtype=torch.float64)
    for i in range(s):
        lo, hi = (i * n) // s, -((-(i + 1) * n) // s)
        p[i, lo:hi] = 1.0 / (hi - lo)
    return p


def tap_matrix(n_out, n_in, align_corners):
    u = torch.zeros(n_out, n_in, dtype=torch.float64)
    for d in range(n_out):
        if align_corners:
            src = d * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
        else:
            src = max(n_in / n_out * (d + 0.5) - 0.5, 0.0)
        i0 = min(int(src), n_in - 1)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        l1 = src - i0
        u[d, i0] += 1.0 - l1
        u[d, i1] += l1
    return u


def pool2d(H, W, s):
    return torch.kron(pool_matrix(H, s), pool_matrix(W, s))                        # [s*s, H*W]


def taps2d(H, W, s, align_corners=False):
    return torch.kron(tap_matrix(H, s, align_corners), tap_matrix(W, s, align_corners))   # [H*W, s*s]


def _split(weight, stage_weights):
    C = stage_weights[0].shape[0]
    w = weight.reshape(weight.shape[0], -1).double()
    ws = [w[:, i * C:(i + 1) * C] for i in range(len(PSP_SIZES))]
    return C, ws, w[:, len(PSP_SIZES) * C:], [c.reshape(C, C).double() for c in stage_weights]


def psp_forward(x, stage_weights, weight, bias):
    """``out [B,Co,H,W]`` of PSPModule, restructured, in float64."""
    B, C, H, W = x.shape
    _, ws, wf, cs = _split(weight, stage_weights)
    xf = x.double().reshape(B, C, H * W)
    z = torch.einsum("oc,bcp->bop", wf, xf) + bias.double()[None, :, None]
    for s, w_s, c_s in zip(PSP_SIZES, ws, cs):
        p = xf @ pool2d(H, W, s).t()                                                 # [B, C, s*s]
        z = z + (w_s @ c_s) @ p @ taps2d(H, W, s).t()
    return torch.relu(z).reshape(B, -1, H, W)


def psp_backward(x, stage_weights, weight, bias, grad_out):
    """``(dx, [dC_s], dweight, dbias)`` of PSPModule for ``grad_out``, restructured, in float64."""
    B, C, H, W = x.shape
    _, ws, wf, cs = _split(weight, stage_weights)
    xf = x.double().reshape(B, C, H * W)
    out = psp_forward(x, stage_weights, weight, bias).reshape(B, -1, H * W)
    g = grad_out.double().reshape(out.shape)
    gz = torch.where(out <= 0, torch.zeros_like(g), g)
    dx = torch.einsum("oc,bop->bcp", wf, gz)
    dws, dcs = [], []
    for s, w_s, c_s in zip(PSP_SIZES, ws, cs):
        a = pool2d(H, W, s)
        p = xf @ a.t()
        dT = gz @ taps2d(H, W, s)                                                   # [B, Co, s*s]
        dM = torch.einsum("bon,bcn->oc", dT, p)
        dws.append(dM @ c_s.t())
        dcs.append((w_s.t() @ dM).reshape(stage_weights[0].shape))
        dx = dx + torch.einsum("oc,bon->bcn", w_s @ c_s, dT) @ a
    dws.append(torch.einsum("bop,bcp->oc", gz, xf))
    return dx.reshape(B, C, H, W), dcs, torch.cat(dws, 1).reshape(weight.shape), gz.sum((0, 2))


def upsample_ac_backward(grad_out, in_size):
    """Backward of ``F.interpolate(mode="bilinear", align_corners=True)`` from ``grad_out [B,C,Ho,Wo]`` to
    ``[B,C,Hi,Wi]``: ``U_H^T grad U_W`` in float64."""
    Ho, Wo = grad_out.shape[2:]
    uy, ux = tap_matrix(Ho, in_size[0], True), tap_matrix(Wo, in_size[1], True)
    return torch.einsum("hi,bchw,wj->bcij", uy, grad_out.double(), ux)
