"""float64 restatement of PSPUpsample's x2 bilinear upsampling (``align_corners=True``) + 3x3 conv (padding 1) in both
orders, with explicit tap matrices (DESIGN.md §4.23):

    reference order      z = b + conv3x3(up(x))
    restructured order   z = b + sum_t S_t(up(W_t x)),   W_t = W[:, :, ky, kx], t = 3 ky + kx

``up`` is ``U_y X U_x^T`` per plane, ``S_t`` the shift to tap t on the upsampled grid, ``S_y X S_x^T`` with zero rows
where the shifted position leaves the grid.  The adjoints of both orders are restated the same way; the restructured
one is what the kernels compute: ``G_t = U_y^T S_y^T dz S_x U_x``, ``dW_t = sum_b G_t x^T``, ``dx = sum_t W_t^T G_t``.
"""
import numpy as np


def up_matrix(n_in, n_out):
    """``[n_out, n_in]``: bilinear interpolation along one axis with ``align_corners=True``."""
    scale = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
    m = np.zeros((n_out, n_in))
    for d in range(n_out):
        src = scale * d
        i0 = min(int(src), n_in - 1)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        l1 = src - i0
        m[d, i0] += 1.0 - l1
        m[d, i1] += l1
    return m


def shift_matrix(n, d):
    """``[n, n]``: ``(S v)[y] = v[y + d]``, 0 where ``y + d`` is outside ``[0, n)``."""
    s = np.zeros((n, n))
    for y in range(n):
        if 0 <= y + d < n:
            s[y, y + d] = 1.0
    return s


def _mats(Hi, Wi):
    Ho, Wo = 2 * Hi, 2 * Wi
    uy, ux = up_matrix(Hi, Ho), up_matrix(Wi, Wo)
    sy = [shift_matrix(Ho, k - 1) for k in range(3)]
    sx = [shift_matrix(Wo, k - 1) for k in range(3)]
    return uy, ux, sy, sx


def _plane(a, left, right):
    """``left . a . right^T`` on the last two axes."""
    return np.einsum("yi,...ij,xj->...yx", left, a, right)


def forward_reference(x, w, b):
    """``conv3x3(up(x)) + b``: x ``[B, Ci, Hi, Wi]``, w ``[Co, Ci, 3, 3]``, b ``[Co]``."""
    uy, ux, sy, sx = _mats(*x.shape[2:])
    u = _plane(x, uy, ux)
    z = np.zeros((x.shape[0], w.shape[0]) + u.shape[2:])
    for ky in range(3):
        for kx in range(3):
            z += np.einsum("oc,bcyx->boyx", w[:, :, ky, kx], _plane(u, sy[ky], sx[kx]))
    return z + b[None, :, None, None]


def forward_restructured(x, w, b):
    """``b + sum_t S_t(up(W_t x))``."""
    uy, ux, sy, sx = _mats(*x.shape[2:])
    z = 0.0
    for ky in range(3):
        for kx in range(3):
            t = np.einsum("oc,bcij->boij", w[:, :, ky, kx], x)
            z = z + _plane(_plane(t, uy, ux), sy[ky], sx[kx])
    return z + b[None, :, None, None]


def backward_reference(x, w, dz):
    """``(dx, dw, db)`` of :func:`forward_reference`: the conv's adjoint on the upsampled map, then ``up^T``."""
    uy, ux, sy, sx = _mats(*x.shape[2:])
    u = _plane(x, uy, ux)
    du = np.zeros(u.shape)
    dw = np.zeros(w.shape)
    for ky in range(3):
        for kx in range(3):
            du += np.einsum("oc,boyx->bcyx", w[:, :, ky, kx], _plane(dz, sy[ky].T, sx[kx].T))
            dw[:, :, ky, kx] = np.einsum("boyx,bcyx->oc", dz, _plane(u, sy[ky], sx[kx]))
    return _plane(du, uy.T, ux.T), dw, dz.sum(axis=(0, 2, 3))


def taps_adjoint(dz, Hi, Wi):
    """``G [B, 9, Co, Hi, Wi]``, ``G_t = U_y^T S_y^T dz S_x U_x``: the kernels' tap adjoint."""
    uy, ux, sy, sx = _mats(Hi, Wi)
    return np.stack([_plane(_plane(dz, sy[ky].T, sx[kx].T), uy.T, ux.T) for ky in range(3) for kx in range(3)], 1)


def backward_restructured(x, w, dz):
    """``(dx, dw, db)`` of :func:`forward_restructured` through :func:`taps_adjoint`."""
    g = taps_adjoint(dz, *x.shape[2:])
    dw = np.zeros(w.shape)
    dx = np.zeros(x.shape)
    for t in range(9):
        ky, kx = divmod(t, 3)
        dw[:, :, ky, kx] = np.einsum("boij,bcij->oc", g[:, t], x)
        dx += np.einsum("oc,boij->bcij", w[:, :, ky, kx], g[:, t])
    return dx, dw, dz.sum(axis=(0, 2, 3))
