"""numpy restatement of the depth-normal estimator (DESIGN.md §4.30, ``ffb6d_depth_normal``).

For pixel (y, x) of a millimetre depth map D with d = D[y,x] and r = k_size:

1. d == 0 or d >= distance_threshold gives (0, 0, 0).
2. Over the 8 offsets (dx, dy) in {-r, 0, r}^2 without (0, 0) whose pixel lies in the image, delta = D[y+dy,x+dx] - d;
   where |delta| < difference_threshold, in int64: A0 += dx dx, A1 += dx dy, A2 += dy dy, b0 += dx delta,
   b1 += dy delta.
3. det = A0 A2 - A1^2, ddx = A2 b0 - A1 b1, ddy = A0 b1 - A1 b0; det == 0 gives (0, 0, 0).
4. In float64: nx = fx ddx, ny = fy ddy, nz = -(det d), s = sqrt((nx nx + ny ny) + nz nz); the normal is
   (nx/s, ny/s, nz/s), each rounded once to float32, negated with point_into_surface.

This is the least-squares depth-gradient fit of OpenCV's LINEMOD (``accumBilateral``) with fx, fy for its fixed focal
length and without quantisation.  The kernel must equal it bit for bit.
"""
import numpy as np


def _frame(D, fx, fy, r, dist, diff, into):
    H, W = D.shape
    d = D.astype(np.int64)
    A0, A1, A2, b0, b1 = (np.zeros((H, W), np.int64) for _ in range(5))
    for dy in (-r, 0, r):
        for dx in (-r, 0, r):
            if (dx == 0 and dy == 0) or abs(dy) >= H or abs(dx) >= W:     # the offset leaves every pixel's image
                continue
            nb = np.zeros((H, W), np.int64)
            inside = np.zeros((H, W), bool)
            ys, yd = slice(max(dy, 0), H + min(dy, 0)), slice(max(-dy, 0), H + min(-dy, 0))
            xs, xd = slice(max(dx, 0), W + min(dx, 0)), slice(max(-dx, 0), W + min(-dx, 0))
            nb[yd, xd] = d[ys, xs]                 # nb[y, x] = d[y + dy, x + dx]
            inside[yd, xd] = True
            delta = nb - d
            acc = inside & (np.abs(delta) < diff)
            A0 += np.where(acc, dx * dx, 0)
            A1 += np.where(acc, dx * dy, 0)
            A2 += np.where(acc, dy * dy, 0)
            b0 += np.where(acc, dx * delta, 0)
            b1 += np.where(acc, dy * delta, 0)
    det = A0 * A2 - A1 * A1
    ddx = A2 * b0 - A1 * b1
    ddy = A0 * b1 - A1 * b0
    valid = (d != 0) & (d < dist) & (det != 0)
    nx = np.float64(fx) * ddx.astype(np.float64)
    ny = np.float64(fy) * ddy.astype(np.float64)
    nz = -(det * d).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.sqrt((nx * nx + ny * ny) + nz * nz)
        n = np.stack([nx / s, ny / s, nz / s], -1).astype(np.float32)
    if into:
        n = -n
    n[~valid] = 0.0
    return n


def depth_normal(dpt_mm, fx, fy, k_size=5, distance_threshold=2000, difference_threshold=20,
                 point_into_surface=False):
    """``dpt_mm`` uint16 ``[H,W]`` or ``[B,H,W]``; ``fx``, ``fy`` scalars or one per frame -> float32 ``[..,H,W,3]``."""
    D = np.asarray(dpt_mm)
    if D.dtype != np.uint16 or D.ndim not in (2, 3):
        raise ValueError("dpt_mm must be uint16 [H,W] or [B,H,W]")
    frames = D[None] if D.ndim == 2 else D
    B = frames.shape[0]
    fx = np.broadcast_to(np.asarray(fx, np.float64), (B,))
    fy = np.broadcast_to(np.asarray(fy, np.float64), (B,))
    out = np.stack([_frame(frames[b], fx[b], fy[b], int(k_size), int(distance_threshold), int(difference_threshold),
                           bool(point_into_surface)) for b in range(B)])
    return out[0] if D.ndim == 2 else out


def depth_normal_K(dpt_mm, K, **kw):
    """:func:`depth_normal` with camera matrices ``[3,3]`` or ``[B,3,3]``, as ``ops.depth_normal`` takes them."""
    K = np.asarray(K, np.float64)
    return depth_normal(dpt_mm, K[..., 0, 0], K[..., 1, 1], **kw)


def ycb_mm(dpt_um):
    """The YCB dataset's millimetre map of the completed depth: ``(dpt_um / 10).astype(np.uint16)``
    (datasets/ycb/ycb_dataset.py:207), a float32 division and a truncation."""
    return (np.asarray(dpt_um, np.float32) / np.float32(10)).astype(np.uint16)
