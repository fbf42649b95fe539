"""numpy restatement of the textured rasteriser (DESIGN.md §4.35, ``ffb6d_render_rgbd_textured``), bit for bit.

Everything but a drawn pixel's colour is oracle/render_oracle.py's (§4.31): the vertex stage, coverage, depth, the
visibility key, labels and empty pixels.  The colour, float64 with one rounding per operation, restated from the
header:

* ``u = ((p0 u0 + p1 u1) + p2 u2) / S`` and ``v`` likewise, from per-vertex float32 UVs (``v = 0`` the bottom row of
  the texture as decoded).
* Screen derivatives per pixel: for the edge ``(a, b) = (V[k+1], V[k+2])`` of ``w_k``, ``gx_k = -256 sgn (b.y - a.y)``
  and ``gy_k = 256 sgn (b.x - a.x)`` (exact integers); ``u_x = (((gx_0 iz_0)(u_0 - u) + (gx_1 iz_1)(u_1 - u)) +
  (gx_2 iz_2)(u_2 - u)) / S``, and ``u_y``, ``v_x``, ``v_y`` likewise.
* ``rho = max(sqrt((u_x Tw)^2 + (v_x Th)^2), sqrt((u_y Tw)^2 + (v_y Th)^2))`` with ``max(a, b) = b if b > a else a``.
  ``not rho > 1``: level 0; ``rho >= 2^(L-1)``: level ``L - 1``; otherwise ``e = floor(log2 rho)`` from the exponent,
  ``t = rho 2^-e - 1`` and ``c = (1 - t) c_e + t c_(e+1)``.
* Bilinear at level ``l`` (``W_l x H_l``): ``x = u W_l - 0.5``, ``y = (1 - v) H_l - 0.5``, ``x0 = floor(x)``,
  ``fx = x - x0`` (and y), REPEAT wrapping, weights ``w00 = (1 - fx)(1 - fy)``, ``w10 = fx (1 - fy)``,
  ``w01 = (1 - fx) fy``, ``w11 = fx fy``, ``c = ((w00 t00 + w10 t10) + w01 t01) + w11 t11``.
* The channel written is ``clamp(floor(c + 0.5), 0, 255)``.
* Mip chain: level ``l + 1`` is ``max(1, n >> 1)`` per side; texel ``(i, j)`` is ``(a + b + c + d + 2) >> 2`` of level
  ``l``'s ``(2i, 2j)``, ``(2i+1, 2j)``, ``(2i, 2j+1)``, ``(2i+1, 2j+1)``, indices clamped to its edge; down to 1 x 1.
"""
import numpy as np

from oracle.render_oracle import EMPTY, _E, _weights, face_pixels, vertex_stage


def mip_chain(texture):
    """``texture [Th,Tw,3]`` uint8 -> the list of its levels, level 0 first, down to 1 x 1 (uint8)."""
    lv = [np.asarray(texture, np.uint8)]
    while lv[-1].shape[0] > 1 or lv[-1].shape[1] > 1:
        s = lv[-1].astype(np.int32)
        h, w = s.shape[:2]
        hd, wd = max(1, h >> 1), max(1, w >> 1)
        ya = np.minimum(2 * np.arange(hd), h - 1)
        yb = np.minimum(2 * np.arange(hd) + 1, h - 1)
        xa = np.minimum(2 * np.arange(wd), w - 1)
        xb = np.minimum(2 * np.arange(wd) + 1, w - 1)
        q = s[ya][:, xa] + s[ya][:, xb] + s[yb][:, xa] + s[yb][:, xb]
        lv.append(((q + 2) >> 2).astype(np.uint8))
    return lv


def bilinear(level, u, v):
    """The unrounded bilinear sample ``[n,3]`` float64 of one level at float64 ``u``, ``v`` ``[n]``."""
    Hl, Wl = level.shape[:2]
    x = u * np.float64(Wl) - 0.5
    y = (1.0 - v) * np.float64(Hl) - 0.5
    xf, yf = np.floor(x), np.floor(y)
    fx, fy = x - xf, y - yf
    gx, gy = 1.0 - fx, 1.0 - fy
    w00, w10, w01, w11 = gx * gy, fx * gy, gx * fy, fx * fy
    x0, y0 = xf.astype(np.int64), yf.astype(np.int64)
    x1, y1 = (x0 + 1) % Wl, (y0 + 1) % Hl           # numpy's % of a positive modulus is never negative: REPEAT
    x0, y0 = x0 % Wl, y0 % Hl
    t = level.astype(np.float64)
    return ((w00[:, None] * t[y0, x0] + w10[:, None] * t[y0, x1]) + w01[:, None] * t[y1, x0]) + w11[:, None] * t[y1, x1]


def lod(ux, uy, vx, vy, Th, Tw):
    """``rho`` of each pixel, and ``(l_a, l_b, t, blend)``: the level(s) and weight the header's rule picks."""
    fw, fh = np.float64(Tw), np.float64(Th)
    ax, bx, ay, by = ux * fw, vx * fh, uy * fw, vy * fh
    r1 = np.sqrt(ax * ax + bx * bx)
    r2 = np.sqrt(ay * ay + by * by)
    rho = np.where(r2 > r1, r2, r1)
    L = max(int(Th), int(Tw)).bit_length()
    with np.errstate(invalid="ignore"):
        blend = (rho > 1.0) & (rho < np.float64(2 ** (L - 1)))
        top = (rho > 1.0) & ~blend
    e = np.where(blend, np.frexp(np.where(blend, rho, 2.0))[1] - 1, 0)
    t = np.where(blend, np.ldexp(np.where(blend, rho, 2.0), -e) - 1.0, 0.0)
    la = np.where(top, L - 1, e)
    return rho, la, la + 1, t, blend


def attributes(uv, fa, x, y, iz, w):
    """``(u, v, u_x, u_y, v_x, v_y)`` ``[n]`` float64 of ``n`` covered pixels: face vertex indices ``fa [n,3]``, their
    fixed-point ``x``, ``y`` ``[n,3]`` int64 and ``iz [n,3]``, sign-normalised edge values ``w [3,n]``; ``uv [V,2]``
    float32."""
    sgn = np.sign(_E(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2]))
    p, S = _weights(w, iz.T)
    uvf = np.asarray(uv, np.float32).astype(np.float64)[fa]          # [n, vertex, 2]
    uk, vk = uvf[:, :, 0], uvf[:, :, 1]
    u = ((p[0] * uk[:, 0] + p[1] * uk[:, 1]) + p[2] * uk[:, 2]) / S
    v = ((p[0] * vk[:, 0] + p[1] * vk[:, 1]) + p[2] * vk[:, 2]) / S
    sx, sy = [], []
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        sx.append((-256 * sgn * (y[:, b] - y[:, a])).astype(np.float64) * iz[:, k])
        sy.append((256 * sgn * (x[:, b] - x[:, a])).astype(np.float64) * iz[:, k])

    def d(s, ck, c):
        return ((s[0] * (ck[:, 0] - c) + s[1] * (ck[:, 1] - c)) + s[2] * (ck[:, 2] - c)) / S

    return u, v, d(sx, uk, u), d(sy, uk, u), d(sx, vk, v), d(sy, vk, v)


def shade(levels, uv, fa, x, y, iz, w):
    """The colours ``[n,3]`` uint8 of ``n`` covered pixels (arguments as :func:`attributes`) from a mip chain."""
    u, v, ux, uy, vx, vy = attributes(uv, fa, x, y, iz, w)
    Th, Tw = levels[0].shape[:2]
    _, la, lb, t, blend = lod(ux, uy, vx, vy, Th, Tw)
    c = np.zeros((len(u), 3))
    for l in np.unique(la):
        sel = la == l
        c[sel] = bilinear(levels[l], u[sel], v[sel])
    for l in np.unique(lb[blend]):
        sel = blend & (lb == l)
        c[sel] = (1.0 - t[sel])[:, None] * c[sel] + t[sel][:, None] * bilinear(levels[l], u[sel], v[sel])
    return np.clip(np.floor(c + 0.5), 0.0, 255.0).astype(np.uint8)


def render_frame(meshes, mesh_idx, RTs, label, K, H, W, z_near=0.01, levels=None):
    """One frame: ``meshes`` a list of ``(xyz [V,3], faces [F,3], uv [V,2], texture [Th,Tw,3] uint8)``; ``mesh_idx
    [M]``, ``RTs [M,3,4]``, ``label [M]``; ``K`` ``(fx, fy, cx, cy)``; ``levels`` each mesh's :func:`mip_chain`
    (None: built here).  Returns ``(depth [H,W] float32, rgb [H,W,3] uint8, labels [H,W] uint8)``."""
    if levels is None:
        levels = [mip_chain(m[3]) for m in meshes]
    max_faces = max(len(m[1]) for m in meshes)
    keys = np.full(H * W, EMPTY, np.uint64)
    setups = {}
    for s, m in enumerate(np.asarray(mesh_idx).reshape(-1)):          # §4.31's visibility, as render_oracle's
        if not 0 <= m < len(meshes):
            continue
        U, V, iz, ok = vertex_stage(meshes[m][0], RTs[s], K, z_near)
        setups[s] = (U, V, iz)
        for f, face in enumerate(np.asarray(meshes[m][1], np.int64)):
            if not ok[face].all():
                continue
            r = face_pixels(U, V, face, H, W)
            if r is None:
                continue
            ii, jj, w, A = r
            _, S = _weights(w, iz[face])
            dd = (np.float64(A) / S).astype(np.float32)
            key = (dd.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(s * max_faces + f)
            np.minimum.at(keys, jj * W + ii, key)
    depth = np.zeros(H * W, np.float32)
    rgb = np.zeros((H * W, 3), np.uint8)
    labels = np.zeros(H * W, np.uint8)
    pix = np.nonzero(keys != EMPTY)[0]
    k = keys[pix]
    depth[pix] = (k >> np.uint64(32)).astype(np.uint32).view(np.float32)
    slot, face_i = np.divmod((k & np.uint64(0xFFFFFFFF)).astype(np.int64), max_faces)
    rows, cols = np.divmod(pix.astype(np.int64), W)
    idx = np.asarray(mesh_idx).reshape(-1)
    for s in np.unique(slot):
        sel = slot == s
        m = int(idx[s])
        U, V, iz = setups[int(s)]
        fa = np.asarray(meshes[m][1], np.int64)[face_i[sel]]
        x, y = U[fa], V[fa]
        sgn = np.sign(_E(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2]))
        px, py = 256 * cols[sel], 256 * rows[sel]
        w = np.stack([sgn * _E(x[:, (q + 1) % 3], y[:, (q + 1) % 3], x[:, (q + 2) % 3], y[:, (q + 2) % 3], px, py)
                      for q in range(3)])
        rgb[pix[sel]] = shade(levels[m], meshes[m][2], fa, x, y, iz[fa], w)
        labels[pix[sel]] = np.uint8(np.asarray(label).reshape(-1)[s])
    return depth.reshape(H, W), rgb.reshape(H, W, 3), labels.reshape(H, W)


def render(meshes, mesh_idx, RTs, label, K, H, W, z_near=0.01, active=None):
    """A batch, as ``render_oracle.render``: ``mesh_idx [B,M]``, ``RTs [B,M,3,4]``, ``label [B,M]``, ``K`` ``[4]`` or
    ``[B,4]``, ``active [B]`` (None: every frame); inactive frames come back as zeros."""
    levels = [mip_chain(m[3]) for m in meshes]
    mesh_idx = np.asarray(mesh_idx)
    B = mesh_idx.shape[0]
    K = np.asarray(K, np.float64)
    depth = np.zeros((B, H, W), np.float32)
    rgb = np.zeros((B, H, W, 3), np.uint8)
    labels = np.zeros((B, H, W), np.uint8)
    for b in range(B):
        if active is not None and not active[b]:
            continue
        depth[b], rgb[b], labels[b] = render_frame(meshes, mesh_idx[b], np.asarray(RTs)[b], np.asarray(label)[b],
                                                   K[b] if K.ndim == 2 else K, H, W, z_near, levels)
    return depth, rgb, labels
