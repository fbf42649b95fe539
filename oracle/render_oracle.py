"""numpy restatement of the z-buffer rasteriser (DESIGN.md §4.31, ``ffb6d_render_rgbd``), bit for bit.

raster_triangle, the renderer the reference's LineMOD `render` pickles come from, is not in the reference's tree, so
this is a specified rasteriser with its own oracle, not a copy of that one.  The specification, restated here:

* Per frame, ``M`` slots: a mesh index (-1, or any index outside the table: the slot draws nothing), a float32 pose
  ``RT [3,4]`` (object to camera, metres) and a uint8 label.  Camera ``(fx, fy, cx, cy)`` float64; ``z_near >= 0.001``.
* Vertex stage, float64, one rounding per operation: ``X = ((r0 x + r1 y) + r2 z) + t`` per row; culled when
  ``not Z >= z_near`` or ``Z`` is not finite (only non-finite poses or vertices make it so); ``u = fx (X / Z) + cx``,
  ``v = fy (Y / Z) + cy``; culled when ``not (|u| <= 2^14 and |v| <= 2^14)`` (the guard band); ``U = rint(256 u)``,
  ``V = rint(256 v)`` (ties to even) as integers.  A face with a culled vertex is not drawn: culled, not clipped.
* Coverage, exact integers.  Pixel (column i, row j) samples ``P = (256 i, 256 j)`` (``dpt_2_pcld``'s pixel
  coordinates, no +0.5).  ``E(a, b, P) = (b.x - a.x)(P.y - a.y) - (b.y - a.y)(P.x - a.x)``; ``w0 = E(V1, V2, P)``,
  ``w1 = E(V2, V0, P)``, ``w2 = E(V0, V1, P)``, ``A = E(V0, V1, V2)``.  ``A == 0``: not drawn.  ``A < 0``: ``A`` and
  every ``w`` negated (no back-face culling).  Covered when every ``w_k > 0``, or ``w_k == 0`` on an owned edge:
  with ``(dx, dy) = sign(A) (b - a)`` of the edge's ``E(a, b, .)``, owned is ``dy < 0 or (dy == 0 and dx > 0)`` --
  the top-left rule, so of two faces sharing an edge exactly one draws a pixel on it.
* Depth and colour, float64, one rounding per operation: ``p_k = w_k (1 / Z_k)``, ``S = (p0 + p1) + p2``,
  ``depth = fl32(A / S)``; each colour channel ``clamp(floor((((p0 c0 + p1 c1) + p2 c2) / S) + 0.5), 0, 255)`` of the
  vertices' ``(red, green, blue)``.
* Visibility: the least key ``bits(depth) << 32 | (slot max_faces + face)`` wins: the nearest depth, a tie the lower
  ``(slot, face)``.  Empty pixels are 0 in depth, colour and label.
* ``dpt_mm = min(trunc(fl32(depth * 1000.0f)), 65535)`` as uint16: LineMOD's ``data['depth'] * 1000.`` (float32 times a
  Python float stays float32) and ``.astype(np.uint16)``.
"""
import numpy as np

GUARD_BAND = 1 << 14
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def vertex_stage(xyz, RT, K, z_near=0.01):
    """``xyz [V,3]`` float32, ``RT [3,4]`` float32, ``K = (fx, fy, cx, cy)`` -> ``(U, V)`` int64, ``1/Z`` float64 and
    a bool ``ok`` (not culled) per vertex."""
    p = np.asarray(xyz, np.float32).astype(np.float64)
    R = np.asarray(RT, np.float32).astype(np.float64)
    fx, fy, cx, cy = (np.float64(k) for k in K)
    with np.errstate(all="ignore"):                  # non-finite inputs are culled below
        c = [((R[r, 0] * p[:, 0] + R[r, 1] * p[:, 1]) + R[r, 2] * p[:, 2]) + R[r, 3] for r in range(3)]
        ok = (c[2] >= z_near) & np.isfinite(c[2])
        Z = np.where(ok, c[2], 1.0)
        u = fx * (c[0] / Z) + cx
        v = fy * (c[1] / Z) + cy
        ok &= (np.abs(u) <= GUARD_BAND) & (np.abs(v) <= GUARD_BAND)
        U = np.where(ok, np.rint(np.where(ok, u, 0.0) * 256.0), 0).astype(np.int64)
        V = np.where(ok, np.rint(np.where(ok, v, 0.0) * 256.0), 0).astype(np.int64)
        iz = np.where(ok, 1.0 / Z, 0.0)
    return U, V, iz, ok


def _E(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def face_pixels(U, V, face, H, W):
    """The pixels face ``face`` (three vertex indices) covers: ``(cols, rows, w [3,n] int64, A)``, ``w`` and ``A``
    sign-normalised; None when it draws nothing (a zero area, an empty box).  Culling is the caller's."""
    x = [int(U[k]) for k in face]
    y = [int(V[k]) for k in face]
    A = _E(x[0], y[0], x[1], y[1], x[2], y[2])
    if A == 0:
        return None
    sgn = 1 if A > 0 else -1
    i0, i1 = max(-((-min(x)) >> 8), 0), min(max(x) >> 8, W - 1)
    j0, j1 = max(-((-min(y)) >> 8), 0), min(max(y) >> 8, H - 1)
    if i0 > i1 or j0 > j1:
        return None
    jj, ii = np.mgrid[j0:j1 + 1, i0:i1 + 1]
    px, py = (ii.ravel() * 256).astype(np.int64), (jj.ravel() * 256).astype(np.int64)
    inside = np.ones(px.shape, bool)
    w = []
    for k in range(3):
        p, q = (k + 1) % 3, (k + 2) % 3
        wk = sgn * _E(x[p], y[p], x[q], y[q], px, py)
        dx, dy = sgn * (x[q] - x[p]), sgn * (y[q] - y[p])
        owned = dy < 0 or (dy == 0 and dx > 0)
        inside &= (wk > 0) | ((wk == 0) & owned)
        w.append(wk)
    w = np.stack(w)[:, inside]
    return ii.ravel()[inside], jj.ravel()[inside], w, sgn * A


def _weights(w, iz):
    p = [w[k].astype(np.float64) * iz[k] for k in range(3)]
    return p, (p[0] + p[1]) + p[2]


def render_frame(meshes, mesh_idx, RTs, label, K, H, W, z_near=0.01, coverage=False):
    """One frame: ``meshes`` a list of ``(xyz [V,3], faces [F,3], rgb [V,3] uint8)``; ``mesh_idx [M]``, ``RTs [M,3,4]``,
    ``label [M]``; ``K`` ``(fx, fy, cx, cy)``.  Returns ``(depth [H,W] float32, rgb [H,W,3] uint8, labels [H,W]
    uint8)``, and with ``coverage`` also ``[H,W]`` int64: how many faces cover each pixel."""
    max_faces = max(len(m[1]) for m in meshes)
    keys = np.full(H * W, EMPTY, np.uint64)
    count = np.zeros(H * W, np.int64)
    setups = {}
    for s, m in enumerate(np.asarray(mesh_idx).reshape(-1)):
        if not 0 <= m < len(meshes):
            continue
        xyz, faces, _ = meshes[m]
        U, V, iz, ok = vertex_stage(xyz, RTs[s], K, z_near)
        setups[s] = (U, V, iz)
        for f, face in enumerate(np.asarray(faces, np.int64)):
            if not ok[face].all():
                continue
            r = face_pixels(U, V, face, H, W)
            if r is None:
                continue
            ii, jj, w, A = r
            _, S = _weights(w, iz[face])
            d = (np.float64(A) / S).astype(np.float32)
            key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(s * max_faces + f)
            pix = jj * W + ii
            np.minimum.at(keys, pix, key)
            np.add.at(count, pix, 1)
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
        _, faces, vrgb = meshes[int(idx[s])]
        U, V, iz = setups[int(s)]
        fa = np.asarray(faces, np.int64)[face_i[sel]]
        x, y = U[fa], V[fa]
        sgn = np.sign(_E(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2]))
        px, py = 256 * cols[sel], 256 * rows[sel]
        w = np.stack([sgn * _E(x[:, (q + 1) % 3], y[:, (q + 1) % 3], x[:, (q + 2) % 3], y[:, (q + 2) % 3], px, py)
                      for q in range(3)])
        p, S = _weights(w, iz[fa].T)
        c = np.asarray(vrgb, np.uint8)[fa].astype(np.float64)          # [n, vertex, channel]
        for ch in range(3):
            n = (p[0] * c[:, 0, ch] + p[1] * c[:, 1, ch]) + p[2] * c[:, 2, ch]
            rgb[pix[sel], ch] = np.clip(np.floor(n / S + 0.5), 0.0, 255.0).astype(np.uint8)
        labels[pix[sel]] = np.uint8(np.asarray(label).reshape(-1)[s])
    out = (depth.reshape(H, W), rgb.reshape(H, W, 3), labels.reshape(H, W))
    return out + (count.reshape(H, W),) if coverage else out


def render(meshes, mesh_idx, RTs, label, K, H, W, z_near=0.01, active=None):
    """A batch: ``mesh_idx [B,M]``, ``RTs [B,M,3,4]``, ``label [B,M]``, ``K`` ``(fx, fy, cx, cy)`` ``[4]`` or
    ``[B,4]``; ``active [B]`` (None: every frame).  Inactive frames come back as zeros (the kernel leaves them
    untouched)."""
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
                                                   K[b] if K.ndim == 2 else K, H, W, z_near)
    return depth, rgb, labels


def dpt_mm(depth):
    """LineMOD's millimetre map of a render's depth: ``(depth * 1000.).astype(np.uint16)`` of a float32 map (float32
    arithmetic), saturating above 65535."""
    mm = np.asarray(depth, np.float32) * np.float32(1000.0)
    return np.minimum(np.trunc(mm), 65535).astype(np.uint16)
