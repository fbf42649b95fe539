"""Textured meshes for the §4.35 tests: the example cracker box (tests/golden/textured_box.npz), seeded textures and
screen-aligned quads."""
import os

import numpy as np

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "textured_box.npz"))


def cuboid(lo, hi, texture, n=8):
    """A box from corner ``lo`` to ``hi``: each of its six sides an ``n x n`` grid of quads (two faces each), its own
    vertices (the seams split, as trimesh splits them), and UVs mapping side ``k`` onto cell ``(k mod 3, k // 3)`` of a
    3 x 2 atlas of ``texture``.  Returns ``(xyz [V,3] float32, faces [F,3] int32, uv [V,2] float32, texture)``."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    g = np.linspace(0.0, 1.0, n + 1)
    s, t = np.meshgrid(g, g, indexing="xy")                     # [n+1, n+1]: s along columns, t along rows
    xyz, uv, faces = [], [], []
    side = 0
    for axis in range(3):
        b, c = [a for a in range(3) if a != axis]
        for end in (lo[axis], hi[axis]):
            p = np.zeros(s.shape + (3,))
            p[..., axis] = end
            p[..., b] = lo[b] + s * (hi[b] - lo[b])
            p[..., c] = lo[c] + t * (hi[c] - lo[c])
            base = side * (n + 1) ** 2
            xyz.append(p.reshape(-1, 3))
            uv.append(np.stack([(side % 3 + s) / 3.0, (side // 3 + t) / 2.0], -1).reshape(-1, 2))
            for r in range(n):
                for q in range(n):
                    v0 = base + r * (n + 1) + q
                    faces += [(v0, v0 + 1, v0 + n + 2), (v0, v0 + n + 2, v0 + n + 1)]
            side += 1
    return (np.concatenate(xyz).astype(np.float32), np.asarray(faces, np.int32), np.concatenate(uv).astype(np.float32),
            np.asarray(texture, np.uint8))


def box_mesh(n=8):
    """The cracker box: the cuboid on its points' bounding box, textured with its texture map (512 x 512)."""
    p = GOLDEN["points"]
    return cuboid(p.min(0), p.max(0), GOLDEN["texture"], n)


def noise_texture(side, seed):
    return np.random.default_rng(seed).integers(0, 256, (side, side, 3), dtype=np.uint8)


def checker_texture(side, cell):
    i = np.arange(side) // cell
    c = ((i[:, None] + i[None, :]) % 2).astype(np.uint8)
    return np.stack([c * 255, (1 - c) * 200 + 20, np.full_like(c, 90)], -1)


def screen_quad(W, H, x0=-0.5, y0=-0.5, x1=None, y1=None, uv0=(0.0, 0.0), uv1=(1.0, 1.0)):
    """Two faces at Z = 1 spanning pixel coordinates ``(x0, y0)`` to ``(x1, y1)`` (default ``(W - 0.5, H - 0.5)``)
    under the camera ``(1, 1, 0, 0)``, so a vertex's pixel position is its ``(X, Y)``.  UVs run from ``uv0`` at the
    bottom-left to ``uv1`` at the top-right: image row 0 (the top) is ``v = uv1[1]``.  ``(xyz, faces, uv)``."""
    x1 = W - 0.5 if x1 is None else x1
    y1 = H - 0.5 if y1 is None else y1
    xyz = np.array([[x0, y0, 1], [x1, y0, 1], [x1, y1, 1], [x0, y1, 1]], np.float32)
    uv = np.array([[uv0[0], uv1[1]], [uv1[0], uv1[1]], [uv1[0], uv0[1]], [uv0[0], uv0[1]]], np.float32)
    return xyz, np.array([[0, 1, 2], [0, 2, 3]], np.int32), uv


IDENTITY = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
UNIT_K = (1.0, 1.0, 0.0, 0.0)
