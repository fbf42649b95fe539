"""Images of the ORB fixture (tests/golden/orb_cases.npz), regenerated from (kind, seed, H, W), and the ape renders.

Kinds: 0 uniform noise; 1 blurred noise (few, strong corners); 2 a repeated 8x8 tile of one bright pixel (FAST and Harris ties at
both cuts); 3 dense random rectangles (the level-0 cut binds); 4 a single bright square on black; 5 black.
"""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = ([(0, s, 480, 640) for s in range(3)] + [(1, s, 240, 320) for s in range(3)] +
         [(2, s, 200, 260) for s in range(2)] + [(3, s, 480, 640) for s in range(3)] +
         [(0, 10 + s, h, w) for s, (h, w) in enumerate([(65, 70), (97, 131), (141, 391), (391, 141), (33, 500)])] +
         [(4, 0, 120, 160), (5, 0, 100, 100), (2, 5, 77, 179), (1, 7, 301, 167)])
APE_VIEWS = (0, 4, 8)


def image(kind, seed, H, W):
    """The RGB uint8 [H,W,3] image of a case."""
    rng = np.random.default_rng(seed)
    if kind == 0:
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if kind == 1:
        x = rng.integers(0, 256, (H // 4 + 2, W // 4 + 2, 3)).astype(np.float64)
        x = np.repeat(np.repeat(x, 4, 0), 4, 1)[:H, :W]
        k = np.ones(5) / 5
        for ax in (0, 1):
            x = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), ax, x)
        return np.clip(x, 0, 255).astype(np.uint8)
    if kind == 2:
        tile = np.full((8, 8), 20, np.uint8)
        tile[3, 3] = 250
        g = np.tile(tile, (H // 8 + 1, W // 8 + 1))[:H, :W]
        return np.repeat(g[..., None], 3, 2)
    if kind == 3:
        x = np.zeros((H, W, 3), np.uint8)
        for _ in range(4000):
            y0, x0 = rng.integers(0, H), rng.integers(0, W)
            x[y0:y0 + rng.integers(2, 12), x0:x0 + rng.integers(2, 12)] = rng.integers(0, 256, 3)
        return x
    if kind == 4:
        x = np.zeros((H, W, 3), np.uint8)
        x[H // 2 - 20:H // 2 + 20, W // 2 - 20:W // 2 + 20] = 255
        return x
    return np.zeros((H, W, 3), np.uint8)


def ape_setup():
    """The ape (render_ape.npz) in metres, the tool's camera and its box radius as the tool computes it (float32)."""
    d = np.load(os.path.join(HERE, "golden", "render_ape.npz"))
    xyz = d["xyz"] / 1000.0
    from ffb6d_b200.objinfo import get_3D_bbox, get_r, TOOL_K, TOOL_H, TOOL_W
    return xyz, TOOL_K, TOOL_H, TOOL_W, get_r(get_3D_bbox(xyz))


def ape_mesh():
    d = np.load(os.path.join(HERE, "golden", "render_ape.npz"))
    return d["xyz"] / 1000.0, d["faces"], d["rgb"]


def ape_render(RT, H=480, W=640):
    """``(depth float32 [H,W], rgb uint8 [H,W,3])`` of the ape at ``RT`` (float64 [4,4]; rendered with its float32
    rounding, as the device path does) by oracle/render_oracle.py."""
    from oracle import render_oracle
    K = np.array([700.0, 700.0, 320.0, 240.0])
    depth, rgb, _ = render_oracle.render_frame([ape_mesh()], [0], RT[None, :3, :].astype(np.float32), [1], K, H, W)
    return depth, rgb
