"""Images of the SIFT fixture (tests/golden/sift_cases.npz), regenerated from (kind, seed, H, W), and the ape views.

Kinds 0-5 are tests/orb_cases.py's (noise, blurred noise, a repeated tile of ties, random rectangles, one square,
black); kind 6 is filled circles of random grey levels on a grey background, the blob-like structure SIFT responds
to, with orientation ties on the round edges.
"""
import numpy as np

import orb_cases as OC

CASES = ([(6, s, 120, 160) for s in range(3)] + [(6, 3, 480, 640), (1, 0, 240, 320), (0, 0, 64, 80),
                                                  (3, 0, 120, 160)] +
         [(4, 0, 120, 160), (5, 0, 100, 100), (2, 5, 77, 179), (1, 7, 301, 167), (6, 4, 97, 131), (6, 5, 33, 251),
          (0, 11, 9, 13), (6, 6, 4, 4)])
APE_VIEWS = (0, 4, 8)


def image(kind, seed, H, W):
    """The RGB uint8 [H,W,3] image of a case."""
    if kind != 6:
        return OC.image(kind, seed, H, W)
    rng = np.random.default_rng(seed)
    g = np.full((H, W), 90, np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    for _ in range(max(H * W // 320, 1)):
        cy, cx = rng.uniform(0, H), rng.uniform(0, W)
        r = rng.uniform(2, max(3, min(H, W) / 6))
        g[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = rng.integers(0, 256)
    return np.repeat(g[..., None], 3, 2)
