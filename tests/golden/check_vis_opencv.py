#!/usr/bin/env python
"""Check the circle restatement of oracle/vis_oracle.py against ``cv2.circle(img, (x, y), r, colour, -1)``.

A build-machine script (needs cv2; not a test).  For every radius 0 .. 64 (``FFB6D_VIS_MAX_RADIUS``) and every
clipping offset against all four borders -- centres up to ``r + 2`` pixels inside each border and on ``x = W`` and
``y = H``, every centre the reference's ``draw_p2ds`` passes on after clipping to ``[0,W] x [0,H]`` -- the
restatement's pixels equal OpenCV's on a 3-channel uint8 image.  The image is larger than the circle so that each
border is met alone, and a corner case meets two at once.

Run:  python tests/golden/check_vis_opencv.py      (exit status 1 on any mismatch)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import vis_oracle as O                                  # noqa: E402


def main():
    import cv2
    bad = checked = 0
    for r in range(0, 65):
        H, W = 2 * r + 11, 2 * r + 17
        offs = range(-r - 2, r + 3)
        centres = [(W // 2, H // 2)]
        centres += [(o, H // 2) for o in offs] + [(W - 1 - o, H // 2) for o in offs] + [(W, H // 2)]
        centres += [(W // 2, o) for o in offs] + [(W // 2, H - 1 - o) for o in offs] + [(W // 2, H)]
        centres += [(o, o) for o in offs] + [(W - 1 - o, H - 1 - o) for o in offs] + [(W, H), (0, H), (W, 0)]
        for cx, cy in centres:
            if not (0 <= cx <= W and 0 <= cy <= H):      # draw_p2ds clips every centre into [0,W] x [0,H] first
                continue
            want = np.zeros((H, W, 3), np.uint8)
            cv2.circle(want, (int(cx), int(cy)), r, (255, 128, 7), -1)
            got = np.zeros((H, W, 3), np.uint8)
            O.draw_sets(got[None], [(0, np.array([[cx, cy]]), r, (255, 128, 7))])
            checked += 1
            if not np.array_equal(got, want):
                bad += 1
                if bad <= 10:
                    print("mismatch: r = %d, centre (%d, %d) on %d x %d" % (r, cx, cy, H, W))
    print("%d circles checked, %d mismatches" % (checked, bad))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
