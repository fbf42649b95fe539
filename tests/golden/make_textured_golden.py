#!/usr/bin/env python
"""Generate tests/golden/textured_box.npz: the reference's example textured object,
``utils/dataset_tools/example_mesh/003_cracker_box`` (YCB's cracker box), for the textured rasteriser and the
pyrender-branch keypoint tests (DESIGN.md §4.35).

Stored: ``points [2621,3]`` float32, the object's ``points.xyz`` as ``np.loadtxt(..., dtype=np.float32)`` reads it
(metres; the ``points`` of ``gen_obj_info``), and ``texture [512,512,3]`` uint8 RGB, its 4096 x 4096
``texture_map.png`` reduced with ``cv2.resize(..., interpolation=cv2.INTER_AREA)``.  The object's ``textured.obj`` is
not in the reference's tree, so the tests build a cuboid on the points' bounding box (tests/textured_cases.py).

Run:  python tests/golden/make_textured_golden.py <reference>/ffb6d/utils/dataset_tools/example_mesh/003_cracker_box
      (rewrites textured_box.npz)
"""
import os
import sys

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "textured_box.npz")
SIDE = 512


def main():
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    import cv2
    points = np.loadtxt(os.path.join(sys.argv[1], "points.xyz"), dtype=np.float32)
    bgr = cv2.imread(os.path.join(sys.argv[1], "texture_map.png"), cv2.IMREAD_COLOR)
    small = cv2.resize(bgr, (SIDE, SIDE), interpolation=cv2.INTER_AREA)
    texture = np.ascontiguousarray(small[:, :, ::-1])
    np.savez_compressed(OUT, points=points, texture=texture)
    print("wrote %s: %d points, texture %s" % (OUT, len(points), texture.shape))


if __name__ == "__main__":
    main()
