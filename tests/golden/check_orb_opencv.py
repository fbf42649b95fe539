#!/usr/bin/env python
"""Check oracle/orb_oracle.py against OpenCV beyond the cases of orb_cases.npz.

A build-machine script (needs cv2; the result belongs to the OpenCV it runs with, so it is not a test).  It checks:
  * ``resize_exact`` against ``cv2.resize(..., INTER_LINEAR_EXACT)`` for 600 random size pairs from 1 to 700 pixels
    on a side, and for size pairs whose source coordinates fall on exact half weights (src / dst = k / 512);
  * ``fast_scores`` + ``nms`` against ``cv2.FastFeatureDetector_create(20, True)`` (points and scores);
  * ``detect`` against ``cv2.ORB_create().detect`` as sets of (octave, pt, response) bit for bit, on random noise,
    blurred noise, repeated tiles (ties at both cuts), dense rectangles (the level-0 cut binds), small images whose
    upper levels vanish, and ape renders from the tool's sphere of views.

Run:  python tests/golden/check_orb_opencv.py      (exit status 1 on any mismatch)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import orb_oracle as O                                   # noqa: E402
import orb_cases as OC                                               # noqa: E402


def keyset(octave, pt, response):
    pt = np.asarray(pt, np.float32).reshape(-1, 2)
    return set(zip(np.asarray(octave).astype(int).tolist(), pt[:, 0].view(np.uint32).tolist(),
                   pt[:, 1].view(np.uint32).tolist(), np.asarray(response, np.float32).view(np.uint32).tolist()))


def check_resize(cv2, rng):
    sizes = [tuple(rng.integers(1, 701, 4)) for _ in range(600)]
    sizes += [(h, 512, 3, k) for k in (1, 3, 255, 256, 257, 511, 513, 700) for h in (5, 129)]   # w = 512 -> k
    sizes += [(512, w, k, 7) for k in (1, 3, 255, 257, 511) for w in (9, 64)]
    bad = 0
    for h, w, dh, dw in sizes:
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        if not np.array_equal(cv2.resize(img, (int(dw), int(dh)), interpolation=cv2.INTER_LINEAR_EXACT),
                              O.resize_exact(img, dw, dh)):
            bad += 1
    print("resize: %d size pairs, %d differ" % (len(sizes), bad))
    return bad


def check_fast(cv2, rng):
    bad = 0
    for i in range(200):
        h, w = rng.integers(7, 200, 2)
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        if i % 2:
            img = (img // 64 * 64).astype(np.uint8)
        want = sorted((int(k.pt[1]), int(k.pt[0]), int(k.response))
                      for k in cv2.FastFeatureDetector_create(20, True).detect(img))
        s = O.fast_scores(img)
        ys, xs = np.nonzero(O.nms(s))
        bad += want != sorted((int(y), int(x), int(s[y, x])) for y, x in zip(ys, xs))
    print("FAST + NMS: 200 images, %d differ" % bad)
    return bad


def images(rng):
    for s in range(80):
        yield "noise", OC.image(0, 1000 + s, *rng.integers(40, 700, 2))
    for s in range(60):
        yield "blurred", OC.image(1, 2000 + s, *rng.integers(64, 500, 2))
    for s in range(40):
        yield "tiles", OC.image(2, s, *rng.integers(64, 500, 2))
    for s in range(30):
        yield "rectangles", OC.image(3, 3000 + s, 480, 640)
    for s in range(60):
        yield "small", OC.image(0, 4000 + s, *rng.integers(2, 90, 2))
    xyz, K, H, W, radius = OC.ape_setup()
    from ffb6d_b200.objinfo import sphere_poses
    for n in (3, 4):
        for RT in sphere_poses(radius, n, n):
            yield "ape", OC.ape_render(RT)[1]


def check_detect(cv2, rng):
    orb = cv2.ORB_create()
    bad, n, per = 0, 0, {}
    for kind, img in images(rng):
        kps = orb.detect(np.ascontiguousarray(img[..., ::-1]), None)
        want = keyset([k.octave for k in kps], [k.pt for k in kps], [k.response for k in kps])
        d = O.detect(img)
        ok = want == keyset(d["octave"], d["pt"], d["response"])
        bad += not ok
        n += 1
        per.setdefault(kind, [0, 0])
        per[kind][0] += 1
        per[kind][1] += not ok
    for kind, (m, b) in per.items():
        print("ORB %-10s: %d images, %d differ" % (kind, m, b))
    return bad


def main():
    import cv2
    print("OpenCV", cv2.__version__)
    rng = np.random.default_rng(20261018)
    bad = check_resize(cv2, rng) + check_fast(cv2, rng) + check_detect(cv2, rng)
    print("mismatches:", bad)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
