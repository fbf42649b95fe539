#!/usr/bin/env python
"""Check the augmentation's restatements against OpenCV and the reference, beyond the cases of aug_cases.npz.

A build-machine script (needs cv2 and the reference's sources; the result depends on the CPU's OpenCV dispatch, so it
is not a test).  It checks:
  * ``aug_oracle.bgr2hsv`` on all 2^24 inputs and ``aug_oracle.hsv2bgr`` on all 180 x 256 x 256 inputs, each in
    OpenCV's vector loop and in the scalar tail of a row;
  * ``augment.motion_kernel`` against the kernel the reference's ``linear_motion_blur`` passes to ``cv2.filter2D``,
    for all 360 x 15 (angle, length) pairs the datasets draw;
  * ``augment.gaussian_taps`` against ``cv2.GaussianBlur``'s impulse response for 12 006 sigmas and both sizes, and
    ``aug_oracle.gaussian`` against ``cv2.GaussianBlur`` on random frames;
  * ``aug_oracle.filter2d`` against ``cv2.filter2D`` for dense random kernels of 1x1 to 30x30: equal up to 11x11
    (OpenCV's direct path); for 12x12 and larger (its DFT path) the differing values are counted.

Run:  python tests/golden/check_aug_opencv.py      (exit status 1 on any mismatch)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader as R                                  # noqa: E402
from oracle import aug_oracle as O                                  # noqa: E402
from ffb6d_b200 import augment as A                                 # noqa: E402


def tail_layout(px, w=48):
    """Put pixels [n,3] into the last w % 32 columns of w-wide rows (OpenCV's scalar loop); returns image, unpack."""
    k = w % 32
    rows = len(px) // k
    img = np.zeros((rows, w, 3), np.uint8)
    img[:, w - k:] = px[: rows * k].reshape(rows, k, 3)
    return img, lambda out: out[:, w - k:].reshape(-1, 3), rows * k


def check_hsv(cv2):
    bad = 0
    a = np.arange(1 << 24, dtype=np.uint32)
    px = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8)
    for name, (img, unpack, n) in (("vector", (px.reshape(4096, 4096, 3), lambda o: o.reshape(-1, 3), len(px))),
                                   ("tail", tail_layout(px))):
        want = unpack(cv2.cvtColor(img, cv2.COLOR_BGR2HSV))
        got = np.stack(O.bgr2hsv(unpack(img)[None])[:3], -1)[0].astype(np.uint8)
        m = np.count_nonzero(np.any(want != got, -1))
        print("BGR2HSV %-6s: %d inputs, %d differ" % (name, n, m))
        bad += m
    h, s, v = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([h, s, v], -1).reshape(-1, 3).astype(np.uint8)
    for name, (img, unpack, n) in (("vector", (hsv.reshape(-1, 4096, 3), lambda o: o.reshape(-1, 3), len(hsv))),
                                   ("tail", tail_layout(hsv))):
        want = unpack(cv2.cvtColor(img, cv2.COLOR_HSV2BGR))
        x = img.astype(np.int64)
        got = unpack(O.hsv2bgr(x[..., 0], x[..., 1], x[..., 2]))
        m = np.count_nonzero(np.any(want != got, -1))
        print("HSV2BGR %-6s: %d inputs, %d differ" % (name, n, m))
        bad += m
    return bad


def check_motion(cv2):
    path = os.path.join(R.REF_ROOT, "ffb6d", "datasets", "ycb", "ycb_dataset.py")
    blur = R._extract(path, "Dataset", ["linear_motion_blur"])["linear_motion_blur"]
    captured = []

    class Cv2:
        line = staticmethod(cv2.line)

        @staticmethod
        def filter2D(img, depth, kern):
            captured.append(kern.copy())
            return img

    blur.__globals__.update(np=np, cv2=Cv2)
    bad = 0
    for angle in range(360):
        for length in range(1, 16):
            captured.clear()
            blur(None, np.zeros((1, 1, 3), np.uint8), angle, length)
            want = captured[0] if captured else None
            got = A.motion_kernel(angle, length)
            if (want is None) != (got is None) or (want is not None and not np.array_equal(want, got)):
                bad += 1
    print("motion kernels: 5400 (angle, length) pairs, %d differ" % bad)
    return bad


def check_gaussian(cv2):
    bad = 0
    rs = np.random.RandomState(1)
    sig = np.concatenate([rs.rand(4000), np.linspace(0, 1, 8001), [1e-300, 1e-160, 1e-9, 0.2, 0.3]])
    img = np.zeros((40, 40, 3), np.uint8)
    img[:, 20] = 255                    # rows constant: the response of a column of 255 gives each side tap exactly
    for n in (3, 5):
        for s in sig:
            resp = cv2.GaussianBlur(img, (n, n), s)[20, 20 - n // 2: 21 + n // 2, 0].astype(np.int64)
            resp[n // 2] = 256 - (resp.sum() - resp[n // 2])
            bad += not np.array_equal(resp, A.gaussian_taps(n, s))
    print("Gaussian taps: %d sigmas x 2 sizes, %d differ" % (len(sig), bad))
    nb = 0
    for h, w in ((33, 47), (480, 640)):
        frame = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        for n in (3, 5):
            for s in list(rs.rand(10)) + [0.0, 1e-5]:
                nb += not np.array_equal(O.gaussian(frame, A.gaussian_taps(n, s)), cv2.GaussianBlur(frame, (n, n), s))
    print("GaussianBlur: 48 frames, %d differ" % nb)
    return bad + nb


def check_filter2d(cv2):
    bad = 0
    rs = np.random.RandomState(0)
    for h, w in ((37, 45), (480, 640)):
        frame = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        for a in range(1, 31):
            k = rs.rand(a, a) * (rs.rand(a, a) < 0.3)
            k[a // 2, a // 2] += 0.5
            k /= k.sum()
            d = np.abs(O.filter2d(frame, k).astype(int) - cv2.filter2D(frame, -1, k))
            if a < 12:
                bad += np.count_nonzero(d)
            else:
                bad += d.max() > 1
                print("filter2D %3dx%-3d a=%2d (DFT path): %d of %d values differ by 1" %
                      (h, w, a, np.count_nonzero(d), d.size))
    print("filter2D direct path (a <= 11): %d mismatches" % bad)
    return bad


def main():
    import cv2
    cv2.setNumThreads(1)
    print("OpenCV", cv2.__version__)
    if not R.reference_sources_present():
        raise SystemExit("needs /root/reference")
    bad = check_hsv(cv2) + check_motion(cv2) + check_gaussian(cv2) + check_filter2d(cv2)
    print("FAIL" if bad else "all equal")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
