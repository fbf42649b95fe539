#!/usr/bin/env python
"""Check oracle/sift_oracle.py against OpenCV beyond the cases of sift_cases.npz.

A build-machine script (needs cv2; the result belongs to the OpenCV it runs with and its CPU dispatch, so it is not a
test).  It checks, printing the mismatch count of each step:
  * ``gaussian_taps`` against ``cv2.getGaussianKernel`` for every sigma of the pyramid;
  * ``blur`` against ``cv2.GaussianBlur`` on float32 images of every width 2..48 and of the pyramid's own sizes for a
    480 x 640 input, at every sigma of the pyramid (elements that differ);
  * ``upscale`` against ``cv2.resize(..., INTER_LINEAR)`` and the octave base against ``INTER_NEAREST``;
  * ``exp32`` / ``atan32`` / ``mag32`` against ``cv2.exp`` / ``cv2.phase`` / ``cv2.magnitude`` over dense grids
    (values that differ, and the largest difference in units in the last place);
  * ``detect`` against ``cv2.SIFT_create().detect``: the keypoint count, the multiset of (octave, pt) bitwise, of
    (octave, pt, size) bitwise, the largest angle difference where those agree, and the tool's integer pixels
    ``int32(pt)`` as a multiset, on filled circles, blurred noise, noise, rectangles, tiles, odd and tiny sizes and
    ape renders from the tool's sphere of views.

Run:  python tests/golden/check_sift_opencv.py      (exit status 1 when the keypoint counts or pixels differ)
"""
import collections
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import sift_oracle as S                                  # noqa: E402
import orb_cases as OC                                               # noqa: E402
import sift_cases as SC                                              # noqa: E402

f32 = np.float32


def sigmas():
    return [S.base_sigma()] + S.layer_sigmas()


def check_taps(cv2):
    bad = sum(not np.array_equal(S.gaussian_taps(s), cv2.getGaussianKernel(len(S.gaussian_taps(s)), s,
                                                                             cv2.CV_32F).ravel()) for s in sigmas())
    print("gaussian taps: %d sigmas, %d differ" % (len(sigmas()), bad))
    return bad


def check_blur(cv2, rng):
    sizes = [(h, w) for w in range(2, 49) for h in (2, 3, 5, 13, 20)]
    sizes += S.octave_sizes(480, 640) + S.octave_sizes(33, 251)
    n = bad = 0
    by_path = collections.Counter()
    for h, w in sizes:
        for s in sigmas():
            img = (rng.random((h, w)) * 255).astype(f32)
            d = cv2.GaussianBlur(img, (0, 0), s, s) != S.blur(img, S.gaussian_taps(s))
            n += d.size
            bad += int(d.sum())
            for x in np.nonzero(d)[1]:
                by_path[int(S.column_modes(w)[x])] += 1
    print("blur: %d sizes x %d sigmas, %d of %d values differ (by column path 0/1/2: %s)"
          % (len(sizes), len(sigmas()), bad, n, dict(by_path)))
    return bad, n


def check_resize(cv2, rng):
    bad = 0
    for h, w in [(4, 4), (5, 7), (33, 251), (97, 131), (480, 640)]:
        g = rng.integers(0, 256, (h, w)).astype(f32)
        up = cv2.resize(g, (2 * w, 2 * h), interpolation=cv2.INTER_LINEAR)
        bad += int((up != S.upscale(g)).sum())
        nn = cv2.resize(up, (w, h), interpolation=cv2.INTER_NEAREST)
        bad += int((nn != up[::2, ::2][:h, :w]).sum())
    print("upscale and octave base: %d values differ" % bad)
    return bad


def ulps(a, b):
    return int(np.max(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)), initial=0))


def check_hal(cv2):
    # exp over the weights calcOrientationHist takes: -(i^2 + j^2) / (2 sigma^2) >= -512 / (2 2.69^2) > -36
    x = np.linspace(-36, 0, 200001).astype(f32)
    e = cv2.exp(x.reshape(1, -1)).ravel()
    o = S.exp32(x)
    rel = float(np.max(np.abs(e.astype(np.float64) / o - 1)))
    print("exp32: %d of %d differ, at most %d ulp (relative %.2g)" % (int((e != o).sum()), x.size, ulps(e, o), rel))
    g = np.arange(-400, 401, dtype=f32) / f32(8)
    X, Y = (a.ravel().astype(f32) for a in np.meshgrid(g, g))
    a = cv2.phase(X, Y, angleInDegrees=True).ravel()
    b = S.atan32(Y, X)
    print("atan32: %d of %d differ, at most %.3g degrees" % (int((a != b).sum()), X.size, float(np.max(np.abs(a - b)))))
    m = cv2.magnitude(X, Y).ravel()
    n = S.mag32(X, Y)
    print("mag32: %d of %d differ, at most %d ulp" % (int((m != n).sum()), X.size, ulps(m, n)))


def images(rng):
    for s in range(12):
        yield "circles", SC.image(6, 100 + s, *rng.integers(60, 300, 2))
    for s in range(6):
        yield "blurred", OC.image(1, 200 + s, *rng.integers(60, 300, 2))
    for s in range(4):
        yield "noise", OC.image(0, 300 + s, *rng.integers(40, 160, 2))
    for s in range(4):
        yield "rectangles", OC.image(3, 400 + s, *rng.integers(60, 240, 2))
    for s in range(3):
        yield "tiles", OC.image(2, s, *rng.integers(40, 200, 2))
    for s in range(10):
        yield "tiny", SC.image(6, 500 + s, *rng.integers(4, 24, 2))
    yield "circles", SC.image(6, 3, 480, 640)
    xyz, K, H, W, radius = OC.ape_setup()
    from ffb6d_b200.objinfo import sphere_poses
    for RT in sphere_poses(radius, 3, 3):
        yield "ape", OC.ape_render(RT)[1]


def check_detect(cv2, rng):
    sift = cv2.SIFT_create()
    per = collections.OrderedDict()
    size_ulps = [0]
    bad = 0
    for kind, img in images(rng):
        kps = sift.detect(np.ascontiguousarray(img[..., ::-1]), None)
        d = S.detect(img)
        cv_loc = collections.Counter((k.octave, f32(k.pt[0]).item(), f32(k.pt[1]).item()) for k in kps)
        or_loc = collections.Counter(zip(d["octave"].tolist(), d["pt"][:, 0].tolist(), d["pt"][:, 1].tolist()))
        cv_sz = collections.Counter((k.octave, f32(k.pt[0]).item(), f32(k.pt[1]).item(), f32(k.size).item())
                                    for k in kps)
        or_sz = collections.Counter(zip(d["octave"].tolist(), d["pt"][:, 0].tolist(), d["pt"][:, 1].tolist(),
                                        d["size"].tolist()))
        cv_px = collections.Counter(tuple(np.array(k.pt, f32).astype(np.int32).tolist()) for k in kps)
        or_px = collections.Counter(map(tuple, d["pt"].astype(np.int32).tolist()))
        ang = {}
        for k in kps:
            ang.setdefault((k.octave, f32(k.pt[0]).item(), f32(k.pt[1]).item(), f32(k.size).item()), []).append(k.angle)
        amax = 0.0
        for key, a in zip(zip(d["octave"].tolist(), d["pt"][:, 0].tolist(), d["pt"][:, 1].tolist(),
                              d["size"].tolist()), d["angle"].tolist()):
            if key in ang:
                dd = np.abs(np.array(ang[key]) - a)
                amax = max(amax, float(np.min(np.minimum(dd, 360 - dd))))
        for key in set(cv_loc) & set(or_loc):
            a = sorted(f32(k.size).view(np.int32).item() for k in kps
                       if (k.octave, f32(k.pt[0]).item(), f32(k.pt[1]).item()) == key)
            b = sorted(f32(z).view(np.int32).item() for o, x, y, z in zip(d["octave"].tolist(), d["pt"][:, 0].tolist(),
                                                                        d["pt"][:, 1].tolist(), d["size"].tolist())
                       if (o, x, y) == key)
            if len(a) == len(b):
                size_ulps[0] = max(size_ulps[0], max(abs(u - v) for u, v in zip(a, b)))
        s = per.setdefault(kind, [0, 0, 0, 0, 0, 0, 0.0])
        s[0] += 1
        s[1] += len(kps)
        s[2] += len(kps) != len(d["octave"])
        s[3] += sum((cv_loc - or_loc).values())
        s[4] += sum((cv_sz - or_sz).values())
        s[5] += sum((cv_px - or_px).values())
        s[6] = max(s[6], amax)
        bad += (len(kps) != len(d["octave"])) + (cv_px != or_px)
    print("detect: kind, images, OpenCV keypoints, images with another count, keypoints whose (octave, pt) / "
          "(octave, pt, size) / int32 pixel is missing, largest angle difference (degrees)")
    for kind, s in per.items():
        print("  %-10s %3d %6d %3d %4d %4d %4d %.3g" % (kind, *s))
    print("largest size difference where (octave, pt) agree: %d ulp" % size_ulps[0])
    return bad


def main():
    import cv2
    print("OpenCV", cv2.__version__)
    rng = np.random.default_rng(20261019)
    check_taps(cv2)
    check_blur(cv2, rng)
    check_resize(cv2, rng)
    check_hal(cv2)
    bad = check_detect(cv2, rng)
    print("images whose keypoint count or integer pixels differ:", bad)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
