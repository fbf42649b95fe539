#!/usr/bin/env python
"""Check the colour-jitter restatement (oracle/jitter_oracle.py) against the installed Pillow beyond the fixture:

- ``convert("HSV")`` of every RGB value and ``convert("RGB")`` of every HSV value (2^24 inputs each);
- ``convert("L")`` of every RGB value;
- ``Image.blend`` on every (a, b) byte pair for a sweep of factors on both of its branches (0 <= f <= 1: truncate;
  otherwise clip and truncate), including factors that round to 1.0 as a C float.

A script, not a test: it needs Pillow, which the GPU machines do not have.  Prints one line per check and exits
non-zero on any difference.

Run:  python tests/golden/check_jitter_pil.py
"""
import os
import sys

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import jitter_oracle as O          # noqa: E402

SLAB = 1 << 20                                 # inputs per slab: a 1024 x 1024 image


def all_triples(k):
    """Slab k of the 2^24 byte triples, as a [1024, 1024, 3] uint8 image."""
    n = np.arange(k * SLAB, (k + 1) * SLAB, dtype=np.int64)
    return np.stack([n >> 16, (n >> 8) & 255, n & 255], -1).astype(np.uint8).reshape(1024, 1024, 3)


def pil(a, mode):
    return Image.frombytes(mode, (a.shape[1], a.shape[0]), np.ascontiguousarray(a).tobytes())


def check_conversions():
    bad = {"rgb2hsv": 0, "hsv2rgb": 0, "L": 0}
    for k in range(1 << 24 >> 20):
        x = all_triples(k)
        want = np.asarray(pil(x, "RGB").convert("HSV"))
        bad["rgb2hsv"] += np.count_nonzero(np.any(O.rgb2hsv(x) != want, -1))
        want = np.asarray(pil(x, "HSV").convert("RGB"))
        bad["hsv2rgb"] += np.count_nonzero(np.any(O.hsv2rgb(x) != want, -1))
        want = np.asarray(pil(x, "RGB").convert("L"))
        bad["L"] += np.count_nonzero(O.luma(x) != want)
    for name, n in bad.items():
        print("%-8s 16777216 inputs: %d differ" % (name, n))
    return sum(bad.values()) == 0


FACTORS = [0.0, 1e-8, 0.25, 0.5, 0.8, 0.8000001, 0.9999999, 1.0, 1.00000001, 1.0000001, 1.05, 1.2, 1.5, 2.0, 3.7,
           255.0, 1e6]


def check_blend():
    a, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    ok = True
    for f in FACTORS:
        want = np.asarray(Image.blend(pil(a, "L"), pil(b, "L"), f))
        n = np.count_nonzero(O.blend(a, b, f) != want)
        branch = "truncate" if 0 <= np.float32(f) <= 1 else "clip"
        print("blend    factor %-11r (%s) 65536 pairs: %d differ" % (f, branch, n))
        ok &= n == 0
    return ok


def main():
    ok = check_conversions()
    ok &= check_blend()
    print("all equal" if ok else "DIFFERENCES FOUND")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
