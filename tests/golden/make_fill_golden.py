#!/usr/bin/env python
"""Generate tests/golden/fill_cases.npz by running THE REFERENCE'S OWN depth completion in this container.

Source of truth: ``Basic_Utils.fill_missing`` (utils/basic_utils.py:467-487) and ip_basic's ``fill_in_multiscale``
(utils/ip_basic/ip_basic/depth_map_utils_ycb.py:290-443), executed from the reference's source text with numpy and
cv2 (basic_utils.py imports normalSpeed, so the method is taken out of the file with ``ast``).  The inputs are the raw
frames of ``ffb6d_b200.synthetic.fill_test_frames``; the tests regenerate them from their seeds.

Stored per frame:
  * small frames: every stage of ``show_process=True`` (s7 / s8 after the bilateral blur) and the output;
  * the two 480x640 frames, to keep the file small: a sha256 per bit-exact stage; which pixels the bilateral blur
    writes (the same run with ``cv2.bilateralFilter`` returning NaN marks them), as a sha256; the sha256 of the output
    with those pixels zeroed (everything else is bit-exact); the sha256 of ``msk_dp = out > 1e-6``; and the
    reference's output at a seeded sample of the blurred pixels.

Run:  python tests/golden/make_fill_golden.py      (needs /root/reference and cv2; rewrites fill_cases.npz)
"""
import hashlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader as R                                              # noqa: E402
from ffb6d_b200.synthetic import fill_test_frames, FILL_CAM_SCALE               # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fill_cases.npz")
EXACT_STAGES = ("s1_inverted_depths", "s2_dilated_depths", "s3_closed_depths", "s4_blurred_depths",
                "s5_combined_depths", "s6_extended_depths")
N_SAMPLE = 8192        # blurred pixels of a full frame whose reference value is stored


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def reference_functions():
    """(fill_missing(dpt, cam_scale, scale_2_80m, ...), fill_in_multiscale, fill_in_multiscale with a NaN bilateral)."""
    import cv2
    utils = os.path.join(R.REF_ROOT, "ffb6d", "utils")
    path = os.path.join(utils, "ip_basic", "ip_basic", "depth_map_utils_ycb.py")

    def load():
        mod = types.ModuleType("depth_map_utils_ycb")
        mod.__file__ = path
        with open(path) as fh:
            exec(compile(fh.read(), path, "exec"), mod.__dict__)
        return mod

    class NanBilateral:
        """cv2 with a bilateralFilter whose every output is NaN: the pixels it is written to stay NaN."""
        def __getattr__(self, name):
            return getattr(cv2, name)

        @staticmethod
        def bilateralFilter(src, *args, **kwargs):
            return np.full_like(src, np.nan)

    dmu, marked = load(), load()
    marked.cv2 = NanBilateral()
    fm = R._extract(os.path.join(utils, "basic_utils.py"), "Basic_Utils", ["fill_missing"])["fill_missing"]
    fm.__globals__.update(np=np, depth_map_utils=dmu)
    return (lambda *a, **kw: fm(None, *a, **kw)), dmu.fill_in_multiscale, marked.fill_in_multiscale


def fill_cases():
    fill_missing, multiscale, multiscale_marked = reference_functions()
    cs = np.float32(FILL_CAM_SCALE)
    kw = dict(max_depth=3.0, extrapolate=False, blur_type='bilateral')
    out = {}
    for name, raw in fill_test_frames().items():
        filled = fill_missing(raw, cs, 1)
        assert filled.dtype == np.float32
        _, st = multiscale(raw / cs * 1, show_process=True, **kw)
        out[name + "/sha256_raw"] = np.array(sha(raw))
        if not name.startswith("full"):
            out[name + "/out"] = filled
            for k in EXACT_STAGES + ("s7_blurred_depths", "s8_inverted_depths"):
                out[name + "/" + k] = st[k]
            continue
        blurred = np.isnan(multiscale_marked(raw / cs * 1, **kw)[0])
        unblurred = filled.copy()
        unblurred[blurred] = 0
        idx = np.sort(np.random.RandomState(len(name)).choice(np.flatnonzero(blurred), N_SAMPLE, replace=False))
        out.update({name + "/sha256_blurred": np.array(sha(blurred)),
                    name + "/sha256_out_unblurred": np.array(sha(unblurred)),
                    name + "/sha256_msk_dp": np.array(sha(filled > np.float32(1e-6))),
                    name + "/sample_idx": idx.astype(np.int32),
                    name + "/sample_out": filled.reshape(-1)[idx]})
        for k in EXACT_STAGES:
            out[name + "/sha256_" + k] = np.array(sha(st[k]))
    return out


def main():
    if not R.reference_sources_present():
        raise SystemExit("needs /root/reference")
    np.savez_compressed(OUT, **fill_cases())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
