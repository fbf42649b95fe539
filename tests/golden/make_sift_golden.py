#!/usr/bin/env python
"""Generate tests/golden/sift_cases.npz: OpenCV's SIFT keypoints of generated images and of ape renders, and the
reference tool's SIFT-branch lifted keypoints of the ape.

Source of truth:
* ``cv2.SIFT_create().detectAndCompute`` on each image's BGR form, as the tool calls it (the OpenCV installed where
  this runs; its version is stored).  The tool calls ``cv2.xfeatures2d.SIFT_create()``, the same algorithm, which
  OpenCV >= 4.4 also exposes as ``cv2.SIFT_create`` (pip builds carry no ``xfeatures2d``);
* the reference's pose and point-cloud helpers, taken out of utils/dataset_tools/utils.py with ``ast`` by
  make_orb_golden.py and composed as ``gen_one_zbuf_render`` composes them (rgbd_rnder_sift_kp3ds.py:138-155).
Nothing of the reference is copied.  Images are stored as generator parameters (``sift_cases.image``), renders as the
ape of render_ape.npz, its poses and oracle/render_oracle.py.

Keys:
* ``cases [n,4]`` int64 (kind, seed, H, W); ``ape_poses [V,4,4]`` float64 (the reference's), ``ape_views [k]``;
* ``kp:<name>`` ``[m,5]`` float32 (x, y, size, angle, response) and ``oct:<name>`` ``[m]`` int32 (packed octave) of
  OpenCV's keypoints, name ``i`` or ``ape<v>``;
* ``lift:ape<v>`` ``[m,3]`` float64: the reference's object-frame points of view v; ``liftpt:ape<v>`` their pixels;
* ``cv2_version``.

The archive is written uncompressed with fixed member times, so a rerun with the same OpenCV reproduces it byte for
byte.

Run:  python tests/golden/make_sift_golden.py      (needs cv2 and the reference's sources; rewrites sift_cases.npz)
"""
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)
import orb_cases as OC                                               # noqa: E402
import sift_cases as SC                                              # noqa: E402
from make_orb_golden import ref_utils                                # noqa: E402

OUT = os.path.join(HERE, "sift_cases.npz")


def keypoints(cv2, rgb):
    kps, _ = cv2.SIFT_create().detectAndCompute(np.ascontiguousarray(rgb[..., ::-1]), None)
    arr = np.array([(k.pt[0], k.pt[1], k.size, k.angle, k.response) for k in kps], np.float32).reshape(-1, 5)
    return kps, arr, np.array([k.octave for k in kps], np.int32)


def save(path, arrays):
    """np.savez with fixed zip member times and sorted keys: the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    import cv2
    out = {"cases": np.array(SC.CASES, np.int64), "cv2_version": np.array(cv2.__version__)}
    for i, case in enumerate(SC.CASES):
        _, out["kp:%d" % i], out["oct:%d" % i] = keypoints(cv2, SC.image(*case))
    u = ref_utils()
    xyz, K, H, W, radius = OC.ape_setup()
    sph_r = radius / 0.035 * 0.18
    poses = np.stack([u["get_o2c_pose_cv"](u["getCameraPose"](p), np.eye(4))
                      for p in u["CameraPositions"](3, 3, sph_r)])
    out.update(ape_poses=poses, ape_views=np.array(SC.APE_VIEWS))
    for v in range(len(poses)):
        depth, rgb = OC.ape_render(poses[v])
        kps, arr, octs = keypoints(cv2, rgb)
        if v in SC.APE_VIEWS:
            out["kp:ape%d" % v], out["oct:ape%d" % v] = arr, octs
        # gen_one_zbuf_render's lift (rgbd_rnder_sift_kp3ds.py:138-155)
        kp_xys = np.array([kp.pt for kp in kps]).astype(np.int32)
        kp_idxs = (kp_xys[:, 1], kp_xys[:, 0])
        dpt_xyz = u["dpt_2_cld"](depth, 1.0, K)
        kp_xyz = np.concatenate([dpt_xyz[:, :, c][kp_idxs][..., None] for c in range(3)], axis=1)
        kp_xyz, msk = u["filter_pcld"](kp_xyz)
        RT = poses[v]
        out["lift:ape%d" % v] = (kp_xyz - RT[:3, 3]).dot(RT[:3, :3])
        out["liftpt:ape%d" % v] = np.array([kp.pt for kp in kps], np.float32).reshape(-1, 2)
        print("ape view", v, len(kps), "keypoints,", int(msk.sum()), "lifted")
    save(OUT, out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes; OpenCV", cv2.__version__)


if __name__ == "__main__":
    main()
