#!/usr/bin/env python
"""Generate tests/golden/orb_cases.npz: OpenCV's ORB keypoints of generated images and of ape renders, and the
reference's sphere poses and lifted keypoints of the ape.

Source of truth:
* ``cv2.ORB_create().detect`` on each image's BGR form (the OpenCV installed where this runs; its version is stored);
* ``PoseUtils.CameraPositions`` / ``getCameraPose`` / ``get_o2c_pose_cv`` and ``ImgPcldUtils.dpt_2_cld`` /
  ``filter_pcld`` of the reference's utils/dataset_tools/utils.py, taken out of the file with ``ast`` and executed,
  composed as ``gen_one_zbuf_render`` composes them (rgbd_rnder_sift_kp3ds.py:138-155).
Nothing of the reference is copied.  Images are stored as generator parameters (``orb_cases.image``), renders as the
ape of render_ape.npz, its poses and oracle/render_oracle.py, so the fixture holds keypoints, not pixels.

Keys:
* ``cases [n,4]`` int64 (kind, seed, H, W); ``ape_poses [V,4,4]`` float64 (the reference's), ``ape_radius`` float32,
  ``ape_views [k]`` the rendered view indices, ``ape_K`` / ``ape_hw``;
* ``kp:<name>`` ``[m,4]`` float32 (octave, x, y, response) of OpenCV's keypoints, name ``i`` or ``ape<v>``;
* ``lift:ape<v>`` ``[m,3]`` float64: the reference's object-frame points of view v;
* ``cv2_version``.

Run:  python tests/golden/make_orb_golden.py      (needs cv2 and the reference's sources; rewrites orb_cases.npz)
"""
import ast
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_loader as R                                   # noqa: E402
import orb_cases as OC                                               # noqa: E402

OUT = os.path.join(HERE, "orb_cases.npz")


def ref_utils():
    """The reference's pose and point-cloud helpers as plain functions of self."""
    path = os.path.join(R.REF_ROOT, "ffb6d", "utils", "dataset_tools", "utils.py")
    with open(path) as fh:
        tree = ast.parse(fh.read())
    want = {"PoseUtils": ("CameraPositions", "getCameraPose", "get_o2c_pose_cv", "get_3x4_RT_matrix_from_blender"),
            "ImgPcldUtils": ("dpt_2_cld", "filter_pcld")}
    ns = {"np": np, "math": math}
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name in want:
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in want[node.name]:
                    exec(compile(ast.Module(body=[item], type_ignores=[]), path, "exec"), ns)

    class Self:
        pass
    me = Self()
    for name in ("get_3x4_RT_matrix_from_blender",):
        setattr(me, name, (lambda f: lambda *a: f(me, *a))(ns[name]))
    return {n: (lambda f: lambda *a: f(me, *a))(ns[n])
            for names in want.values() for n in names}


def keypoints(cv2, rgb):
    kps = cv2.ORB_create().detect(np.ascontiguousarray(rgb[..., ::-1]), None)
    return kps, np.array([(k.octave, k.pt[0], k.pt[1], k.response) for k in kps], np.float32).reshape(-1, 4)


def main():
    import cv2
    out = {"cases": np.array(OC.CASES, np.int64), "cv2_version": np.array(cv2.__version__)}
    for i, case in enumerate(OC.CASES):
        out["kp:%d" % i] = keypoints(cv2, OC.image(*case))[1]
    u = ref_utils()
    xyz, K, H, W, radius = OC.ape_setup()
    sph_r = radius / 0.035 * 0.18
    poses = np.stack([u["get_o2c_pose_cv"](u["getCameraPose"](p), np.eye(4))
                      for p in u["CameraPositions"](3, 3, sph_r)])
    out.update(ape_poses=poses, ape_radius=np.asarray(radius), ape_views=np.array(OC.APE_VIEWS),
               ape_K=K, ape_hw=np.array([H, W]))
    for v in OC.APE_VIEWS:
        depth, rgb = OC.ape_render(poses[v])
        kps, arr = keypoints(cv2, rgb)
        out["kp:ape%d" % v] = arr
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
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes; OpenCV", cv2.__version__)


if __name__ == "__main__":
    main()
