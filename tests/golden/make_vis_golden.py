#!/usr/bin/env python
"""Generate tests/golden/vis_cases.npz from the reference's own drawing code.

Source of truth: ``Basic_Utils.project_p3d`` / ``draw_p2ds`` / ``get_label_color`` and train_ycb.py's
``view_labels`` / ``color_lst``, taken out of the reference's files with ``ast`` and run with cv2 and numpy on this
machine (oracle/vis_oracle.reference_functions); the demo's drawing block (demo.py:116-145) is restated over them.
Inputs are rebuilt from seeds by tests/vis_cases.py.  Nothing of the reference is copied.

Before writing, the fma chains of oracle/vis_oracle.dot3 are checked against ``np.dot`` for N = 1, 2, 3, 8, 9,
2621 and 12288 points, for the intrinsics and the pose products; the script refuses to write if they differ (the
golden data would then depend on a BLAS kernel the projection kernel does not restate).

Keys:
* ``proj:<name>`` -- the reference's ``project_p3d`` of ``vis_cases.proj_cases()[name]`` (posed first with
  ``np.dot(p, R.T) + t`` where the case has a pose), int32 ``[N,2]``; over 1 000 points ``proj:<name>:sha256``;
* ``draw:<name>`` -- ``draw_p2ds`` applied in order to a copy of the case's 64 x 80 background, the whole image;
* ``demo:<dataset>:sha256`` -- the BGR image of the demo's drawing block on ``vis_cases.demo_frames()``;
* ``view_labels:sha256`` -- ``view_labels`` of ``vis_cases.view_labels_frame()`` with the YCB K;
* ``color:mode0`` / ``color:mode1`` ``[22,3]``, ``color:mode2:<n_obj>`` ``[n_obj + 3,3]``, ``color_lst:<n>``.

Run:  python tests/golden/make_vis_golden.py      (needs the reference's sources and cv2; rewrites vis_cases.npz)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import vis_oracle as O              # noqa: E402
import vis_cases as VC                          # noqa: E402

OUT = os.path.join(HERE, "vis_cases.npz")


def check_fma_chain():
    rs = np.random.RandomState(99)
    for n in VC.PROJ_SIZES:
        for K in (VC.K_YCB, VC.K_LM, VC.K_INT):
            p = rs.normal(0, 0.3, (n, 3)) + [0, 0, 1]
            if not np.array_equal(np.dot(p, K.T), O.dot3(p, K)):
                raise SystemExit("np.dot(p, K.T) differs from the fma chain at N = %d: not writing" % n)
        R = VC.pose_in_front(rs)
        p = rs.normal(0, 0.05, (n, 3))
        if not np.array_equal(np.dot(p, R[:, :3].T) + R[:, 3], O.dot3(p, R[:, :3]) + R[:, 3]):
            raise SystemExit("the posing np.dot differs from the fma chain at N = %d: not writing" % n)


def main():
    check_fma_chain()
    fns = O.reference_functions()
    out = {}
    with np.errstate(all="ignore"):
        for name, (p, cs, K, pose) in VC.proj_cases().items():
            if pose is not None:
                p = np.dot(p, pose[:, :3].T) + pose[:, 3]
            got = fns["project_p3d"](p.copy(), cs, K)
            if len(got) > VC.STORE_WHOLE:
                out["proj:%s:sha256" % name] = np.array(VC.sha(got))
            else:
                out["proj:" + name] = got
    for name, (bg, sets) in VC.draw_cases().items():
        img = bg.copy()
        for p2ds, r, cols in sets:
            img = fns["draw_p2ds"](img, p2ds.copy(), r, list(cols))
        out["draw:" + name] = img
    for ds, f in VC.demo_frames().items():
        bgr = O.demo_draw(f["rgb"], f["cls_ids"], f["pred_cls_ids"], f["pred_pose_lst"], f["mesh_pts"], f["K"], ds,
                          f["obj_id"], fns)
        out["demo:%s:sha256" % ds] = np.array(VC.sha(bgr))
    import torch
    cld, labels = VC.view_labels_frame()
    rgb = torch.zeros((1, 3, 480, 640))
    show = fns["view_labels"](rgb, torch.from_numpy(cld), torch.from_numpy(labels), VC.K_YCB)
    out["view_labels:sha256"] = np.array(VC.sha(show))
    for mode in (0, 1):
        out["color:mode%d" % mode] = np.array([fns["get_label_color"](c, mode=mode) for c in range(22)], np.int64)
    for n in (2, 13, 22):
        out["color:mode2:%d" % n] = np.array([fns["get_label_color"](c, n_obj=n, mode=2) for c in range(n + 3)],
                                             np.int64)
    for n in (2, 22):
        out["color_lst:%d" % n] = np.array(O.reference_functions(n)["color_lst"], np.int64)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d keys, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
