#!/usr/bin/env python
"""Generate tests/golden/fps_cases.npz from the reference's own farthest point sampling and mesh arithmetic.

Source of truth:
* the unmodified utils/dataset_tools/fps/src/farthest_point_sampling.cpp, compiled by oracle/fps_ref.mk
  (oracle/fps_oracle.py calls it through ctypes);
* ``MeshUtils.get_3D_bbox``, ``get_r`` and ``get_centers_3d`` of utils/dataset_tools/utils.py, taken out of the file
  with ``ast`` and executed (importing the file needs cv2 and plyfile).
Nothing of the reference is copied: the clouds are regenerated from seeds (tests/fps_cases.py) and only the
reference's outputs are stored.

Keys:
* ``<case>:ic`` / ``<case>:rs`` -- int32 [S] indices with init_center, and from the reference's random start (its
  first index);
* ``batch:ic`` / ``batch:rs`` [G,S] -- each cloud of ``batch_clouds()``; ``ragged:ic`` [G,S] -- each cloud cut to
  its first ``BATCH_N[g]`` points;
* ``objinfo:<array>:corners`` / ``:radius`` / ``:center`` -- the MeshUtils functions on ``objinfo_arrays()``.

Run:  python tests/golden/make_fps_golden.py      (needs the reference's sources, see oracle/ref_loader.py; rewrites fps_cases.npz)
"""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import fps_oracle, ref_loader as R                       # noqa: E402
import fps_cases as FC                                               # noqa: E402

OUT = os.path.join(HERE, "fps_cases.npz")
BATCH_S = 40


def mesh_utils():
    """{'get_3D_bbox', 'get_r', 'get_centers_3d'} of the reference's MeshUtils as plain functions of self."""
    path = os.path.join(R.REF_ROOT, "ffb6d", "utils", "dataset_tools", "utils.py")
    with open(path) as fh:
        tree = ast.parse(fh.read())
    names = ("get_3D_bbox", "get_r", "get_centers_3d")
    ns = {"np": np}
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == "MeshUtils":
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in names:
                    exec(compile(ast.Module(body=[item], type_ignores=[]), path, "exec"), ns)
    return {n: (lambda f: lambda *a: f(None, *a))(ns[n]) for n in names}


def main():
    out = {}
    for name, (make, S) in FC.CASES.items():
        pts = make()
        out[name + ":ic"] = fps_oracle.fps(pts, S, init_center=True)
        out[name + ":rs"] = fps_oracle.fps(pts, S, init_center=False)
        print(name, pts.shape, S, out[name + ":ic"][:8], out[name + ":rs"][:8])
    clouds = FC.batch_clouds()
    out["batch:ic"] = np.stack([fps_oracle.fps(c, BATCH_S, True) for c in clouds])
    out["batch:rs"] = np.stack([fps_oracle.fps(c, BATCH_S, False) for c in clouds])
    out["ragged:ic"] = np.stack([fps_oracle.fps(c[:n], BATCH_S, True) for c, n in zip(clouds, FC.BATCH_N)])
    mu = mesh_utils()
    for name, a in FC.objinfo_arrays().items():
        c = mu["get_3D_bbox"](a)
        out["objinfo:%s:corners" % name] = c
        out["objinfo:%s:radius" % name] = np.asarray(mu["get_r"](c))
        out["objinfo:%s:center" % name] = mu["get_centers_3d"](c)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
