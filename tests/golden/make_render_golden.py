#!/usr/bin/env python
"""Generate tests/golden/render_ape.npz: the vertices, faces and vertex colours of the reference's example mesh
``utils/dataset_tools/example_mesh/ape.ply`` (ASCII PLY, 5841 vertices, 11678 faces, millimetres), the mesh the
rasteriser tests render (DESIGN.md §4.31).

Stored: ``xyz [V,3]`` float32 millimetres as the file writes them, ``faces [F,3]`` int32 and ``rgb [V,3]`` uint8
(the vertices' red, green, blue; the normals and alpha are dropped).  The file is read by the small ASCII-PLY reader
below (plyfile is not needed).

Run:  python tests/golden/make_render_golden.py <reference>/ffb6d/utils/dataset_tools/example_mesh/ape.ply
      (rewrites render_ape.npz)
"""
import os
import sys

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "render_ape.npz")


def read_ascii_ply(path):
    """``(xyz float32 [V,3], faces int32 [F,3], rgb uint8 [V,3])`` of an ASCII PLY with x, y, z, red, green, blue
    vertex properties and triangle faces."""
    with open(path) as f:
        if f.readline().strip() != "ply" or f.readline().strip() != "format ascii 1.0":
            raise ValueError("%s: not an ASCII PLY" % path)
        elements, props = [], {}
        for line in f:
            tok = line.split()
            if tok[0] == "end_header":
                break
            if tok[0] == "element":
                elements.append((tok[1], int(tok[2])))
                props[tok[1]] = []
            elif tok[0] == "property":
                props[elements[-1][0]].append(tok[-1])
        out = {}
        for name, n in elements:
            out[name] = [f.readline().split() for _ in range(n)]
    vp = props["vertex"]
    v = np.array(out["vertex"], dtype=np.float64)
    xyz = np.ascontiguousarray(v[:, [vp.index("x"), vp.index("y"), vp.index("z")]], dtype=np.float32)
    rgb = np.ascontiguousarray(v[:, [vp.index("red"), vp.index("green"), vp.index("blue")]], dtype=np.uint8)
    rows = out["face"]
    if any(int(r[0]) != 3 for r in rows):
        raise ValueError("%s: only triangle faces are supported" % path)
    faces = np.array([r[1:4] for r in rows], dtype=np.int32)
    return xyz, faces, rgb


def main():
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    xyz, faces, rgb = read_ascii_ply(sys.argv[1])
    np.savez_compressed(OUT, xyz=xyz, faces=faces, rgb=rgb)
    print("wrote %s: %d vertices, %d faces" % (OUT, len(xyz), len(faces)))


if __name__ == "__main__":
    main()
