#!/usr/bin/env python
"""Time the textured rasteriser (DESIGN.md §4.35) on the GPU.

* ``render_rgbd`` of the example cracker box (tests/golden/textured_box.npz, the cuboid of tests/textured_cases.py)
  from a :class:`TexturedMeshTable` against a :class:`RenderMeshTable` of the same geometry, at 480 x 640 for
  B = 1, 8 and 32 frames of the tool's views (repeated): three windows of each, alternated, median and range.
* The mip build of one 4096^2 texture (``TexturedMeshTable`` construction's device part, ``ffb6d_render_texture_mips``).
* The whole ``objinfo.textured_kp3ds`` of the box, ORB and SIFT.

Times are CUDA events around ``--iters`` calls after ``--warmup``; the card's name and power limit are read in the same
run.  Prints one JSON object (and writes it to ``--out`` when given).

    python tools/textured_render_bench.py [--iters 50] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import ffb6d_b200 as F  # noqa: E402
from ffb6d_b200 import _lib, objinfo  # noqa: E402
from ffb6d_b200.render import RenderMeshTable, TexturedMeshTable  # noqa: E402
import textured_cases as TC  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q.stdout.strip())


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def windows(fns, iters, warmup, n=3):
    """``{name: [ms per call] * n}``: ``n`` windows of each function, alternated."""
    out = {k: [] for k in fns}
    for _ in range(n):
        for k, fn in fns.items():
            out[k].append(timed(fn, iters, warmup))
    return out


def summary(ts):
    return dict(median_ms=float(np.median(ts)), min_ms=float(min(ts)), max_ms=float(max(ts)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("textured_render_bench: needs a CUDA device")
    res = dict(card=card())
    mesh = TC.box_mesh()
    tex_t = TexturedMeshTable([mesh])
    flat_t = RenderMeshTable([(mesh[0], mesh[1], np.full(mesh[0].shape, 128, np.uint8))])
    pts = TC.GOLDEN["points"]
    centre = np.mean(pts.astype(np.float64), axis=0)
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(pts)), centre=centre)
    Kd = torch.tensor([700.0, 700.0, 320.0, 240.0], dtype=torch.float64, device="cuda")
    res["render"] = {}
    for B in (1, 8, 32):
        idx = torch.zeros((B, 1), dtype=torch.int32, device="cuda")
        RT = torch.from_numpy(poses[np.arange(B) % 9][:, None, :3, :].astype(np.float32)).cuda()
        lab = torch.ones((B, 1), dtype=torch.uint8, device="cuda")
        out = (torch.empty((B, 480, 640), dtype=torch.uint16, device="cuda"),
               torch.empty((B, 480, 640, 3), dtype=torch.uint8, device="cuda"),
               torch.empty((B, 480, 640), dtype=torch.uint8, device="cuda"))
        w = windows({"textured": lambda: F.render_rgbd(tex_t, idx, RT, lab, Kd, 480, 640, out=out),
                     "vertex_coloured": lambda: F.render_rgbd(flat_t, idx, RT, lab, Kd, 480, 640, out=out)},
                    args.iters, args.warmup)
        res["render"]["B=%d" % B] = {k: summary(v) for k, v in w.items()}
    # the mip build of one 4096^2 texture: the library call alone, on a table already packed
    big = TexturedMeshTable([(mesh[0], mesh[1], mesh[2], TC.noise_texture(4096, 1))])

    def mips():
        _lib.launch(_lib.lib.ffb6d_render_texture_mips, big.device, big.tex.data_ptr(), big.tex_hw.data_ptr(),
                    big.tex_off.data_ptr(), 1, big.max_tex_side)

    res["mips_4096"] = summary(windows({"m": mips}, args.iters, args.warmup)["m"])
    r = objinfo.get_r(objinfo.get_3D_bbox(pts))
    kp = windows({e: (lambda e=e: objinfo.textured_kp3ds(tex_t, 0, radius=r, centre=centre, extractor=e))
                  for e in ("ORB", "SIFT")}, max(1, args.iters // 5), 2)
    res["textured_kp3ds"] = {k: summary(v) for k, v in kp.items()}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
