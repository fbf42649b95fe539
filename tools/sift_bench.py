#!/usr/bin/env python
"""Device time of the SIFT textured keypoint stages (DESIGN.md §4.33).

    python tools/sift_bench.py [--reps 20] [--rounds 5] [--out results/sift_bench.json]
    python tools/sift_bench.py --cpu                 # the CPU comparison: cv2 SIFT detect on the ape's views

GPU: CUDA-graph replays of ``sift_detect`` at 480x640 for B = 9 (one object's sphere of views) and B = 189 (21
objects x 9 views) of ape renders, and the whole ``textured_kp3ds(extractor="SIFT")`` of the ape (render, detect
with its count check, lift; eager).  Every shape is warmed up first; each figure is the mean over ``--reps`` calls
between CUDA events, repeated ``--rounds`` times (median, min and max reported), with the card's name and power limit
read in the same command.  ``--cpu`` times ``cv2.SIFT_create().detect`` on the ape's 9 views on the machine it runs
on (a CPU number, not a GPU one).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import orb_cases as OC                                              # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return dict(gpu=name, power_limit=power)


def timed(fn, reps, rounds):
    import torch
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) / reps)
    return dict(median=float(np.median(out)), min=min(out), max=max(out))


def graphed_detect(x):
    """A CUDA graph of one ``sift_detect(x, check=False)`` call; returns its replay."""
    import torch
    import ffb6d_b200 as F
    count = F.sift_detect(x)[0]                                     # warm-up, and the cap the frames need
    cap = max(int(count.max()), 1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        F.sift_detect(x, cap=cap, check=False)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        F.sift_detect(x, cap=cap, check=False)
    return g.replay


def gpu(reps, rounds):
    import ffb6d_b200 as F
    from ffb6d_b200 import objinfo
    from ffb6d_b200.render import RenderMeshTable
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(xyz)))
    _, img, _ = F.render_rgbd(table, np.zeros((9, 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                              np.ones((9, 1), np.uint8), objinfo.TOOL_K, 480, 640)
    res = card()
    replays = {B: graphed_detect(img.repeat(B // 9, 1, 1, 1).contiguous()) for B in (9, 189)}
    res["sift_detect_graph_ms"] = {str(B): timed(r, reps, rounds) for B, r in replays.items()}
    radius = objinfo.get_r(objinfo.get_3D_bbox(xyz))
    res["textured_kp3ds_sift_ape_ms"] = timed(
        lambda: objinfo.textured_kp3ds(table, 0, radius=radius, extractor="SIFT"), reps, rounds)
    res["shape"] = "480x640, ape renders; graph replays of sift_detect, eager textured_kp3ds"
    return res


def cpu(reps):
    import cv2
    from ffb6d_b200 import objinfo
    xyz, K, H, W, radius = OC.ape_setup()
    frames = [OC.ape_render(RT)[1] for RT in objinfo.sphere_poses(radius)]
    sift = cv2.SIFT_create()

    def run():
        for rgb in frames:
            sift.detect(np.ascontiguousarray(rgb[..., ::-1]), None)
    run()
    t = time.perf_counter()
    for _ in range(reps):
        run()
    return {"cpu_ape_9_views_ms": (time.perf_counter() - t) / reps * 1e3, "cv2": cv2.__version__,
            "threads": cv2.getNumThreads(), "note": "CPU number: cv2 SIFT detect only, renders excluded"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    res = cpu(args.reps) if args.cpu else gpu(args.reps, args.rounds)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
