#!/usr/bin/env python
"""Device time of the textured keypoint stages (DESIGN.md §4.32).

    python tools/orb_bench.py [--reps 20] [--out results/orb_bench.json]
    python tools/orb_bench.py --cpu                  # the CPU comparison: cv2 ORB + the numpy lift (needs cv2)

GPU: ``orb_detect`` at 480x640 for B = 9 (one object's sphere of views) and B = 189 (21 objects x 9 views), and the
whole ``textured_kp3ds`` of the ape (render, detect, lift), each timed with CUDA events over ``--reps`` calls after a
warm-up, with the card's name and power limit.  ``--cpu`` times ``cv2.ORB_create().detect`` plus
oracle/orb_oracle.py's lift on the ape's 9 views on the machine it runs on (a CPU number, not a GPU one).
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


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def gpu(reps):
    import torch
    import ffb6d_b200 as F
    from ffb6d_b200 import objinfo
    from ffb6d_b200.render import RenderMeshTable
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(xyz)))
    _, img, _ = F.render_rgbd(table, np.zeros((9, 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                              np.ones((9, 1), np.uint8), objinfo.TOOL_K, 480, 640)
    res = card()
    res["orb_detect_ms"] = {str(B): timed(lambda x=img.repeat(B // 9, 1, 1, 1).contiguous(): F.orb_detect(x), reps)
                            for B in (9, 189)}
    radius = objinfo.get_r(objinfo.get_3D_bbox(xyz))
    res["textured_kp3ds_ape_ms"] = timed(lambda: objinfo.textured_kp3ds(table, 0, radius=radius), reps)
    return res


def cpu(reps):
    import cv2
    from oracle import orb_oracle as O
    from ffb6d_b200 import objinfo
    xyz, K, H, W, radius = OC.ape_setup()
    poses = objinfo.sphere_poses(radius)
    frames = [OC.ape_render(RT) for RT in poses]
    orb = cv2.ORB_create()

    def run():
        for (depth, rgb), RT in zip(frames, poses):
            kps = orb.detect(np.ascontiguousarray(rgb[..., ::-1]), None)
            O.lift(np.array([k.pt for k in kps], np.float32).reshape(-1, 2), depth, K, RT)
    run()
    t = time.perf_counter()
    for _ in range(reps):
        run()
    return {"cpu_ape_9_views_ms": (time.perf_counter() - t) / reps * 1e3, "cv2": cv2.__version__,
            "note": "build-container CPU number: cv2 ORB detect + numpy lift, renders excluded"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    res = cpu(args.reps) if args.cpu else gpu(args.reps)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
