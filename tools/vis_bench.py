#!/usr/bin/env python
"""Time pose and label drawing: the demo's posed meshes and the trainers' label view, on the GPU and in the
reference's host loop.

Workloads:
* demo -- 8 frames x 5 objects x 2 621-point meshes at r = 1: ``vis.draw_poses`` (projection of every posed point
  and the drawing, one call) against the demo's loop of ``project_p3d`` + ``draw_p2ds`` per object;
* labels -- 8 frames x 12 288 points at r = 3: ``vis.view_labels`` (its label check is one host sync) against the
  trainers' ``view_labels`` per frame.

Device time: CUDA events around each call, ``--reps`` calls per repeat, repeats of the two workloads alternated;
the median and range over repeats are printed with the card's name and power limit, read in the same run.  The
reference's loop (``project_p3d`` / ``draw_p2ds`` / ``view_labels`` taken from its sources with ``ast``, cv2) runs
where its sources are present; it is a host number, timed with a host clock per frame over the same batch.  The
GPU images are checked against the numpy restatement (oracle/vis_oracle.py), and against the reference's images
when that loop ran; the sha256 of both sets of images are printed, so runs on two machines can be compared.
``--host-only`` runs the reference loop alone, without a GPU.

Run:  python tools/vis_bench.py [--reps 20] [--repeats 7] [--host-only]
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
from oracle import ref_loader as R, vis_oracle as O      # noqa: E402
import vis_cases as VC                                   # noqa: E402

B, N_OBJ, N_MESH, N_LABEL = 8, 5, 2621, 12288


def workloads():
    rs = np.random.RandomState(7)
    meshes = {c: VC.mesh(rs, N_MESH, np.float32) for c in range(1, 22)}
    ids = np.zeros((B, 22, 1), np.int32)
    present = np.zeros((B, 22), bool)
    poses = np.zeros((B, 22, 3, 4))
    for b in range(B):
        cls = rs.choice(np.arange(1, 22), N_OBJ, replace=False)
        ids[b, :N_OBJ, 0] = cls
        for c in cls:
            present[b, c] = True
            poses[b, c] = VC.pose_in_front(rs)
    rgb = rs.randint(0, 256, (B, 3, 480, 640)).astype(np.uint8)
    from ffb6d_b200.synthetic import make_frame
    clds = np.stack([make_frame(100 + b, intrinsics="ycb_K1")["cld"].T for b in range(B)])
    labels = rs.randint(0, 22, (B, N_LABEL))
    return dict(meshes=meshes, ids=ids, present=present, poses=poses, rgb=rgb, clds=clds, labels=labels)


def demo_lists(w, b):
    pred = np.flatnonzero(w["present"][b])
    return pred, [w["poses"][b, c] for c in pred]


def host_loop(w, fns):
    """The reference's loops, per frame; returns (demo seconds, labels seconds, demo images, label images)."""
    import torch
    t0 = time.perf_counter()
    demo = [O.demo_draw(w["rgb"][b].astype(np.float32), w["ids"][b], *demo_lists(w, b), w["meshes"], VC.K_YCB, "ycb",
                        -1, fns) for b in range(B)]
    t1 = time.perf_counter()
    lab = [fns["view_labels"](torch.from_numpy(w["rgb"][b:b + 1]), torch.from_numpy(w["clds"][b]),
                              torch.from_numpy(w["labels"][b]), VC.K_YCB) for b in range(B)]
    t2 = time.perf_counter()
    return t1 - t0, t2 - t1, np.stack(demo), np.stack(lab)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--host-only", action="store_true")
    a = ap.parse_args()
    w = workloads()
    res = {"frames": B, "objects": N_OBJ, "mesh_points": N_MESH, "label_points": N_LABEL}
    host = None
    if R.reference_sources_present():
        host = host_loop(w, O.reference_functions())
        res["host_loop_demo_ms"] = host[0] * 1e3
        res["host_loop_labels_ms"] = host[1] * 1e3
        res["host_loop_demo_sha256"], res["host_loop_labels_sha256"] = VC.sha(host[2]), VC.sha(host[3])
    else:
        res["host_loop"] = "not run: the reference's sources are absent"
    if a.host_only:
        print(json.dumps(res))
        return

    import torch
    from ffb6d_b200 import ops, pose, vis
    dev = torch.device("cuda:0")
    res["card"], res["power_limit"] = card()
    table = pose.MeshTable(w["meshes"], dev, torch.float64)
    ids = torch.from_numpy(w["ids"]).to(dev)
    present = torch.from_numpy(w["present"]).to(dev)
    poses = torch.from_numpy(w["poses"]).to(dev)
    K = torch.from_numpy(VC.K_YCB).to(dev)
    colors = torch.tensor([vis.get_label_color(c, n_obj=22, mode=2) for c in range(22)], dtype=torch.uint8,
                          device=dev)
    base = torch.from_numpy(w["rgb"]).to(dev).permute(0, 2, 3, 1).flip(-1).contiguous()
    img = base.clone()
    ws = ops.draw_p2ds_workspace(img)
    rgb = torch.zeros((B, 3, 480, 640), device=dev)
    clds = torch.from_numpy(w["clds"]).to(dev)
    labels = torch.from_numpy(w["labels"]).to(dev)

    def demo():
        return vis.draw_poses(img, table, ids, present, poses, K, colors, ws=ws)

    def labels_view():
        return vis.view_labels(rgb, clds, labels, K)

    # outputs first: one call on fresh images, against the restatement (and the reference's images)
    img.copy_(base)
    got_demo = demo().cpu().numpy()
    got_lab = labels_view().cpu().numpy()
    want_demo = np.stack([O.demo_draw(w["rgb"][b].astype(np.float32), w["ids"][b], *demo_lists(w, b), w["meshes"],
                                      VC.K_YCB, "ycb") for b in range(B)])
    want_lab = np.stack([O.view_labels(480, 640, w["clds"][b].T, w["labels"][b], VC.K_YCB) for b in range(B)])
    res["demo_equal_restatement"] = bool(np.array_equal(got_demo, want_demo))
    res["labels_equal_restatement"] = bool(np.array_equal(got_lab, want_lab))
    res["gpu_demo_sha256"], res["gpu_labels_sha256"] = VC.sha(got_demo), VC.sha(got_lab)
    if host is not None:
        res["demo_equal_host_loop"] = bool(np.array_equal(got_demo, host[2]))
        res["labels_equal_host_loop"] = bool(np.array_equal(got_lab, host[3]))

    for _ in range(3):
        demo()
        labels_view()
    torch.cuda.synchronize()
    times = {"demo": [], "labels": []}
    for _ in range(a.repeats):
        for name, fn in (("demo", demo), ("labels", labels_view)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.reps)
    for name, t in times.items():
        res["gpu_%s_ms_median" % name] = float(np.median(t))
        res["gpu_%s_ms_range" % name] = [float(min(t)), float(max(t))]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
