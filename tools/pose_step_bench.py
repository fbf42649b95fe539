#!/usr/bin/env python
"""Time pose estimation from decoded frames: ``estimate_poses`` (eager) against ``GraphedPoseStep`` (one CUDA graph
per batch), per frame.

Workloads: YCB-shaped frames (FFB6D with 22 classes, depth completion, the refined vote) and LineMOD-shaped frames
(2 classes, raw depth, the two-class vote), each at B = 1 and B = 8, 480x640, N = 12800 points (the reference's
``config.n_sample_points``), 8 keypoints.  Frames come from ``synthetic.make_item_frame``.

Device time from CUDA events.  Each repeat runs ``--reps`` eager calls then ``--reps`` graphed calls of every
workload, so the two arms alternate; the median and range over repeats of the per-frame time are printed with the
card's name and power limit, read in the same run.  The eager arm is split into its three steps with events between
them (``build_ffb6d_inputs`` and the rgb cast; the forward, argmax and cloud; the vote), restated from
``estimate.py`` and checked to give ``estimate_poses``' outputs bit for bit; the eager total is ``estimate_poses``
itself.  The graphed outputs are checked against ``estimate_poses`` once per workload.

The weights are untrained (seeded), so the network's predictions are noise: every class is predicted somewhere and
the mean shift runs to its 301-round cap.  The vote share of these figures is therefore not what a deployment with
trained weights sees.  For context only, the reference's README reports 57 ms network + 18 ms post-processing =
75 ms per frame on an RTX 2080Ti with trained weights on LineMOD.

Run:  python tools/pose_step_bench.py [--repeats 5] [--reps 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, N, N_KPS = 480, 640, 480 * 640 // 24, 8
CAM_SCALE = {"ycb": 10000.0, "linemod": 1000.0}
N_CLS = {"ycb": 22, "linemod": 2}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception as e:                                   # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def workload(dataset, B, dev):
    import torch
    from ffb6d_b200 import estimate, ops
    from ffb6d_b200.model import FFB6D
    from ffb6d_b200.synthetic import INTRINSICS, make_item_frame
    torch.manual_seed(0)
    model = FFB6D(n_classes=N_CLS[dataset], n_pts=N, n_kps=N_KPS).to(dev).eval()
    if dataset == "ycb":
        fr = [make_item_frame(200 + b, n_kps=N_KPS, cls_ids=(1 + b % 7, 9, 14, 21), blobs=(1 + b % 7, 9, 14, 3))
              for b in range(B)]
        K = INTRINSICS["ycb_K1"]
    else:
        fr = [make_item_frame(300 + b, dataset="linemod", n_kps=N_KPS, cls_ids=(1,), blobs=(1,)) for b in range(B)]
        K = INTRINSICS["linemod"]
    frames = {"dpt": torch.from_numpy(np.stack([f["raw"] for f in fr])).to(dev),
              "rgb": torch.from_numpy(np.stack([f["rgb"] for f in fr])).to(dev),
              "nrm_map": torch.from_numpy(np.stack([f["nrm"] for f in fr])).to(dev)}
    rs = np.random.RandomState(7)
    if dataset == "ycb":
        mesh = {c: rs.uniform(-0.08, 0.08, (N_KPS + 1, 3)).astype(np.float32) for c in range(1, 22)}
        radius = list(rs.uniform(0.04, 0.12, 21))
    else:
        mesh, radius = rs.uniform(-0.08, 0.08, (N_KPS + 1, 3)).astype(np.float32), None
    table = estimate.vote_table(dataset, mesh, N_CLS[dataset], radius, dev)
    intr = ops.intrinsics_to_device(K, dev)                 # device intrinsics: no host copy per call
    kw = dict(dataset=dataset, cam_scale=CAM_SCALE[dataset], K=intr, mesh_kps=table)
    return model, frames, kw


def split_call(model, frames, kw, events):
    """estimate_poses' steps with an event after each (restated from estimate.py)."""
    import torch
    from ffb6d_b200 import pose
    from ffb6d_b200.schedule import build_ffb6d_inputs
    ds, table = kw["dataset"], kw["mesh_kps"]
    events[0].record()
    item = build_ffb6d_inputs(frames["dpt"], kw["cam_scale"], kw["K"], frames["rgb"], frames["nrm_map"], N,
                              fill=ds == "ycb")
    item["rgb"] = item["rgb"].to(torch.float32)
    events[1].record()
    with torch.no_grad():
        ep = model(item)
        mask = torch.max(ep["pred_rgbd_segs"], 1)[1]
        pcld = item["cld_rgb_nrm"][:, :3, :].permute(0, 2, 1).contiguous()
        events[2].record()
        if ds == "ycb":
            out = pose.cal_batch_poses(pcld, mask, ep["pred_ctr_ofs"], ep["pred_kp_ofs"], True, table.n_cls, True,
                                       mesh_kps=table)
        else:
            out = pose._vote(table, pcld, mask == 1, ep["pred_ctr_ofs"], ep["pred_kp_ofs"], True, False, False)
    events[3].record()
    return dict(zip(("present", "count", "kps", "poses", "valid"), tuple(out) + (item["valid"],)))


def same(a, b):
    import torch
    return all(torch.equal(a[k].contiguous().view(torch.uint8), b[k].contiguous().view(torch.uint8)) for k in a)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="calls per arm per repeat")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    import torch
    import ffb6d_b200 as F
    if not torch.cuda.is_available():
        raise SystemExit("pose_step_bench needs a GPU")
    dev = torch.device("cuda:0")
    name, power = card()
    shapes = [("ycb", 1), ("ycb", 8), ("linemod", 1), ("linemod", 8)]
    runs = {}
    for ds, B in shapes:
        model, frames, kw = workload(ds, B, dev)
        step = F.GraphedPoseStep(model, frames, **kw)
        eager = F.estimate_poses(model, frames, **kw)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        split = split_call(model, frames, kw, ev)
        graphed = {k: v.clone() for k, v in step(frames).items()}
        torch.cuda.synchronize()
        checks = dict(split_equals_eager=same(split, eager), graphed_equals_eager=same(graphed, eager))
        assert all(checks.values()), checks
        runs[(ds, B)] = dict(model=model, frames=frames, kw=kw, step=step, checks=checks,
                             eager=[], inputs=[], forward=[], vote=[], graphed=[],
                             n_present=int(eager["present"].sum()), valid=int(eager["valid"].sum()))
    for _ in range(args.repeats):
        for (ds, B), r in runs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            parts = np.zeros(3)
            tot = 0.0
            for _ in range(args.reps):
                t0.record()
                F.estimate_poses(r["model"], r["frames"], **r["kw"])
                t1.record()
                split_call(r["model"], r["frames"], r["kw"], ev)
                torch.cuda.synchronize()
                tot += t0.elapsed_time(t1)
                parts += [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])]
            r["eager"].append(tot / args.reps / B)
            for key, v in zip(("inputs", "forward", "vote"), parts / args.reps / B):
                r[key].append(float(v))
            t0.record()
            for _ in range(args.reps):
                r["step"](r["frames"])
            t1.record()
            torch.cuda.synchronize()
            r["graphed"].append(t0.elapsed_time(t1) / args.reps / B)

    def stat(v):
        return dict(median=round(float(np.median(v)), 3), min=round(float(np.min(v)), 3), max=round(float(np.max(v)), 3))

    results = []
    print("card: %s, power limit %s; %d repeats x %d calls per arm; ms per frame, median [min, max]"
          % (name, power, args.repeats, args.reps))
    for (ds, B), r in runs.items():
        row = dict(workload="%s_b%d" % (ds, B), dataset=ds, B=B, n_points=N, n_classes=N_CLS[ds], gpu=name,
                   power_limit=power, classes_voted=r["n_present"], **r["checks"],
                   **{k + "_ms_per_frame": stat(r[k]) for k in ("eager", "inputs", "forward", "vote", "graphed")})
        results.append(row)
        print("%-10s eager %7.2f [%.2f, %.2f]  (inputs %.2f, forward %.2f, vote %.2f)  graphed %7.2f [%.2f, %.2f]"
              % (row["workload"], *[row["eager_ms_per_frame"][k] for k in ("median", "min", "max")],
                 row["inputs_ms_per_frame"]["median"], row["forward_ms_per_frame"]["median"],
                 row["vote_ms_per_frame"]["median"], *[row["graphed_ms_per_frame"][k] for k in ("median", "min", "max")]))
    for row in results:
        print(json.dumps(row))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
