"""Surface normals on the device (``depth_normal``, DESIGN.md §4.30, §8): the kernel's device time, and what
``normals="device"`` costs a graphed step against the same step given a normal map.

    python tools/normal_bench.py [--repeats 3] [--reps 20] [--out results/normal_bench.json]

* ``depth_normal`` on B = 1, 8 and 32 LineMOD-shaped 480x640 millimetre maps (k_size 5, the datasets' arguments):
  device time from CUDA events around ``--reps`` calls, and the bytes the kernel must move (2 B of depth read and
  12 B of normals written per pixel) over that time.
* ``GraphedPoseStep`` on YCB-shaped frames at B = 1 and 8 (depth completion, 22 classes, 12 800 points): replay time
  per batch with ``normals="device"`` against ``normals="input"`` (a given ``nrm_map``).  With untrained weights the
  vote's work depends on the normals fed in (the frames' random ones, or fitted ones), so this pair shows the
  replay times, not the cost of the normals alone.
* ``GraphedFrameTrainStep`` at config 3 (LineMOD, B = 8, 2 classes, fused image head): wall ms per step, each window
  ending in one synchronise, both ways.

The arms alternate over ``--repeats`` windows; the median and range are reported with the card's name and power limit
read in the same run.  Weights are untrained and seeded."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

import ffb6d_b200 as F                                        # noqa: E402
from ffb6d_b200 import estimate, ops                          # noqa: E402
from ffb6d_b200.model import FFB6D                            # noqa: E402
from ffb6d_b200.synthetic import INTRINSICS, make_item_frame  # noqa: E402
from frame_batches import CAM_SCALE, K_OF, make_train_batch   # noqa: E402

H, W, N, N_KPS = 480, 640, 480 * 640 // 24, 8
BYTES_PER_PIXEL = 2 + 12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return dict(gpu=name, power_limit=power)


def summary(xs):
    s = sorted(xs)
    return dict(median=s[len(s) // 2], min=s[0], max=s[-1], windows=xs)


def kernel(repeats, reps):
    out = {}
    fr = [make_item_frame(400 + i, dataset="linemod") for i in range(32)]
    dev = torch.device("cuda")
    intr = ops.intrinsics_to_device(INTRINSICS["linemod"], dev)
    for B in (1, 8, 32):
        dpt = torch.from_numpy(np.stack([f["raw"] for f in fr[:B]])).to(dev)
        for _ in range(3):
            F.depth_normal(dpt, intr)
        ms = []
        for _ in range(repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                F.depth_normal(dpt, intr)
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1) / reps)
        s = summary(ms)
        out["B%d" % B] = dict(ms=s, bytes=B * H * W * BYTES_PER_PIXEL,
                              GB_per_s=B * H * W * BYTES_PER_PIXEL / (s["median"] * 1e-3) / 1e9)
    return out


def pose_step(B, repeats, reps):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = FFB6D(n_classes=22, n_pts=N, n_kps=N_KPS).to(dev).eval()
    fr = [make_item_frame(200 + b, n_kps=N_KPS, cls_ids=(1 + b % 7, 9, 14, 21), blobs=(1 + b % 7, 9, 14, 3))
          for b in range(B)]
    frames = {"dpt": torch.from_numpy(np.stack([f["raw"] for f in fr])).to(dev),
              "rgb": torch.from_numpy(np.stack([f["rgb"] for f in fr])).to(dev),
              "nrm_map": torch.from_numpy(np.stack([f["nrm"] for f in fr])).to(dev)}
    rs = np.random.RandomState(7)
    mesh = {c: rs.uniform(-0.08, 0.08, (N_KPS + 1, 3)).astype(np.float32) for c in range(1, 22)}
    table = estimate.vote_table("ycb", mesh, 22, list(rs.uniform(0.04, 0.12, 21)), dev)
    kw = dict(dataset="ycb", cam_scale=CAM_SCALE["ycb"], K=ops.intrinsics_to_device(K_OF["ycb"], dev), mesh_kps=table)
    no_nrm = {k: v for k, v in frames.items() if k != "nrm_map"}
    arms = {"input": (F.GraphedPoseStep(model, frames, **kw), frames),
            "device": (F.GraphedPoseStep(model, no_nrm, normals="device", **kw), no_nrm)}
    ms = {a: [] for a in arms}
    for _ in range(repeats):
        for a, (step, f) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                step(f)
            e1.record()
            e1.synchronize()
            ms[a].append(e0.elapsed_time(e1) / reps)
    return {a: dict(ms_per_batch=summary(v), captures=arms[a][0].captures) for a, v in ms.items()}


def frame_train_step(repeats, steps):
    batches = [make_train_batch(s, "linemod", 8, H, W, 2) for s in (1, 2)]
    kw = dict(dataset="linemod", cam_scale=CAM_SCALE["linemod"], K=K_OF["linemod"], n_points=N)
    arms = {}
    for arm in ("input", "device"):
        torch.manual_seed(0)
        model = FFB6D(n_classes=2, n_pts=N, n_kps=8, fused_image_head=True).cuda().train()
        opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device="cuda"), capturable=True)
        bs = batches if arm == "input" else [{k: v for k, v in b.items() if k != "nrm_map"} for b in batches]
        step = F.GraphedFrameTrainStep(model, opt, bs[0], normals=arm, **kw)
        for it in range(3):
            step(bs[it % 2], seed=it)
        arms[arm] = dict(step=step, batches=bs, ms=[])
    torch.cuda.synchronize()
    it = 0
    for _ in range(repeats):
        for a in arms.values():
            t0 = time.perf_counter()
            for _ in range(steps):
                loss, _ = a["step"](a["batches"][it % 2], seed=it)
                it += 1
            torch.cuda.synchronize()
            a["ms"].append((time.perf_counter() - t0) * 1e3 / steps)
            assert torch.isfinite(loss).item()
    return {k: dict(ms_per_step=summary(a["ms"]), captures=a["step"].captures) for k, a in arms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20, help="calls per window (kernel, pose step)")
    ap.add_argument("--steps", type=int, default=10, help="training steps per window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("normal_bench needs a GPU")
    res = dict(card(), depth_normal=kernel(args.repeats, args.reps),
               pose_step={"B%d" % B: pose_step(B, args.repeats, args.reps) for B in (1, 8)},
               frame_train_step_config3=frame_train_step(args.repeats, args.steps))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
