"""Training from decoded frames: the eager ``build_ffb6d_train_item`` followed by a ``GraphedTrainStep`` replay,
against one ``GraphedFrameTrainStep`` replay (DESIGN.md §4.28, §8).

    python tools/frame_step_bench.py [--repeats 3] [--steps 20] [--out results/frame_step_bench.json]

Workloads: LineMOD-shaped config 3 (FFB6D, B = 8, 2 classes, fused image head, 480x640, 12 800 points) and
YCB-shaped config 4 (B = 4, 22 classes, depth completion, a camera matrix per frame).  The arms run alternated,
``--repeats`` times ``--steps`` steps each, every window ending in one synchronise.  Reported per arm: wall ms per
step (median and spread over the windows) and the package's host launches per step; with the card's name and power
limit read in the same run.  Weights are untrained; the batch alternates between two seeded batches."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

import ffb6d_b200 as F                                        # noqa: E402
from ffb6d_b200 import _lib                                   # noqa: E402
from ffb6d_b200.model import FFB6D                            # noqa: E402
from frame_batches import CAM_SCALE, K_OF, make_train_batch   # noqa: E402

N_POINTS = 480 * 640 // 24
WORKLOADS = {
    "config3_linemod_B8": dict(dataset="linemod", B=8, n_cls=2, per_frame_K=False),
    "config4_ycb_B4": dict(dataset="ycb", B=4, n_cls=22, per_frame_K=True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return dict(gpu=name, power_limit=power)


def run(name, cfg, repeats, steps, warmup):
    ds = cfg["dataset"]
    batches = [make_train_batch(s, ds, cfg["B"], 480, 640, cfg["n_cls"], per_frame_K=cfg["per_frame_K"])
               for s in (1, 2)]
    kw = dict(dataset=ds, cam_scale=CAM_SCALE[ds], K=K_OF[ds], n_points=N_POINTS)
    arms = {}
    for arm in ("eager_item+graphed_step", "graphed_frame_step"):
        torch.manual_seed(0)
        model = FFB6D(n_classes=cfg["n_cls"], n_pts=N_POINTS, n_kps=8, fused_image_head=True).cuda().train()
        opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device="cuda"), capturable=True)
        if arm == "graphed_frame_step":
            step = F.GraphedFrameTrainStep(model, opt, batches[0], warmup=warmup, **kw)
            call = (lambda st: lambda b, it: st(b, seed=it))(step)
        else:
            step = F.GraphedTrainStep(model, opt, F.build_ffb6d_train_item(batches[0], seed=0, **kw), warmup=warmup)
            call = (lambda st: lambda b, it: st(F.build_ffb6d_train_item(b, seed=it, **kw)))(step)
        for it in range(warmup):
            call(batches[it % 2], it)
        arms[arm] = dict(call=call, step=step, ms=[], launches=[])
    torch.cuda.synchronize()
    it = 0
    for _ in range(repeats):
        for arm, a in arms.items():
            n0 = _lib.launch_count()
            t0 = time.perf_counter()
            for _ in range(steps):
                loss, _ = a["call"](batches[it % 2], it)
                it += 1
            torch.cuda.synchronize()
            a["ms"].append((time.perf_counter() - t0) * 1e3 / steps)
            a["launches"].append((_lib.launch_count() - n0) / steps)
            assert torch.isfinite(loss).item()
    out = {}
    for arm, a in arms.items():
        ms = sorted(a["ms"])
        out[arm] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_min=ms[0], ms_per_step_max=ms[-1],
                        ms_per_step_windows=a["ms"], launches_per_step=a["launches"][-1],
                        captures=a["step"].captures)
    return dict(workload=name, B=cfg["B"], n_classes=cfg["n_cls"], dataset=ds, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "frame_step_bench needs a GPU"
    res = dict(card(), repeats=args.repeats, steps=args.steps, results=[])
    for name in args.workloads.split(","):
        r = run(name, WORKLOADS[name], args.repeats, args.steps, args.warmup)
        print(json.dumps(r), flush=True)
        res["results"].append(r)
        torch.cuda.empty_cache()
    res.update(card_after=card())
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
