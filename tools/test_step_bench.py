"""The reference's test loop per batch: the eager chain (``build_ffb6d_item``, a ``GraphedEvalStep`` replay,
``TorchEval.eval_pose_parallel`` and ``model_fn``'s per-batch ``.item()`` of every loss) against one
``GraphedTestStep`` replay (DESIGN.md §4.29, §8).

    python tools/test_step_bench.py [--repeats 3] [--steps 5] [--out results/test_step_bench.json]

Workloads: YCB (B = 8, 22 classes, depth completion, a camera matrix per frame) and LineMOD (B = 8, 2 classes), both
480x640 with 12 800 points.  The arms run alternated, ``--repeats`` windows of ``--steps`` batches each, every window
ending in one synchronise (the graphed arm's window starts with ``reset()``).  Reported per arm: wall ms per batch
(median and spread over the windows) and the package's host launches per batch; with the card's name and power limit
read in the same run.  Weights are untrained, so the vote runs to its iteration cap; the batch alternates between
two seeded batches."""
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
from ffb6d_b200 import _lib, pose                             # noqa: E402
from ffb6d_b200.model import FFB6D                            # noqa: E402
from frame_batches import CAM_SCALE, K_OF, make_train_batch   # noqa: E402

N_POINTS = 480 * 640 // 24
N_KPS = 8
TEST_KEYS = ("dpt", "rgb", "labels", "nrm_map", "K", "RTs", "kp_3ds", "ctr_3ds", "cls_ids", "obj_cls", "obj_kps",
             "obj_ctr")
WORKLOADS = {
    "ycb_B8": dict(dataset="ycb", B=8, n_cls=22, per_frame_K=True),
    "linemod_B8": dict(dataset="linemod", B=8, n_cls=2, per_frame_K=False),
}
LM_OBJ = 1


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return dict(gpu=name, power_limit=power)


def tables(ds, n_cls):
    rs = np.random.RandomState(9)
    ids = range(1, n_cls) if ds == "ycb" else (LM_OBJ,)
    kps = {c: rs.uniform(-0.08, 0.08, (N_KPS + 1, 3)).astype(np.float32) for c in ids}
    pts = {c: rs.uniform(-0.08, 0.08, (2000, 3)).astype(np.float32) for c in ids}
    return pts, kps, (list(rs.uniform(0.04, 0.12, 21)) if ds == "ycb" else None)


def run(name, cfg, repeats, steps, warmup):
    ds, B = cfg["dataset"], cfg["B"]
    batches = [{k: v for k, v in make_train_batch(s, ds, B, 480, 640, cfg["n_cls"], per_frame_K=cfg["per_frame_K"])
                .items() if k in TEST_KEYS} for s in (1, 2)]
    torch.manual_seed(0)
    model = FFB6D(n_classes=cfg["n_cls"], n_pts=N_POINTS, n_kps=N_KPS).cuda().eval()
    pts, kps, radius = tables(ds, cfg["n_cls"])
    sym = (13, 16, 19, 20, 21) if ds == "ycb" else ()
    obj = LM_OBJ if ds == "linemod" else 0
    fill = ds == "ycb"

    def item_of(b):
        K = F.ops._frame_intrinsics(b["K"]) if "K" in b else K_OF[ds]
        it = F.build_ffb6d_item(b["dpt"], CAM_SCALE[ds], K, b["rgb"], b["labels"], b["nrm_map"], b, N_POINTS,
                                fill=fill)
        it["rgb"] = it["rgb"].float()
        return it

    te = pose.TorchEval(pts, kps, radius, sym, n_cls=cfg["n_cls"] if ds == "ycb" else 22)
    ev = F.GraphedEvalStep(model, item_of(batches[0]), warmup=warmup)

    def eager(b):
        item = item_of(b)
        ep, loss, info = ev(item)
        {k: v.item() for k, v in info.items()}                 # model_fn's loss_dict / acc_dict
        cld = item["cld_rgb_nrm"][:, :3, :].permute(0, 2, 1).contiguous()
        te.eval_pose_parallel(cld, item["rgb"], torch.max(ep["pred_rgbd_segs"], 1)[1], ep["pred_ctr_ofs"],
                              item["ctr_targ_ofst"], item["labels"], 0, item["cls_ids"], item["RTs"],
                              ep["pred_kp_ofs"], item["kp_3ds"], item["ctr_3ds"], min_cnt=1, use_ctr_clus_flter=True,
                              use_ctr=True, obj_id=obj, ds=ds)
        return loss

    kw = dict(dataset=ds, cam_scale=CAM_SCALE[ds], K=K_OF[ds], mesh_pts=pts, mesh_kps=kps, cls_radius=radius,
              sym_cls_ids=sym, n_points=N_POINTS, capacity=max(warmup, steps) * B)
    if ds == "linemod":
        kw["obj_id"] = LM_OBJ
    step = F.GraphedTestStep(model, batches[0], warmup=warmup, **kw)
    arms = {"eager_item+GraphedEvalStep+TorchEval": dict(call=eager, start=lambda: None),
            "GraphedTestStep": dict(call=lambda b: step(b)[1], start=step.reset)}
    for a in arms.values():
        a["start"]()
        for it in range(warmup):
            a["call"](batches[it % 2])
        a.update(ms=[], launches=[])
    torch.cuda.synchronize()
    for _ in range(repeats):
        for arm, a in arms.items():
            a["start"]()
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            t0 = time.perf_counter()
            for it in range(steps):
                loss = a["call"](batches[it % 2])
            torch.cuda.synchronize()
            a["ms"].append((time.perf_counter() - t0) * 1e3 / steps)
            a["launches"].append((_lib.launch_count() - n0) / steps)
            assert torch.isfinite(loss).item()
    res = step.summary(100.0)
    out = {}
    for arm, a in arms.items():
        ms = sorted(a["ms"])
        out[arm] = dict(ms_per_batch_median=ms[len(ms) // 2], ms_per_batch_min=ms[0], ms_per_batch_max=ms[-1],
                        ms_per_batch_windows=a["ms"], launches_per_batch=a["launches"][-1])
    return dict(workload=name, B=B, n_classes=cfg["n_cls"], dataset=ds, captures=step.captures,
                objects_last_run=len(res["add_dis_lst"][0]), **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "test_step_bench needs a GPU"
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
