#!/usr/bin/env python
"""Time ADD / ADD-S scoring of a test batch three ways:

(a) ``pose.add_adds``: every object of the batch in one ``ffb6d_pose_add_adds`` launch (CUDA events over
    ``--repeats`` calls);
(b) the reference's algorithm as ``eval_metric`` runs it, restated here in stock torch ops (the reference's tree is not
    needed): per object two ``torch.mm``, the N x N ``repeat`` / ``norm`` / ``min`` of ``cal_adds_cuda``, the
    ``cal_add_cuda`` mean, and two ``.item()`` host syncs (wall clock, ending in those syncs);
(c) ``TorchEval.eval_pose_parallel`` on the same batch of seeded frames (``synthetic.make_pose_frame``), with the
    time of its one scoring call shown apart from the voting.

Arms (a) and (b) are alternated per repeat after a warm-up of each, and their results compared.  Batches: YCB-test-like
(8 frames x 5 objects, 2 621-point meshes) and LineMOD (8 frames x 1 object, 2 000 points).  Prints the GPU's name
and power limit with one JSON line.

    python tools/pose_eval_bench.py [--repeats 20] [--out pose_eval_bench.json]
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

# (name, frames, objects per frame, mesh points, distinct meshes)
BATCHES = [("ycb_8x5_2621", 8, 5, 2621, 21), ("lm_8x1_2000", 8, 1, 2000, 1)]


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def torch_reference(torch, pts, pred, gt):
    """``cal_add_cuda`` + ``cal_adds_cuda`` of one object in stock torch ops, and their two ``.item()``."""
    N = pts.shape[0]
    pd = torch.mm(pts, pred[:, :3].transpose(1, 0)) + pred[:, 3]
    g = torch.mm(pts, gt[:, :3].transpose(1, 0)) + gt[:, 3]
    add = torch.mean(torch.norm(pd - g, dim=1))
    pdr = pd.view(1, N, 3).repeat(N, 1, 1)
    gtr = g.view(N, 1, 3).repeat(1, N, 1)
    adds = torch.mean(torch.min(torch.norm(pdr - gtr, dim=2), dim=1)[0])
    return add.item(), adds.item()


def make_batch(rs, B, K, n, n_mesh):
    meshes = {c: rs.uniform(-0.1, 0.1, (n, 3)).astype(np.float32) for c in range(1, n_mesh + 1)}
    cls = rs.randint(1, n_mesh + 1, B * K)
    gt = []
    for _ in range(B * K):
        R = np.linalg.qr(rs.normal(size=(3, 3)))[0]
        gt.append(np.concatenate((R * np.sign(np.linalg.det(R)), rs.uniform(-0.3, 0.3, (3, 1)) + [[0], [0], [1]]), 1))
    gt = np.asarray(gt, np.float32)
    pred = (gt + rs.normal(0, 0.005, gt.shape)).astype(np.float32)
    return meshes, cls, pred, gt


def bench_scoring(torch, pose, name, B, K, n, n_mesh, repeats):
    rs = np.random.RandomState(n + K)
    meshes, cls, pred, gt = make_batch(rs, B, K, n, n_mesh)
    table = pose.MeshTable(meshes)
    dev = table.device
    pr, g = torch.as_tensor(pred, device=dev), torch.as_tensor(gt, device=dev)
    dmesh = {c: torch.as_tensor(m, device=dev) for c, m in meshes.items()}
    add, adds = pose.add_adds(table, cls, pr, g)
    want = np.array([torch_reference(torch, dmesh[c], pr[m], g[m]) for m, c in enumerate(cls)])
    got = torch.stack((add, adds), 1).cpu().numpy()
    max_diff = float(np.abs(got - want).max())
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    t_dev, t_ref = [], []
    for _ in range(repeats):
        ev[0].record()
        for _ in range(10):
            pose.add_adds(table, cls, pr, g)
        ev[1].record()
        torch.cuda.synchronize()
        t_dev.append(ev[0].elapsed_time(ev[1]) / 10)
        t0 = time.perf_counter()
        for m, c in enumerate(cls):
            torch_reference(torch, dmesh[c], pr[m], g[m])
        t_ref.append((time.perf_counter() - t0) * 1e3)
    return dict(batch=name, objects=B * K, points=n, add_adds_ms=float(np.median(t_dev)),
                add_adds_ms_range=[float(min(t_dev)), float(max(t_dev))], torch_ref_ms=float(np.median(t_ref)),
                torch_ref_ms_range=[float(min(t_ref)), float(max(t_ref))],
                speedup=float(np.median(t_ref) / np.median(t_dev)), max_abs_diff_m=max_diff)


def bench_torch_eval(torch, pose, synthetic, name, B, K, n, repeats):
    """TorchEval.eval_pose_parallel over B copies of one seeded frame; its scoring call timed on its own."""
    fr = synthetic.make_pose_frame(7, n_kps=8)
    rs = np.random.RandomState(8)
    ids = (1, 2, 3, 4, 5)[:K] if name.startswith("ycb") else (1,)
    meshes = {c: rs.uniform(-0.08, 0.08, (n, 3)).astype(np.float32) for c in range(1, 6)}
    kps = dict(fr["mesh"])
    kps[5] = fr["mesh"][2]
    dev = torch.device("cuda", torch.cuda.current_device())
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=dev)
    cls_ids = np.zeros((B, len(ids), 1), np.int64)
    cls_ids[:, :, 0] = ids
    RTs = np.stack([[fr["poses"][min(c, 4)] for c in ids]] * B).astype(np.float32)
    args = dict(pclds=t(np.stack([fr["pcld"]] * B)), masks=t(np.stack([fr["mask"]] * B)),
                ctr=t(np.stack([fr["ctr_of"]] * B)), kp=t(np.stack([fr["kp_of"]] * B)), cls_ids=t(cls_ids), RTs=t(RTs),
                gt_kps=t(np.zeros((B, len(ids), 8, 3), np.float32)), gt_ctrs=t(np.zeros((B, len(ids), 3), np.float32)))
    ds = "ycb" if name.startswith("ycb") else "linemod"
    orig = pose._score
    spent = []

    def timed_score(*a):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = orig(*a)
        spent.append((time.perf_counter() - t0) * 1e3)
        return r

    pose._score = timed_score
    try:
        totals = []
        for i in range(repeats + 1):
            te = pose.TorchEval(meshes, kps if ds == "ycb" else {1: fr["mesh"][1]}, fr["cls_radius"], ())
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            te.eval_pose_parallel(args["pclds"], None, args["masks"], args["ctr"], None, [None] * B, 0,
                                  args["cls_ids"], args["RTs"], args["kp"], args["gt_kps"], args["gt_ctrs"],
                                  obj_id=1, ds=ds)
            torch.cuda.synchronize()
            if i:                                       # the first run is the warm-up
                totals.append((time.perf_counter() - t0) * 1e3)
    finally:
        pose._score = orig
    score = spent[1:]
    return dict(batch=name, eval_pose_parallel_ms=float(np.median(totals)), scoring_ms=float(np.median(score)),
                voting_ms=float(np.median(totals) - np.median(score)), objects=B * len(ids))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from ffb6d_b200 import pose, synthetic
    if not torch.cuda.is_available():
        raise SystemExit("pose_eval_bench needs a CUDA device")
    info = gpu_info()
    print("GPU: %s" % info)
    res = {"gpu": info, "scoring": [], "torch_eval": []}
    for name, B, K, n, n_mesh in BATCHES:
        r = bench_scoring(torch, pose, name, B, K, n, n_mesh, a.repeats)
        print("%-14s %3d objects: add_adds %.3f ms, torch reference %.2f ms (%.0fx), max |diff| %.2e m"
              % (name, r["objects"], r["add_adds_ms"], r["torch_ref_ms"], r["speedup"], r["max_abs_diff_m"]))
        res["scoring"].append(r)
    for name, B, K, n, _ in BATCHES:
        r = bench_torch_eval(torch, pose, synthetic, name, B, K, n, max(3, a.repeats // 4))
        print("%-14s eval_pose_parallel %.1f ms: voting %.1f ms, scoring %.2f ms"
              % (name, r["eval_pose_parallel_ms"], r["voting_ms"], r["scoring_ms"]))
        res["torch_eval"].append(r)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
