#!/usr/bin/env python
"""Time ADD / ADD-S scoring of a test batch two ways:

(a) ``pose.add_adds``: every object of the batch in one ``ffb6d_pose_add_adds`` launch (CUDA events over
    ``--repeats`` calls);
(b) the reference's algorithm as ``eval_metric`` runs it, restated here in stock torch ops (the reference's tree is not
    needed): per object two ``torch.mm``, the N x N ``repeat`` / ``norm`` / ``min`` of ``cal_adds_cuda``, the
    ``cal_add_cuda`` mean, and two ``.item()`` host syncs (wall clock, ending in those syncs);

Arms (a) and (b) are alternated per repeat after a warm-up of each, and their results compared.  Batches: YCB-test-like
(8 frames x 5 objects, 2 621-point meshes) and LineMOD (8 frames x 1 object, 2 000 points).

Then time the voting of a test batch three ways, alternated per repeat: the parent commit's per-object loop of
``mean_shift_fit`` / ``best_fit_transform`` (restated here), one ``pose.cal_batch_poses`` call, and
``TorchEval.eval_pose_parallel`` end to end; the loop and the batched call are compared bitwise, and one batched call
is profiled per kernel (``torch.profiler``).  Batches: 8 frames of ``synthetic.make_pose_frame`` (2 150 points) and
1 and 8 frames of ``synthetic.make_pose_batch`` (12 288 points, 22 classes, 5 objects).  Prints the GPU's name and
power limit with one JSON line.

    python tools/pose_eval_bench.py [--repeats 20] [--out pose_eval_bench.json] [--profile-dir DIR]
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


def loop_frame(torch, F, pcld, mask, ctr_of, kp_of, mesh, thr, use_ctr=True, flt=True):
    """One frame the way the parent commit voted it: one object at a time through ``mean_shift_fit`` and
    ``best_fit_transform``, with its host syncs (the class list, each class's count, each result's copy), and the
    refinement in the reference's difference form (numpy float32, first minimum).  Returns the op's four rows."""
    n_kps, N = kp_of.shape[:2]
    n_cls, R = thr.shape[0], n_kps + int(use_ctr)
    pred_ctr, pred_kp = pcld - ctr_of[0], pcld[None] - kp_of
    ids = np.unique(mask[mask > 0].cpu().numpy()).tolist()
    if flt and ids:
        ctrs, _, _ = F.mean_shift_fit(pred_ctr[None].expand(len(ids), N, 3).contiguous(),
                                      torch.stack([mask == c for c in ids]), 0.04, 300)
        pc, cc = pred_ctr.cpu().numpy(), ctrs.cpu().numpy()
        d = np.sqrt(((pc[:, None, :] - cc[None]) ** 2).sum(2, dtype=np.float32))
        j = d.argmin(1)
        near = np.asarray(ids)[j]
        upd = (mask.cpu().numpy() > 0) & (d[np.arange(N), j] < thr[near])
        mask = torch.where(torch.from_numpy(upd).to(mask.device), torch.from_numpy(near).to(mask.device), mask)
    present = torch.zeros(n_cls, dtype=torch.bool)
    present[ids] = True
    count = torch.zeros(n_cls, dtype=torch.int32)
    kps, poses = torch.zeros(n_cls, R, 3), torch.zeros(n_cls, 3, 4, dtype=torch.float64)
    for c in ids:
        msk = mask == c
        count[c] = int(msk.sum())
        if count[c] == 0:
            poses[c] = torch.eye(3, 4, dtype=torch.float64)
            continue
        ctr, lab, _ = F.mean_shift_fit(pred_ctr[None], msk, 0.04, 300)
        lab = lab[0]
        if flt and not lab.any():
            lab[int(torch.nonzero(msk)[0])] = True
        kp, _, _ = F.mean_shift_fit(pred_kp, lab if flt else msk, 0.04, 300)
        kpc = torch.cat((kp, ctr)) if use_ctr else kp
        kps[c] = kpc.cpu()
        poses[c] = F.best_fit_transform(mesh[c, :R], kpc).cpu()
    return present, count, kps, poses


def voting_batches(synthetic):
    """name -> (numpy batch, mesh keypoints, radii, n_cls): the 2 150-point frames of make_pose_frame and full-size
    make_pose_batch frames (N = 12288, 22 classes, 5 objects)."""
    out = {}
    frs = [synthetic.make_pose_frame(7 + b, n_kps=8) for b in range(8)]
    small = {k: np.stack([f[k] for f in frs]) for k in ("pcld", "mask", "ctr_of", "kp_of")}
    out["frames_8x2150"] = (small, frs[0]["mesh"], frs[0]["cls_radius"], 5)
    for B in (1, 8):
        bt = synthetic.make_pose_batch(11, B)
        out["full_%dx12288" % B] = (bt, bt["mesh"], bt["cls_radius"], 22)
    return out


def bench_voting(torch, F, pose, name, batch, mesh, radius, n_cls, repeats):
    """Arms alternated per repeat after a warm-up: (a) the parent's per-object loop, (b) one cal_batch_poses call,
    (c) eval_pose_parallel end to end (voting + scoring of every object); (a) and (b) compared bitwise."""
    dev = torch.device("cuda", torch.cuda.current_device())
    t = {k: torch.as_tensor(np.ascontiguousarray(batch[k]), device=dev) for k in ("pcld", "mask", "ctr_of", "kp_of")}
    B = t["pcld"].shape[0]
    table = pose.VoteTable(mesh, n_cls, radius, dev)
    thr = table.refine_thr.cpu().numpy()
    ids = [sorted(set(np.unique(m[m > 0]).tolist()))[:5] for m in batch["mask"]]
    n_obj = max(len(i) for i in ids)
    cls_ids = np.zeros((B, n_obj, 1), np.int64)
    for b, i in enumerate(ids):
        cls_ids[b, :len(i), 0] = i
    rs = np.random.RandomState(5)
    meshes = {c: rs.uniform(-0.08, 0.08, (2621, 3)).astype(np.float32) for c in range(1, n_cls)}
    RTs = torch.as_tensor(np.tile(np.eye(3, 4, dtype=np.float32), (B, n_obj, 1, 1)), device=dev)
    gt_kps = torch.zeros(B, n_obj, batch["kp_of"].shape[1], 3, device=dev)
    cls_t = torch.as_tensor(cls_ids, device=dev)

    def arm_a():
        return [loop_frame(torch, F, *(t[k][b] for k in ("pcld", "mask", "ctr_of", "kp_of")), table.kps, thr)
                for b in range(B)]

    def arm_b():
        out = pose.cal_batch_poses(t["pcld"], t["mask"], t["ctr_of"], t["kp_of"], True, n_cls, True, mesh_kps=table)
        torch.cuda.synchronize()
        return out

    def arm_c():
        te = pose.TorchEval(meshes, mesh, radius, (), n_cls=n_cls)
        te.eval_pose_parallel(t["pcld"], None, t["mask"], t["ctr_of"], None, None, 0, cls_t, RTs, t["kp_of"], gt_kps,
                              None)
        torch.cuda.synchronize()

    loop, batched = arm_a(), arm_b()
    arm_c()
    same = all(torch.equal(x[b].cpu().contiguous().view(torch.uint8), w.to(x.dtype).contiguous().view(torch.uint8))
               for b in range(B) for x, w in zip(batched, loop[b]))
    times = {"loop": [], "batched": [], "eval_pose_parallel": []}
    for _ in range(repeats):
        for key, fn in (("loop", arm_a), ("batched", arm_b), ("eval_pose_parallel", arm_c)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            times[key].append((time.perf_counter() - t0) * 1e3)
    med = {k: float(np.median(v)) for k, v in times.items()}
    return dict(batch=name, frames=B, points=int(t["pcld"].shape[1]), objects=int(sum(len(i) for i in ids)),
                loop_ms=med["loop"], batched_ms=med["batched"], eval_pose_parallel_ms=med["eval_pose_parallel"],
                ranges={k: [float(min(v)), float(max(v))] for k, v in times.items()},
                speedup=med["loop"] / med["batched"], bitwise_equal=bool(same))


def profile_voting(torch, pose, name, batch, mesh, radius, n_cls, out_dir):
    """Per-kernel CUDA times of one cal_batch_poses call (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda", torch.cuda.current_device())
    t = {k: torch.as_tensor(np.ascontiguousarray(batch[k]), device=dev) for k in ("pcld", "mask", "ctr_of", "kp_of")}
    table = pose.VoteTable(mesh, n_cls, radius, dev)
    run = lambda: pose.cal_batch_poses(t["pcld"], t["mask"], t["ctr_of"], t["kp_of"], True, n_cls, True,
                                       mesh_kps=table)
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0):
            rows[e.key] = dict(calls=e.count, ms=getattr(e, "self_device_time_total", 0.0) / 1e3)
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "vote_%s.json" % name))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile-dir", default=None, help="write a chrome trace of each voting batch here")
    a = ap.parse_args()
    import torch
    import ffb6d_b200 as F
    from ffb6d_b200 import pose, synthetic
    if not torch.cuda.is_available():
        raise SystemExit("pose_eval_bench needs a CUDA device")
    info = gpu_info()
    print("GPU: %s" % info)
    res = {"gpu": info, "scoring": []}
    for name, B, K, n, n_mesh in BATCHES:
        r = bench_scoring(torch, pose, name, B, K, n, n_mesh, a.repeats)
        print("%-14s %3d objects: add_adds %.3f ms, torch reference %.2f ms (%.0fx), max |diff| %.2e m"
              % (name, r["objects"], r["add_adds_ms"], r["torch_ref_ms"], r["speedup"], r["max_abs_diff_m"]))
        res["scoring"].append(r)
    res["voting"], res["voting_kernels"] = [], {}
    for name, (batch, mesh, radius, n_cls) in voting_batches(synthetic).items():
        r = bench_voting(torch, F, pose, name, batch, mesh, radius, n_cls, max(3, a.repeats // 4))
        print("%-14s %2d objects: per-object loop %.1f ms, cal_batch_poses %.1f ms (%.1fx), eval_pose_parallel "
              "%.1f ms, bitwise equal %s" % (name, r["objects"], r["loop_ms"], r["batched_ms"], r["speedup"],
                                             r["eval_pose_parallel_ms"], r["bitwise_equal"]))
        res["voting"].append(r)
        res["voting_kernels"][name] = profile_voting(torch, pose, name, batch, mesh, radius, n_cls, a.profile_dir)
        for k, v in sorted(res["voting_kernels"][name].items(), key=lambda kv: -kv[1]["ms"])[:8]:
            print("    %-60s %3d calls %8.3f ms" % (k[:60], v["calls"], v["ms"]))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
