#!/usr/bin/env python
"""Generate tests/golden/pose_eval_cases.npz from the reference's own ADD / ADD-S scoring.

Source of truth: ``Basic_Utils.cal_add_cuda`` / ``cal_adds_cuda`` / ``cal_auc``, ``VOCap``, ``eval_metric``,
``eval_metric_lm`` and ``TorchEval`` of the reference, taken out of its files with ``ast`` and run on the CPU in
float32 torch (oracle/pose_eval_oracle.eval_functions).  Nothing of the reference is copied.  The seeded inputs
(meshes, distance lists, voting frames) are rebuilt by tests/pose_eval_cases.py wherever they are used; this file
stores the reference's outputs, the poses and the small fixed inputs only.

Keys (``<i>`` numbers a case):
* ``adds:<i>:n`` (the mesh is ``pose_eval_cases.adds_mesh(n)``; ``n = 0`` marks the symmetric ring, stored as
  ``adds:ring``), ``:pred`` / ``:gt`` [3,4] float32, ``:add`` / ``:adds`` float32 scalars, ``:kind`` -- the reference's
  ``cal_add_cuda`` / ``cal_adds_cuda`` for meshes of 1, 31, 32, 33, 2000 and 2621 points under identical poses, a zero
  predicted pose, mm perturbations, 180 degree turns and 10 m offsets, and a symmetric ring turned about its axis;
* ``auc:<name>:auc`` (``cal_auc``) and ``:vocap`` (``VOCap`` of the sorted, capped list and its float32 cumulative
  accuracy) of each list of ``pose_eval_cases.auc_lists()``;
* ``metric:*`` -- one YCB frame's ``eval_metric`` and an ``eval_metric_lm`` call with fixed predicted poses; lists
  stored flat as ``(class index, value)`` pairs in append order;
* ``te:*`` / ``telm:*`` -- a whole ``TorchEval.eval_pose_parallel`` + ``cal_auc`` run over seeded frames with YCB
  class ids (``te``), and ``eval_pose_parallel(ds='linemod')`` + ``cal_lm_add`` for one LineMOD object (``telm``);
  ``te:fingerprint`` / ``telm:fingerprint``: ``frame_fingerprint`` of the batches they were given.

Run:  python tests/golden/make_pose_eval_golden.py      (needs the reference's sources; rewrites pose_eval_cases.npz)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import pose_eval_oracle as PO, ref_loader as R     # noqa: E402
import pose_eval_cases as PC                                     # noqa: E402

OUT = os.path.join(HERE, "pose_eval_cases.npz")


def rot(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose(R_, t):
    return np.concatenate((R_, np.asarray(t, np.float64)[:, None]), 1).astype(np.float32)


def pose_kinds(rs):
    """(name, pred, gt) float32 [3,4] pairs of every kind the tests name."""
    gt = pose(rot(rs), rs.uniform(-0.2, 0.2, 3) + [0, 0, 1])
    small = rot(np.random.RandomState(rs.randint(1 << 30)))
    turn = np.diag([-1.0, -1.0, 1.0])
    far = pose(rot(rs), rs.uniform(-0.1, 0.1, 3) + [10.0, -10.0, 10.0])
    ang = 0.002
    dR = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]])
    return [("identical", gt.copy(), gt),
            ("zero_pred", np.zeros((3, 4), np.float32), gt),
            ("mm", pose(dR @ gt[:, :3].astype(np.float64), gt[:, 3] + rs.uniform(-0.003, 0.003, 3)), gt),
            ("turn180", pose(gt[:, :3].astype(np.float64) @ turn, gt[:, 3]), gt),
            ("offset10m", pose(far[:, :3].astype(np.float64), far[:, 3] + [0.002, -0.001, 0.003]), far),
            ("random", pose(small, rs.uniform(-0.2, 0.2, 3) + [0, 0, 1]), gt)]


def ring(n_ang=24, n_z=6, r=0.05, h=0.08):
    """A mesh symmetric under turns of 2 pi / n_ang about z."""
    a = np.arange(n_ang) * 2 * np.pi / n_ang
    z = np.linspace(-h / 2, h / 2, n_z)
    return np.stack([np.repeat(r * np.cos(a)[None], n_z, 0).ravel(), np.repeat(r * np.sin(a)[None], n_z, 0).ravel(),
                     np.repeat(z[:, None], n_ang, 1).ravel()], 1).astype(np.float32)


def flat(lists):
    cls = np.array([c for c, lst in enumerate(lists) for _ in lst], np.int32)
    val = np.array([float(v) for lst in lists for v in lst], np.float64)
    return cls, val


def adds_cases(F, out):
    rs = np.random.RandomState(7)
    i = 0
    for n in PC.MESH_SIZES:
        for kind, pred, gt in pose_kinds(rs):
            out_case(F, out, i, n, PC.adds_mesh(n), pred, gt, kind)
            i += 1
    mesh = ring()
    out["adds:ring"] = mesh
    gt = pose(rot(rs), [0.05, -0.02, 0.9])
    turn = 2 * np.pi / 24 * 5
    Rz = np.array([[np.cos(turn), -np.sin(turn), 0], [np.sin(turn), np.cos(turn), 0], [0, 0, 1]])
    out_case(F, out, i, 0, mesh, pose(gt[:, :3].astype(np.float64) @ Rz, gt[:, 3]), gt, "symmetric")


def out_case(F, out, i, n, mesh, pred, gt, kind):
    p3 = torch.from_numpy(mesh)
    k = "adds:%d:" % i
    out[k + "n"], out[k + "pred"], out[k + "gt"] = np.int32(n), pred, gt
    out[k + "add"] = np.float32(F["cal_add_cuda"](torch.from_numpy(pred), torch.from_numpy(gt), p3).item())
    out[k + "adds"] = np.float32(F["cal_adds_cuda"](torch.from_numpy(pred), torch.from_numpy(gt), p3).item())
    out[k + "kind"] = np.array(kind)


def auc_cases(F, out):
    for name, dis in PC.auc_lists().items():
        k = "auc:%s:" % name
        out[k + "auc"] = np.float64(F["cal_auc"](dis))
        D = np.array(dis)
        D[np.where(D > 0.1)] = np.inf
        acc = np.cumsum(np.ones((1, len(dis))), dtype=np.float32) / len(dis) if dis else np.zeros(0, np.float32)
        out[k + "vocap"] = np.float64(F["VOCap"](np.sort(D), acc))


def torch_batch(batch):
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in batch.items()}


def main():
    frs, mesh_kps, radius = PC.frames()
    meshes = PC.ycb_meshes()
    batch_lm_np, lm_kps = PC.lm_batch()
    batch_lm = torch_batch(batch_lm_np)
    lm_mesh = PC.lm_mesh()
    LM_OBJ = PC.LM_OBJ
    out = {}
    with R.cuda_is_identity():
        F = PO.eval_functions(meshes, mesh_kps, radius, PC.YCB_SYM, PC.LM_SYM, {LM_OBJ: PC.LM_DIAMETER})
        adds_cases(F, out)
        auc_cases(F, out)

        # eval_metric of frame 0 with fixed predictions: classes 2 and 7 predicted, 13 predicted with another pose,
        # 16 not predicted, then a zero id (the rest is never read)
        rs = np.random.RandomState(5)
        b0_np = PC.ycb_batch(frs)
        b0 = torch_batch(b0_np)
        ids = torch.tensor([[2], [13], [7], [16], [0], [5]])
        pred_cls_ids = np.array([2, 7, 13, 20])
        pred_pose_lst = [np.asarray(frs[0]["poses"][c], np.float64) + rs.normal(0, 0.002, (3, 4)) for c in (1, 3, 2)]
        pred_pose_lst.append(np.eye(4)[:3])
        pred_kpc_lst = [rs.normal(0, 0.1, (PC.N_KPS + 1, 3)).astype(np.float32) for _ in range(4)]
        RTs = torch.stack([b0["RTs"][0, i] for i in (0, 1, 2, 3, 0, 0)])
        gt_kps = torch.stack([b0["gt_kps"][0, i] for i in (0, 1, 2, 3, 0, 0)])
        res = F["eval_metric"](ids, pred_pose_lst, pred_cls_ids, RTs, None, None, gt_kps, None, pred_kpc_lst)
        out["metric:ids"], out["metric:pred_cls_ids"] = ids.numpy(), pred_cls_ids
        out["metric:pred_pose_lst"], out["metric:pred_kpc_lst"] = np.stack(pred_pose_lst), np.stack(pred_kpc_lst)
        out["metric:RTs"], out["metric:gt_kps"] = RTs.numpy(), gt_kps.numpy()
        for name, lst in zip(("add", "adds", "kp_err"), res):
            out["metric:%s:cls" % name], out["metric:%s:val" % name] = flat(lst)
        lm_pred = np.asarray(batch_lm["RTs"][1, 0].numpy(), np.float64) + rs.normal(0, 0.003, (3, 4))
        F_lm = PO.eval_functions({LM_OBJ: lm_mesh}, {LM_OBJ: lm_kps}, radius, PC.YCB_SYM, PC.LM_SYM,
                                 {LM_OBJ: PC.LM_DIAMETER})
        res = F_lm["eval_metric_lm"](batch_lm["cls_ids"][1], [lm_pred], batch_lm["RTs"][1], None, None, LM_OBJ)
        out["metric_lm:pred"], out["metric_lm:RTs"] = lm_pred, batch_lm["RTs"][1].numpy()
        for name, lst in zip(("add", "adds"), res):
            out["metric_lm:%s:cls" % name], out["metric_lm:%s:val" % name] = flat(lst)

        # a whole YCB run: eval_pose_parallel over the three frames, then cal_auc
        te = F["TorchEval"]()
        te.eval_pose_parallel(b0["pclds"], None, b0["masks"], b0["pred_ctr_ofs"], None, [None] * 3, 0, b0["cls_ids"],
                              b0["RTs"], b0["pred_kp_ofs"], b0["gt_kps"], b0["gt_ctrs"])
        te.cal_auc()
        sv = F["dumped"][0]
        out["te:fingerprint"] = PC.frame_fingerprint(b0_np)
        for name in ("add_dis_lst", "adds_dis_lst", "pred_kp_errs"):
            out["te:%s:cls" % name], out["te:%s:val" % name] = flat(sv[name])
        for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
            out["te:" + name] = np.array(sv[name], np.float64)

        # a LineMOD run of one object
        te = F_lm["TorchEval"]()
        te.eval_pose_parallel(batch_lm["pclds"], None, batch_lm["masks"], batch_lm["pred_ctr_ofs"], None, [None] * 3, 0,
                              batch_lm["cls_ids"], batch_lm["RTs"], batch_lm["pred_kp_ofs"], batch_lm["gt_kps"],
                              batch_lm["gt_ctrs"], obj_id=LM_OBJ, ds="linemod")
        te.cal_lm_add(LM_OBJ)
        sv = F_lm["dumped"][0]
        out["telm:fingerprint"] = PC.frame_fingerprint(batch_lm_np)
        for name in ("add_dis_lst", "adds_dis_lst"):
            out["telm:%s:cls" % name], out["telm:%s:val" % name] = flat(sv[name])
        for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst", "add", "adds"):
            out["telm:" + name] = np.array(sv[name], np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
