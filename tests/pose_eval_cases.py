"""The seeded inputs of the pose-scoring cases, rebuilt where they are used: tests/golden/make_pose_eval_golden.py
stores only the reference's outputs for them, with the poses and the small fixed inputs, in
tests/golden/pose_eval_cases.npz.

Meshes and distance lists come from ``RandomState.uniform``, which is bitwise the same everywhere.  The voting frames
come from ``synthetic.make_pose_frame`` and a few small matrix products; the golden file keeps fingerprints of them
(``frame_fingerprint``), so a platform that rebuilt them differently fails loudly rather than comparing other inputs.
"""
import numpy as np

from ffb6d_b200 import synthetic

MESH_SIZES = (1, 31, 32, 33, 2000, 2621)
N_KPS = 8
YCB_SYM = (13, 16, 19, 20, 21)
LM_SYM = (10, 11)
# each frame's classes 1-4 of synthetic.make_pose_frame as YCB ids, and one absent YCB id scored unpredicted
FRAME_IDS = ((2, 13, 7, 16), (21, 5, 19, 11), (9, 20, 1, 14))
ABSENT = (6, 13, 4)
LM_OBJ, LM_DIAMETER = 10, 172.0


def adds_mesh(n):
    """The mesh of n points the single-object cases are scored on."""
    return np.random.RandomState(1000 + n).uniform(-0.1, 0.1, (n, 3)).astype(np.float32)


def auc_lists():
    """name -> the distance list of each ``cal_auc`` edge case."""
    return {"empty": [], "one": [0.03], "above": [0.2, 0.5, 0.11], "exact": [0.1, 0.1, 0.05],
            "duplicates": [0.02, 0.02, 0.02, 0.07, 0.07], "zeros": [0.0, 0.0, 0.04], "nan": [0.01, float("nan"), 0.03],
            "random": list(np.random.RandomState(11).uniform(0, 0.15, 10000))}


def frames():
    """Three seeded frames of synthetic.make_pose_frame with classes 1-4 renamed to FRAME_IDS; the keypoints they
    were voted from (``{YCB id: [N_KPS+1,3]}``, centre last), and per-id radii (``cls_radius``, 21 entries)."""
    out, mesh_kps, radius = [], {}, [0.1] * 21
    for f, ids in enumerate(FRAME_IDS):
        fr = synthetic.make_pose_frame(300 + f, n_kps=N_KPS)
        remap = np.zeros(5, np.int64)
        remap[1:] = ids
        fr["mask"] = remap[fr["mask"]]
        for c in (1, 2, 3, 4):
            mesh_kps[ids[c - 1]] = fr["mesh"][c]
            radius[ids[c - 1] - 1] = fr["cls_radius"][c - 1]
        fr["ids"] = ids
        out.append(fr)
    return out, mesh_kps, radius


def ycb_meshes():
    """``{YCB id: [P,3]}``: the scoring meshes of every id the YCB frames name, 200-899 points each."""
    ids = sorted(set(c for ids in FRAME_IDS for c in ids) | set(ABSENT))
    rs = np.random.RandomState(21)
    return {c: rs.uniform(-0.08, 0.08, (int(rs.randint(200, 900)), 3)).astype(np.float32) for c in ids}


def lm_mesh():
    """The 2 000-point scoring mesh of the LineMOD object."""
    return np.random.RandomState(22).uniform(-0.08, 0.08, (2000, 3)).astype(np.float32)


def ycb_batch(frs):
    """The numpy batch of ``eval_pose_parallel`` over the frames of :func:`frames`: per frame its objects 1-3,
    class 4, its absent id and a 0 row."""
    bs, n_obj = len(frs), 6
    cls_ids = np.zeros((bs, n_obj, 1), np.int64)
    RTs = np.zeros((bs, n_obj, 3, 4), np.float32)
    gt_kps = np.zeros((bs, n_obj, N_KPS, 3), np.float32)
    gt_ctrs = np.zeros((bs, n_obj, 3), np.float32)
    for b, fr in enumerate(frs):
        objs = [(fr["ids"][c - 1], fr["poses"][c], fr["mesh"][c]) for c in (1, 2, 3, 4)]
        objs.append((ABSENT[b], fr["poses"][2], fr["mesh"][2]))
        for i, (cid, P, mk) in enumerate(objs):
            cls_ids[b, i, 0] = cid
            RTs[b, i] = P
            cam = mk @ P[:, :3].T + P[:, 3]
            gt_kps[b, i], gt_ctrs[b, i] = cam[:N_KPS], cam[N_KPS]
    return dict(pclds=np.stack([f["pcld"] for f in frs]), masks=np.stack([f["mask"] for f in frs]),
                pred_ctr_ofs=np.stack([f["ctr_of"] for f in frs]), pred_kp_ofs=np.stack([f["kp_of"] for f in frs]),
                cls_ids=cls_ids, RTs=RTs, gt_kps=gt_kps, gt_ctrs=gt_ctrs)


def lm_batch():
    """Three LineMOD frames of one object, class 1: a make_pose_frame frame and two rigid motions of it (so all
    three share the object-frame keypoints).  Returns the numpy batch and the keypoints ``[N_KPS+1,3]``."""
    fr = synthetic.make_pose_frame(350, n_kps=N_KPS)
    rs = np.random.RandomState(351)
    pcld, ctr, kp, RT = [], [], [], []
    for b in range(3):
        Rm = np.eye(3) if b == 0 else np.linalg.qr(np.eye(3) + 0.1 * rs.normal(size=(3, 3)))[0]
        if np.linalg.det(Rm) < 0:
            Rm[:, 0] = -Rm[:, 0]
        t = np.zeros(3) if b == 0 else rs.uniform(-0.05, 0.05, 3)
        pcld.append((fr["pcld"] @ Rm.T + t).astype(np.float32))
        ctr.append((fr["ctr_of"] @ Rm.T).astype(np.float32))
        kp.append((fr["kp_of"] @ Rm.T).astype(np.float32))
        P = fr["poses"][1]
        RT.append(np.concatenate((Rm @ P[:, :3], (Rm @ P[:, 3] + t)[:, None]), 1).astype(np.float32)[None])
    mask = np.where(fr["mask"] == 1, 1, 0).astype(np.int64)
    return dict(pclds=np.stack(pcld), masks=np.stack([mask] * 3), pred_ctr_ofs=np.stack(ctr),
                pred_kp_ofs=np.stack(kp), RTs=np.stack(RT), cls_ids=np.ones((3, 1, 1), np.int64),
                gt_kps=np.zeros((3, 1, N_KPS, 3), np.float32), gt_ctrs=np.zeros((3, 1, 3), np.float32)), fr["mesh"][1]


def frame_fingerprint(batch):
    """float64 [n]: the sum and the sum of squares of every float array of a batch, in key order."""
    return np.array([f(np.asarray(batch[k], np.float64)) for k in sorted(batch) if batch[k].dtype.kind == "f"
                     for f in (np.sum, lambda a: np.sum(a * a))])
