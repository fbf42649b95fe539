"""Keypoint voting and pose fitting on the GPU: the step after the network (SURVEY.md §8 f-4).

Mirrors of the reference's evaluation helpers, same names and argument meaning:

* :class:`MeanShiftTorch` -- ``utils/meanshift_pytorch.py:27-57`` (``fit``; ``fit_multi_clus`` is only used by
  that file's own ``__main__`` and is not provided);
* :func:`best_fit_transform` -- ``utils/pvn3d_eval_utils_kpls.py:28-59`` (numpy in, numpy ``[3,4]`` out);
* :func:`cal_frame_poses`, :func:`cal_frame_poses_lm` -- ``utils/pvn3d_eval_utils_kpls.py:65-160, 220-284``, B = 1
  calls of :func:`cal_batch_poses`, which votes every object of a batch without a host sync;
* :func:`cal_add_cuda`, :func:`cal_adds_cuda`, :func:`cal_auc`, :func:`VOCap` -- ``utils/basic_utils.py:34-46,
  642-669`` (``Basic_Utils`` methods there, functions here);
* :func:`eval_metric`, :func:`eval_metric_lm`, :class:`TorchEval` -- ``utils/pvn3d_eval_utils_kpls.py:162-195,
  287-304, 326-505``: ADD / ADD-S scoring, every object of a frame (``eval_metric``) or of a batch
  (``TorchEval.eval_pose_parallel``) in one :func:`ffb6d_b200.ops.pose_add_adds` launch over a :class:`MeshTable`.

The reference reads mesh keypoints, mesh centres and object radii from dataset files through its module-level
``bs_utils`` / ``config``; here the caller passes them (``mesh_kps``, ``cls_radius``).  Everything numeric runs in
:func:`ffb6d_b200.ops.vote_poses` (all vote sets of a batch in one persistent mean-shift kernel per stage instead of
one N x N torch program per keypoint and a host sync per iteration), :func:`ffb6d_b200.ops.mean_shift_fit` and
:func:`ffb6d_b200.ops.best_fit_transform`.
"""
import numpy as np
import torch

from . import _lib, ops


class MeanShiftTorch:
    def __init__(self, bandwidth=0.05, max_iter=300):
        self.bandwidth = bandwidth
        self.stop_thresh = bandwidth * 1e-3
        self.max_iter = max_iter

    def fit(self, A, ret_mid_res=False):
        """``A [N,3]`` CUDA float32 -> ``(centre [3], labels [N] bool)``; with ``ret_mid_res`` the converged
        positions ``[N,3]`` and their pairwise distances ``[N,N]`` like the reference (that matrix is built
        with torch, for callers that want it; ``fit`` itself never forms it)."""
        out = ops.mean_shift_fit(A[None].float(), None, self.bandwidth, self.max_iter, return_modes=ret_mid_res)
        if not ret_mid_res:
            return out[0][0], out[1][0]
        C = out[3][0]
        return C, torch.cdist(C, C)

    def fit_batch(self, votes, valid=None):
        """``votes [G,N,3]``, ``valid [N]`` or ``[G,N]`` -> ``(centres [G,3], labels [G,N] bool)``: ``fit`` of every
        ``votes[g][valid]`` in one launch (labels are in the unmasked point order)."""
        centres, labels, _ = ops.mean_shift_fit(votes, valid, self.bandwidth, self.max_iter)
        return centres, labels


def best_fit_transform(A, B):
    """numpy ``[M,3]`` x2 -> numpy float64 ``[3,4]`` (pvn3d_eval_utils_kpls.py:28-59), computed on the GPU."""
    dev = torch.device("cuda", torch.cuda.current_device())
    a = torch.as_tensor(np.asarray(A, dtype=np.float32), device=dev)
    b = torch.as_tensor(np.asarray(B, dtype=np.float32), device=dev)
    return ops.best_fit_transform(a, b).cpu().numpy()


class VoteTable:
    """The per-class inputs of :func:`cal_batch_poses`, resident on the GPU and indexed by class id ``0 .. n_cls-1``.

    ``mesh_kps``: mapping ``cls_id -> [rows,3]`` object-frame keypoints, the centre last (what the reference loads
    with ``bs_utils.get_kps`` / ``get_ctr``), every one with the same number of rows; ``cls_radius``: sequence
    indexed by ``cls_id - 1`` (``config.ycb_r_lst``) or None.  Holds ``kps [n_cls,rows,3]`` float32 (zero for ids
    without keypoints), ``has_mesh [n_cls]`` uint8 and ``refine_thr [n_cls]`` float32, the refinement distance
    ``float32(float64(r) * 0.8)`` as the reference rounds it (None without ``cls_radius``)."""

    def __init__(self, mesh_kps, n_cls, cls_radius=None, device=None):
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        arrs = {int(c): np.asarray(torch.as_tensor(v).detach().cpu(), np.float32) for c, v in mesh_kps.items()}
        if any(c < 0 or c >= n_cls for c in arrs):
            raise ValueError("mesh_kps ids must lie in [0, %d), got %s" % (n_cls, sorted(arrs)))
        shapes = {a.shape for a in arrs.values()}
        if len(shapes) > 1 or any(len(sh) != 2 or sh[1] != 3 for sh in shapes):
            raise ValueError("mesh_kps must all be [rows,3] with one row count, got %s" % sorted(shapes))
        rows = shapes.pop()[0] if shapes else 1
        kps = np.zeros((n_cls, rows, 3), np.float32)
        has = np.zeros(n_cls, np.uint8)
        for c, a in arrs.items():
            kps[c], has[c] = a, 1
        self.n_cls = n_cls
        self.kps = torch.as_tensor(kps, device=dev)
        self.has_mesh = torch.as_tensor(has, device=dev)
        self.refine_thr = None
        if cls_radius is not None:
            r = np.asarray(cls_radius, np.float64).reshape(-1)
            if r.shape[0] < n_cls - 1:
                raise ValueError("cls_radius needs n_cls - 1 = %d entries, got %d" % (n_cls - 1, r.shape[0]))
            thr = np.zeros(n_cls, np.float32)
            thr[1:] = (r[:n_cls - 1] * 0.8).astype(np.float32)
            self.refine_thr = torch.as_tensor(thr, device=dev)
        self.device = dev

    def rows(self, R):
        """``[n_cls,R,3]``: the first ``R`` keypoint rows of every class."""
        if R > self.kps.shape[1]:
            raise ValueError("mesh_kps have %d rows, %d needed" % (self.kps.shape[1], R))
        return self.kps[:, :R].contiguous()


def _vote(table, pclds, masks, ctr_ofs, kp_ofs, use_ctr, ctr_filter, refine):
    n_kps = kp_ofs.shape[1]
    return ops.vote_poses(pclds, masks.long(), ctr_ofs, kp_ofs, table.rows(n_kps + int(bool(use_ctr))),
                          table.has_mesh, table.refine_thr if refine else None, use_ctr, ctr_filter, bandwidth=0.04,
                          max_iter=300)


def cal_batch_poses(pclds, masks, ctr_ofs, kp_ofs, use_ctr, n_cls, use_ctr_clus_flter, *, mesh_kps, cls_radius=None):
    """:func:`cal_frame_poses` of a whole batch in one :func:`ffb6d_b200.ops.vote_poses` call, without a host
    synchronisation: ``pclds [B,N,3]``, ``masks [B,N]``, ``ctr_ofs [B,1,N,3]``, ``kp_ofs [B,n_kps,N,3]`` as the
    network's ``end_points`` hold them.  ``mesh_kps``: a :class:`VoteTable`, or the mapping one is built from with
    ``n_cls`` and ``cls_radius``.  ``use_ctr_clus_flter`` turns on the centre-clustering refinement of the mask
    (when there are radii) and the centre-label filter of the keypoint votes, as in the reference.

    Returns ``(present [B,n_cls] bool, count [B,n_cls] int32, kps [B,n_cls,n_kps+use_ctr,3] float32,
    poses [B,n_cls,3,4] float64)`` CUDA tensors: ``present`` the classes of the unrefined mask (the reference's
    ``pred_cls_ids``), ``count`` their points after refinement; a class left without points has the identity pose
    and zero keypoints, an absent class zeros, and a frame with a mask id outside ``[0, n_cls)`` NaN rows, as does a
    present class without keypoints in ``mesh_kps``."""
    table = mesh_kps if isinstance(mesh_kps, VoteTable) else VoteTable(mesh_kps, n_cls, cls_radius, pclds.device)
    return _vote(table, pclds, masks, ctr_ofs, kp_ofs, use_ctr, use_ctr_clus_flter,
                 use_ctr_clus_flter and table.refine_thr is not None)


def _to_host(*ts):
    """Numpy copies of the CUDA tensors ``ts``, through one device-to-host copy."""
    flat = torch.cat([t.contiguous().reshape(-1).view(torch.uint8) for t in ts]).cpu().numpy()
    out, o = [], 0
    for t in ts:
        dt = np.dtype(str(t.dtype).replace("torch.", "")) if t.dtype != torch.bool else np.dtype(np.bool_)
        n = t.numel() * dt.itemsize
        out.append(flat[o:o + n].view(dt).reshape(tuple(t.shape)))
        o += n
    return out


def _frame_lists(present, count, kps, poses, has_mesh, n_kps):
    """The reference's ``(pred_cls_ids, pred_pose_lst, pred_kps_lst)`` of one frame from its host rows."""
    if np.isnan(poses[0]).any():
        raise ValueError("the mask holds a class id outside [0, %d)" % present.shape[0])
    ids = np.flatnonzero(present).astype(np.int64)
    missing = [int(c) for c in ids if not has_mesh[c]]
    if missing:
        raise ValueError("no mesh keypoints for predicted class(es) %s" % missing)
    pose_lst, kps_lst = [], []
    for c in ids:
        empty = count[c] == 0
        pose_lst.append(np.identity(4)[:3, :] if empty else poses[c])
        kps_lst.append(np.zeros((n_kps + 1, 3)) if empty else kps[c])
    return ids, pose_lst, kps_lst


def cal_frame_poses(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter, gt_kps=None, gt_ctrs=None,
                    debug=False, kp_type="farthest", *, mesh_kps, cls_radius=None):
    """YCB-style multi-object voting (pvn3d_eval_utils_kpls.py:65-160): :func:`cal_batch_poses` of one frame.

    ``pcld [N,3]``, ``mask [N]`` predicted class ids in ``[0, n_cls)``, ``ctr_of [1,N,3]``, ``pred_kp_of
    [n_kps,N,3]`` (CUDA).  ``mesh_kps``: mapping ``cls_id -> [n_kps(+1),3]`` array of object-frame keypoints (the
    centre last when ``use_ctr``), what the reference loads with ``bs_utils.get_kps`` / ``get_ctr``; ``cls_radius``:
    sequence indexed by ``cls_id - 1`` (``config.ycb_r_lst``), needed for the centre-clustering mask refinement.
    Returns ``(pred_cls_ids, pred_pose_lst, pred_kps_lst)`` like the reference; raises ValueError for a mask id out
    of range or a predicted class without keypoints."""
    n_kps = pred_kp_of.shape[0]
    table = VoteTable(mesh_kps, n_cls, cls_radius, pcld.device)
    present, count, kps, poses = _vote(table, pcld[None], mask[None], ctr_of[None], pred_kp_of[None], use_ctr,
                                       use_ctr_clus_flter, use_ctr_clus_flter and cls_radius is not None)
    poses, kps, count, present, has = _to_host(poses[0], kps[0], count[0], present[0], table.has_mesh)
    return _frame_lists(present, count, kps, poses, has, n_kps)


def _lm_table(mesh_kps, device):
    return VoteTable({1: mesh_kps}, 2, None, device)


def cal_frame_poses_lm(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter, obj_id, debug=False, *,
                       mesh_kps):
    """LineMOD-style single-object voting (pvn3d_eval_utils_kpls.py:220-284): class 1 is the object, every other id
    background; a :func:`cal_batch_poses` of one frame with two classes and no refinement.
    ``mesh_kps [n_kps(+1),3]``: object-frame keypoints of ``obj_id`` (centre last when ``use_ctr``)."""
    table = _lm_table(mesh_kps, pcld.device)
    present, _, _, poses = _vote(table, pcld[None], (mask == 1)[None], ctr_of[None], pred_kp_of[None], use_ctr,
                                 use_ctr_clus_flter, False)
    poses, present = _to_host(poses[0, 1], present[0, 1])
    return [poses if present else np.identity(4)[:3, :]]


# ---------------------------------------------------------------------------------------------------- pose scoring
class MeshTable:
    """The meshes that ADD / ADD-S are computed over, resident on the GPU and indexed by class id.

    ``mesh_pts``: mapping ``cls_id -> [P,3]`` vertices in metres, what the reference's ``bs_utils.get_pointxyz(_cuda)``
    returns (YCB: ``models/<cls>/points.xyz``; LineMOD: the 2 000-vertex subsample the caller drew, the reference
    redraws it in every process).  Holds ``pts [sum P,3]`` float32, ``off [max id + 2]`` int32 (mesh ``c`` is rows
    ``off[c] .. off[c+1]``; ids without a mesh are empty, and scoring one gives NaN) and ``max_points``.

    ``dtype=torch.float64`` keeps the vertices in float64, for drawing (:func:`ffb6d_b200.vis.draw_poses`): the demo
    poses the meshes in float64, and rounding them to float32 would move points that lie near a half-pixel.  Scoring
    (:func:`add_adds`) needs the float32 table."""

    def __init__(self, mesh_pts, device=None, dtype=torch.float32):
        if dtype not in (torch.float32, torch.float64):
            raise ValueError("MeshTable dtype must be torch.float32 or torch.float64, got %s" % dtype)
        np_dtype = np.float32 if dtype == torch.float32 else np.float64
        if not mesh_pts:
            raise ValueError("MeshTable needs at least one mesh")
        ids = sorted(int(c) for c in mesh_pts)
        if ids[0] < 0:
            raise ValueError("class ids must be >= 0, got %d" % ids[0])
        arrs = {int(c): np.asarray(torch.as_tensor(v).detach().cpu(), np_dtype) for c, v in mesh_pts.items()}
        sizes = np.zeros(ids[-1] + 1, np.int64)
        for c, a in arrs.items():
            if a.ndim != 2 or a.shape[1] != 3 or a.shape[0] < 1:
                raise ValueError("mesh %d must be [P,3] with P >= 1, got %s" % (c, a.shape))
            sizes[c] = a.shape[0]
        off = np.concatenate(([0], np.cumsum(sizes)))
        if off[-1] > 2 ** 31 - 1:
            raise ValueError("%d mesh points in all: more than int32 offsets address" % off[-1])
        self.max_points = int(sizes.max())
        if self.max_points > _lib.POSE_EVAL_MAX_POINTS:
            raise ValueError("a mesh of %d points: at most %d" % (self.max_points, _lib.POSE_EVAL_MAX_POINTS))
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.pts = torch.as_tensor(np.concatenate([arrs[c] for c in ids]), device=dev)
        self.off = torch.as_tensor(off.astype(np.int32), device=dev)
        self.device = dev


def add_adds(table, cls_ids, pred_RT, gt_RT):
    """ADD and ADD-S of ``M`` objects in one launch: object ``m`` is mesh ``cls_ids[m]`` of ``table`` under the
    poses ``pred_RT[m]``, ``gt_RT[m]`` (``[M,3,4]``, numpy or torch).  Returns ``(add [M], adds [M])`` float32
    CUDA tensors; see :func:`ffb6d_b200.ops.pose_add_adds`."""
    if table.pts.dtype != torch.float32:
        raise ValueError("add_adds scores a float32 MeshTable, got %s" % table.pts.dtype)
    dev = table.device
    ids = torch.as_tensor(np.asarray(cls_ids, np.int64) if not torch.is_tensor(cls_ids) else cls_ids)
    ids = ids.to(dev, torch.int32).reshape(-1)
    pr = torch.as_tensor(pred_RT).to(dev, torch.float32).reshape(-1, 3, 4)
    gt = torch.as_tensor(gt_RT).to(dev, torch.float32).reshape(-1, 3, 4)
    return ops.pose_add_adds(table.pts, table.off, ids, pr, gt, table.max_points)


def _one_object(pred_RT, gt_RT, p3ds):
    p = ops._tensor(p3ds, "p3ds", torch.float32, 2)
    dev = p.device
    off = torch.tensor([0, p.shape[0]], dtype=torch.int32, device=dev)
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    pr = torch.as_tensor(pred_RT).to(dev, torch.float32).reshape(1, 3, 4)
    gt = torch.as_tensor(gt_RT).to(dev, torch.float32).reshape(1, 3, 4)
    return ops.pose_add_adds(p, off, zero, pr, gt, max(int(p.shape[0]), 1))


def cal_add_cuda(pred_RT, gt_RT, p3ds):
    """``Basic_Utils.cal_add_cuda`` (basic_utils.py:651-657): mean ``|pred_RT x - gt_RT x|`` over ``p3ds [N,3]``
    (CUDA float32), as a 0-d float32 CUDA tensor; an ``M = 1`` :func:`ffb6d_b200.ops.pose_add_adds`."""
    return _one_object(pred_RT, gt_RT, p3ds)[0][0]


def cal_adds_cuda(pred_RT, gt_RT, p3ds):
    """``Basic_Utils.cal_adds_cuda`` (basic_utils.py:659-669): mean over the gt-posed points of the distance to the
    nearest pred-posed point, as a 0-d float32 CUDA tensor; an ``M = 1`` :func:`ffb6d_b200.ops.pose_add_adds`."""
    return _one_object(pred_RT, gt_RT, p3ds)[1][0]


def VOCap(rec, prec):
    """The area under the accuracy-threshold curve (basic_utils.py:34-46), times 10: ``rec`` the sorted distances
    (``inf`` entries dropped, the curve closed at 0.1 m), ``prec`` the cumulative accuracy.  Returns 0 when no
    distance is finite; a NaN distance makes it NaN."""
    keep = rec != np.inf
    if not keep.any():
        return 0
    rec, prec = rec[keep], prec[keep]
    mrec = np.concatenate(([0.0], rec, [0.1]))
    mpre = np.concatenate(([0.0], prec, [prec[-1]]))
    k = prec.shape[0]
    mpre[:k] = np.maximum.accumulate(mpre[:k])      # the reference's running max covers entries 1 .. k - 1
    step = np.flatnonzero(mrec[1:] != mrec[:-1]) + 1
    return np.sum((mrec[step] - mrec[step - 1]) * mpre[step]) * 10


def cal_auc(add_dis, max_dis=0.1):
    """``Basic_Utils.cal_auc`` (basic_utils.py:642-649): the ADD(-S) AUC in percent of a list of distances.  Those
    ``> max_dis`` count as misses (exactly ``max_dis`` stays); the accuracy is a float32 cumulative count; an empty
    list gives 0 and a NaN distance a NaN AUC."""
    D = np.array(add_dis)
    D = np.sort(np.where(D > max_dis, np.inf, D))
    n = len(add_dis)
    acc = np.cumsum(np.ones(n), dtype=np.float32) / n
    return VOCap(D, acc) * 100


def _ids_column(cls_ids):
    """``cls_ids [n_obj(,1)]`` (tensor or array) -> int64 numpy [n_obj]: the first column, as the reference's
    ``cls_id[0]``."""
    a = np.asarray(cls_ids.detach().cpu() if torch.is_tensor(cls_ids) else cls_ids)
    return a.reshape(a.shape[0], -1)[:, 0].astype(np.int64) if a.size else np.zeros(0, np.int64)


def _frame_objects(ids, pred_pose_lst, pred_cls_ids, gt_kps_h, pred_kpc_lst):
    """The scored objects of one YCB frame, up to its first zero class id (pvn3d_eval_utils_kpls.py:170-186): their
    class ids, float32 predicted poses (zero for a class that was not predicted) and keypoint errors."""
    cls, poses, kp_errs = [], [], []
    pred_cls_ids = np.asarray(pred_cls_ids)
    for icls, cid in enumerate(ids):
        if cid == 0:
            break
        gt_kp = gt_kps_h[icls]
        hit = np.where(pred_cls_ids == cid)[0]
        if len(hit) == 0:
            pred_RT = np.zeros((3, 4), np.float32)
            pred_kp = np.zeros(gt_kp.shape)
        else:
            pred_RT = np.asarray(pred_pose_lst[hit[0]]).astype(np.float32)
            pred_kp = pred_kpc_lst[hit[0]][:-1, :]
        kp_errs.append(np.linalg.norm(gt_kp - pred_kp, axis=1).mean())
        cls.append(int(cid))
        poses.append(pred_RT)
    return cls, poses, kp_errs


def _score(table, cls, poses, gt_RT):
    """ADD / ADD-S of the objects ``cls`` (class ids) under the float32 numpy poses ``poses`` and the device poses
    ``gt_RT [M,3,4]``: one host-to-device copy, one launch, one device-to-host copy.  Returns two lists of floats."""
    if not cls:
        return [], []
    dev = table.device
    ids = torch.as_tensor(np.asarray(cls, np.int32)).to(dev)
    pr = torch.as_tensor(np.stack(poses)).to(dev)
    add, adds = ops.pose_add_adds(table.pts, table.off, ids, pr, gt_RT.to(dev, torch.float32).contiguous(),
                                  table.max_points)
    both = torch.stack((add, adds)).cpu().numpy()
    return both[0].tolist(), both[1].tolist()


def eval_metric(cls_ids, pred_pose_lst, pred_cls_ids, RTs, mask, label, gt_kps, gt_ctrs, pred_kpc_lst, *, mesh_table,
                n_cls=22):
    """``eval_metric`` (pvn3d_eval_utils_kpls.py:162-195) of one YCB frame: ``(cls_add_dis, cls_adds_dis,
    cls_kp_err)``, ``n_cls`` lists each, class 0 collecting every object.  ``mesh_table``: a :class:`MeshTable`
    keyed by class id (what the reference loads with ``bs_utils.get_pointxyz_cuda``).  Objects are taken up to the
    first zero class id; every one of them is scored in one launch."""
    ids = _ids_column(cls_ids)
    gt_kps_h = gt_kps.detach().cpu().numpy() if torch.is_tensor(gt_kps) else np.asarray(gt_kps)
    cls, poses, kp_errs = _frame_objects(ids, pred_pose_lst, pred_cls_ids, gt_kps_h, pred_kpc_lst)
    add, adds = _score(mesh_table, cls, poses, torch.as_tensor(RTs[:len(cls)]))
    cls_add_dis, cls_adds_dis, cls_kp_err = ([[] for _ in range(n_cls)] for _ in range(3))
    for c, a, s, e in zip(cls, add, adds, kp_errs):
        cls_kp_err[c].append(e)
        cls_add_dis[c].append(a)
        cls_adds_dis[c].append(s)
        cls_add_dis[0].append(a)
        cls_adds_dis[0].append(s)
    return cls_add_dis, cls_adds_dis, cls_kp_err


def eval_metric_lm(cls_ids, pred_pose_lst, RTs, mask, label, obj_id, *, mesh_table, n_cls=22):
    """``eval_metric_lm`` (pvn3d_eval_utils_kpls.py:287-304): ADD / ADD-S of ``pred_pose_lst[0]`` against
    ``RTs[0]`` on mesh ``obj_id`` of ``mesh_table``; returns ``(cls_add_dis, cls_adds_dis)``."""
    add, adds = _score(mesh_table, [int(obj_id)], [np.asarray(pred_pose_lst[0]).astype(np.float32)],
                       torch.as_tensor(RTs[:1]))
    cls_add_dis, cls_adds_dis = [[] for _ in range(n_cls)], [[] for _ in range(n_cls)]
    for i in (int(obj_id), 0):
        cls_add_dis[i].append(add[0])
        cls_adds_dis[i].append(adds[0])
    return cls_add_dis, cls_adds_dis


def _ycb_scores(mesh_table, vote_table, pclds, masks, ctr_ofs, kp_ofs, cls_ids, RTs, use_ctr, use_ctr_clus_flter):
    """The device half of a YCB batch of :meth:`TorchEval.eval_pose_parallel`: the vote, each ground-truth object's
    predicted pose (zero for a class the vote did not find) and its ADD / ADD-S.  Returns ``(votes, ids [B,n_obj]
    int32, pred [B*n_obj,3,4] float32, add, adds)``; no host synchronisation."""
    bs, n_obj = RTs.shape[0], RTs.shape[1]
    dev = mesh_table.device
    gt = RTs.reshape(bs * n_obj, 3, 4).to(dev, torch.float32)
    votes = _vote(vote_table, pclds, masks, ctr_ofs, kp_ofs, use_ctr, use_ctr_clus_flter,
                  use_ctr_clus_flter and vote_table.refine_thr is not None)
    poses = votes[3]
    ids = torch.as_tensor(cls_ids).to(dev).reshape(bs, n_obj, -1)[:, :, 0].long()
    ok = (ids >= 0) & (ids < vote_table.n_cls)
    pick = torch.where(ok, ids, 0)
    pred = poses[torch.arange(bs, device=dev)[:, None], pick].float()     # absent classes: zero rows
    pred = torch.where(ok[..., None, None], pred, 0.0).reshape(bs * n_obj, 3, 4).contiguous()
    om = ids.clamp(-1, 2 ** 31 - 1).int()                      # an id without a mesh scores NaN
    add, adds = ops.pose_add_adds(mesh_table.pts, mesh_table.off, om.reshape(-1), pred, gt.contiguous(),
                                  mesh_table.max_points)
    return votes, om, pred, add, adds


def _ycb_record(rows, state, votes, ids, pred, add, adds, gt_kps, valid=None, frame_poses=None, frame_flags=None):
    present, _, kps, poses = votes
    bs, n_obj = ids.shape
    gk = torch.as_tensor(gt_kps).to(kps.device, torch.float32)
    ops.eval_record(rows, state, ids, present, pred.reshape(bs, n_obj, 3, 4), add, adds, kps=kps, gt_kps=gk,
                    valid=valid, poses=poses if frame_poses is not None else None, frame_poses=frame_poses,
                    frame_flags=frame_flags)


def _lm_scores(mesh_table, lm_table, obj_id, pclds, masks, ctr_ofs, kp_ofs, RTs, use_ctr, use_ctr_clus_flter):
    """The device half of a LineMOD batch: the two-class vote on ``masks == 1``, the object's predicted pose (the
    identity where the vote found no point) and its ADD / ADD-S.  Returns ``(votes, pred [B,3,4], add, adds)``."""
    bs, n_obj = RTs.shape[0], RTs.shape[1]
    dev = mesh_table.device
    gt = RTs.reshape(bs, n_obj, 3, 4)[:, 0].to(dev, torch.float32).contiguous()
    votes = _vote(lm_table, pclds, masks == 1, ctr_ofs, kp_ofs, use_ctr, use_ctr_clus_flter, False)
    present, poses = votes[0], votes[3]
    eye = torch.eye(3, 4, dtype=torch.float32, device=dev)
    pred = torch.where(present[:, 1, None, None], poses[:, 1].float(), eye).contiguous()
    om = torch.full((bs,), obj_id, dtype=torch.int32, device=dev)
    add, adds = ops.pose_add_adds(mesh_table.pts, mesh_table.off, om, pred, gt, mesh_table.max_points)
    return votes, pred, add, adds


def _lm_record(rows, state, votes, obj_id, n_obj, pred, add, adds, valid=None):
    bs = pred.shape[0]
    ids = torch.zeros((bs, n_obj), dtype=torch.int32, device=pred.device)      # read for its shape only
    ops.eval_record(rows, state, ids, votes[0], pred, add, adds, valid=valid, obj_id=obj_id)


def _append_rows(rows, cls_add_dis, cls_adds_dis, kp_errs=None):
    """Append the host record rows ``rows [n, EVAL_ROW_WORDS]`` int32 to the per-class lists in row order: every
    object to its class's list and to list 0, its keypoint error (with ``kp_errs``) to its class's."""
    vals = rows.view(np.float32)
    for r in np.flatnonzero(rows[:, 0] != -1):
        cid = int(rows[r, 0])
        if kp_errs is not None:
            kp_errs[cid].append(float(vals[r, 5]))
        for i in (cid, 0):
            cls_add_dis[i].append(float(vals[r, 3]))
            cls_adds_dis[i].append(float(vals[r, 4]))


class TorchEval:
    """The reference's ``TorchEval`` (pvn3d_eval_utils_kpls.py:326-505): per-class ADD / ADD-S lists over a test run
    and their AUCs.

    The constructor takes what the reference reads from its module-level ``config`` / ``bs_utils``: ``mesh_pts``
    (mapping ``cls_id -> [P,3]``, the scoring meshes; LineMOD: keyed by ``obj_id``), ``mesh_kps`` (mapping
    ``cls_id -> [n_kps(+1),3]``, see :func:`cal_frame_poses`), ``cls_radius`` (``config.ycb_r_lst``) and
    ``sym_cls_ids`` (``config.ycb_sym_cls_ids`` or ``config_lm.lm_sym_cls_ids``).

    :meth:`eval_pose_parallel` votes the batch in one :func:`cal_batch_poses` call and scores every object of it in
    one :func:`ffb6d_b200.ops.pose_add_adds` launch; the lists grow frame by frame, object by object, as the
    reference's ``executor.map`` makes them.  :meth:`cal_auc` and :meth:`cal_lm_add`
    return the dict the reference pickles plus the averages it prints; they print nothing and write no file.

    One deliberate difference: the reference's ``cal_auc`` / ``cal_lm_add`` append to ``cls_add_s_dis[0]`` on every
    call, so a second call counts the objects twice.  Here the ADD(-S) lists are rebuilt on each call; a single call
    gives the reference's result."""

    def __init__(self, mesh_pts, mesh_kps, cls_radius=None, sym_cls_ids=(), n_cls=22):
        self.n_cls = n_cls
        self.mesh_table = MeshTable(mesh_pts)
        dev = self.mesh_table.device
        self.vote_table = VoteTable({c: k for c, k in mesh_kps.items() if 0 <= int(c) < n_cls}, n_cls, cls_radius, dev)
        self.lm_tables = {int(c): _lm_table(k, dev) for c, k in mesh_kps.items()}
        self.sym_cls_ids = list(sym_cls_ids)
        self.cls_add_dis = [[] for _ in range(n_cls)]
        self.cls_adds_dis = [[] for _ in range(n_cls)]
        self.cls_add_s_dis = [[] for _ in range(n_cls)]
        self.pred_kp_errs = [[] for _ in range(n_cls)]
        self.pred_id2pose_lst = []

    def eval_pose_parallel(self, pclds, rgbs, masks, pred_ctr_ofs, gt_ctr_ofs, labels, cnt, cls_ids, RTs,
                           pred_kp_ofs, gt_kps, gt_ctrs, min_cnt=20, merge_clus=False, use_ctr_clus_flter=True,
                           use_ctr=True, obj_id=0, kp_type="farthest", ds="ycb"):
        """Vote and score one batch (pvn3d_eval_utils_kpls.py:448-500), appending to the per-class lists.  ``rgbs``,
        ``gt_ctr_ofs``, ``labels``, ``cnt``, ``min_cnt`` and ``merge_clus`` are accepted and unread, as in the
        reference.  One :func:`cal_batch_poses` call votes the batch, each ground-truth object's predicted pose is
        taken on the device, one :func:`ffb6d_b200.ops.pose_add_adds` launch scores every object, one
        :func:`ffb6d_b200.ops.eval_record` launch lays the objects out as the lists take them (with their keypoint
        errors), and one device-to-host copy brings back what the lists need."""
        bs, n_obj = RTs.shape[0], RTs.shape[1]
        dev = self.mesh_table.device
        rows = torch.empty((bs * n_obj, _lib.EVAL_ROW_WORDS), dtype=torch.int32, device=dev)
        state = torch.zeros(4, dtype=torch.int64, device=dev)
        if ds == "ycb":
            n_kps = pred_kp_ofs.shape[1]
            votes, ids, pred, add, adds = _ycb_scores(self.mesh_table, self.vote_table, pclds, masks, pred_ctr_ofs,
                                                      pred_kp_ofs, cls_ids, RTs, use_ctr, use_ctr_clus_flter)
            _ycb_record(rows, state, votes, ids, pred, add, adds, gt_kps)
            present, count, kps, poses = votes
            rows, poses, kps, count, present, has = _to_host(rows, poses, kps, count, present,
                                                             self.vote_table.has_mesh)
            for b in range(bs):
                pred_cls_ids, pred_poses, _ = _frame_lists(present[b], count[b], kps[b], poses[b], has, n_kps)
                self.pred_id2pose_lst.append({cid: pose for cid, pose in zip(pred_cls_ids, pred_poses)})
        else:
            votes, pred, add, adds = _lm_scores(self.mesh_table, self.lm_tables[int(obj_id)], int(obj_id), pclds,
                                                masks, pred_ctr_ofs, pred_kp_ofs, RTs, use_ctr, use_ctr_clus_flter)
            _lm_record(rows, state, votes, int(obj_id), n_obj, pred, add, adds)
            rows, = _to_host(rows)
        _append_rows(rows, self.cls_add_dis, self.cls_adds_dis, self.pred_kp_errs if ds == "ycb" else None)

    def _add_s_lists(self, cls_range):
        self.cls_add_s_dis = [[] for _ in range(self.n_cls)]
        for c in cls_range:
            self.cls_add_s_dis[c] = list(self.cls_adds_dis[c] if c in self.sym_cls_ids else self.cls_add_dis[c])
            self.cls_add_s_dis[0] += self.cls_add_s_dis[c]

    def cal_auc(self):
        """The YCB summary (pvn3d_eval_utils_kpls.py:338-399): the dict the reference pickles (``add_dis_lst``,
        ``adds_dis_lst``, ``add_auc_lst``, ``adds_auc_lst``, ``add_s_auc_lst``, ``pred_kp_errs``; entry 0 of each
        AUC list is over all objects) plus what it prints: ``mean_kp_err`` (NaN without objects, where the reference
        divides by zero) and ``add_auc_mean`` / ``adds_auc_mean`` / ``add_s_auc_mean`` over classes 1 .. n_cls-1."""
        self._add_s_lists(range(1, self.n_cls))
        add_auc_lst = [cal_auc(self.cls_add_dis[i]) for i in range(self.n_cls)]
        adds_auc_lst = [cal_auc(self.cls_adds_dis[i]) for i in range(self.n_cls)]
        add_s_auc_lst = [cal_auc(self.cls_add_s_dis[i]) for i in range(self.n_cls)]
        n_objs = sum(len(lst) for lst in self.pred_kp_errs)
        all_errs = 0.0
        for c in range(1, self.n_cls):
            all_errs += sum(self.pred_kp_errs[c])
        return dict(add_dis_lst=self.cls_add_dis, adds_dis_lst=self.cls_adds_dis, add_auc_lst=add_auc_lst,
                    adds_auc_lst=adds_auc_lst, add_s_auc_lst=add_s_auc_lst, pred_kp_errs=self.pred_kp_errs,
                    mean_kp_err=all_errs / n_objs if n_objs else float("nan"),
                    add_auc_mean=np.mean(add_auc_lst[1:]), adds_auc_mean=np.mean(adds_auc_lst[1:]),
                    add_s_auc_mean=np.mean(add_s_auc_lst[1:]))

    def cal_lm_add(self, obj_id, diameter, test_occ=False):
        """The LineMOD summary of ``obj_id`` (pvn3d_eval_utils_kpls.py:401-446): the dict the reference pickles --
        the lists, one-entry AUC lists, and ``add`` / ``adds``, the percentage of distances below 0.1 of
        ``diameter`` (the object's ``models_info.yml`` diameter, mm).  ``test_occ`` only named the reference's
        output file and is accepted for its callers."""
        self._add_s_lists([obj_id])
        d = diameter / 1000.0 * 0.1
        return dict(add_dis_lst=self.cls_add_dis, adds_dis_lst=self.cls_adds_dis,
                    add_auc_lst=[cal_auc(self.cls_add_dis[obj_id])], adds_auc_lst=[cal_auc(self.cls_adds_dis[obj_id])],
                    add_s_auc_lst=[cal_auc(self.cls_add_s_dis[obj_id])],
                    add=np.mean(np.array(self.cls_add_dis[obj_id]) < d) * 100,
                    adds=np.mean(np.array(self.cls_adds_dis[obj_id]) < d) * 100)

    def merge_lst(self, targ, src):
        """``targ[i] += src[i]`` for every class; returns ``targ``."""
        for i in range(len(targ)):
            targ[i] += src[i]
        return targ
