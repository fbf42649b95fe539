"""Keypoint voting and pose fitting on the GPU: the step after the network (SURVEY.md §8 f-4).

Mirrors of the reference's evaluation helpers, same names and argument meaning:

* :class:`MeanShiftTorch` -- ``utils/meanshift_pytorch.py:27-57`` (``fit``; ``fit_multi_clus`` is only used by
  that file's own ``__main__`` and is not provided);
* :func:`best_fit_transform` -- ``utils/pvn3d_eval_utils_kpls.py:28-59`` (numpy in, numpy ``[3,4]`` out);
* :func:`cal_frame_poses`, :func:`cal_frame_poses_lm` -- ``utils/pvn3d_eval_utils_kpls.py:65-160, 220-284``;
* :func:`cal_add_cuda`, :func:`cal_adds_cuda`, :func:`cal_auc`, :func:`VOCap` -- ``utils/basic_utils.py:34-46,
  642-669`` (``Basic_Utils`` methods there, functions here);
* :func:`eval_metric`, :func:`eval_metric_lm`, :class:`TorchEval` -- ``utils/pvn3d_eval_utils_kpls.py:162-195,
  287-304, 326-505``: ADD / ADD-S scoring, every object of a frame (``eval_metric``) or of a batch
  (``TorchEval.eval_pose_parallel``) in one :func:`ffb6d_b200.ops.pose_add_adds` launch over a :class:`MeshTable`.

The reference reads mesh keypoints, mesh centres and object radii from dataset files through its module-level
``bs_utils`` / ``config``; here the caller passes them (``mesh_kps``, ``cls_radius``).  Everything numeric runs in
:func:`ffb6d_b200.ops.mean_shift_fit` (one persistent kernel for all keypoints of an object instead of one
N x N torch program per keypoint and a host sync per iteration) and :func:`ffb6d_b200.ops.best_fit_transform`.
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


def _vote_object(pred_ctr, pred_kp, cls_msk, radius, use_ctr, use_ctr_clus_flter):
    """Centre + keypoints of one object: the two clustering steps of pvn3d_eval_utils_kpls.py:122-137."""
    ms = MeanShiftTorch(bandwidth=radius)
    ctr, ctr_labels = ms.fit_batch(pred_ctr[None], cls_msk)
    kp_msk = ctr_labels[0] if use_ctr_clus_flter else cls_msk       # `cls_voted_kps[:, ctr_labels, :]`
    kps, _ = ms.fit_batch(pred_kp, kp_msk)
    return torch.cat((kps, ctr), 0) if use_ctr else kps


def cal_frame_poses(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter, gt_kps=None, gt_ctrs=None,
                    debug=False, kp_type="farthest", *, mesh_kps, cls_radius=None):
    """YCB-style multi-object voting (pvn3d_eval_utils_kpls.py:65-160).

    ``pcld [N,3]``, ``mask [N]`` predicted class ids, ``ctr_of [1,N,3]``, ``pred_kp_of [n_kps,N,3]`` (CUDA).
    ``mesh_kps``: mapping ``cls_id -> [n_kps(+1),3]`` array of object-frame keypoints (the centre last when
    ``use_ctr``), what the reference loads with ``bs_utils.get_kps`` / ``get_ctr``; ``cls_radius``: sequence
    indexed by ``cls_id - 1`` (``config.ycb_r_lst``), needed for the centre-clustering mask filter.
    Returns ``(pred_cls_ids, pred_pose_lst, pred_kps_lst)`` like the reference."""
    n_kps, n_pts, _ = pred_kp_of.shape
    pred_ctr = pcld - ctr_of[0]
    pred_kp = pcld.view(1, n_pts, 3) - pred_kp_of
    radius = 0.04
    pred_cls_ids = np.unique(mask[mask > 0].contiguous().cpu().numpy())
    if use_ctr_clus_flter and len(pred_cls_ids) > 0 and cls_radius is not None:
        # refine the mask: a point takes the class of the nearest voted centre when it is close enough (:85-109)
        ms = MeanShiftTorch(bandwidth=radius)
        msks = torch.stack([mask == int(c) for c in pred_cls_ids])
        ctrs, _ = ms.fit_batch(pred_ctr[None].expand(len(pred_cls_ids), n_pts, 3).contiguous(), msks)
        min_dis, min_idx = torch.cdist(pred_ctr, ctrs).min(dim=1)
        ids_t = torch.as_tensor(pred_cls_ids.astype(np.int64), device=mask.device)
        closest = ids_t[min_idx].to(mask.dtype)
        r = torch.as_tensor(np.asarray(cls_radius, np.float32), device=mask.device)[(ids_t - 1).clamp(min=0)][min_idx]
        update = (mask > 0) & (min_dis < r * 0.8)
        mask = torch.where(update, closest, mask)
    pred_pose_lst, pred_kps_lst = [], []
    for cls_id in pred_cls_ids:
        if cls_id == 0:
            break
        cls_msk = mask == int(cls_id)
        if int(cls_msk.sum()) < 1:
            pred_pose_lst.append(np.identity(4)[:3, :])
            pred_kps_lst.append(np.zeros((n_kps + 1, 3)))
            continue
        kpc = _vote_object(pred_ctr, pred_kp, cls_msk, radius, use_ctr, use_ctr_clus_flter)
        mk = torch.as_tensor(np.asarray(mesh_kps[int(cls_id)], np.float32), device=kpc.device)
        pred_pose_lst.append(ops.best_fit_transform(mk, kpc).cpu().numpy())
        pred_kps_lst.append(kpc.cpu().numpy())
    return pred_cls_ids, pred_pose_lst, pred_kps_lst


def cal_frame_poses_lm(pcld, mask, ctr_of, pred_kp_of, use_ctr, n_cls, use_ctr_clus_flter, obj_id, debug=False, *,
                       mesh_kps):
    """LineMOD-style single-object voting (pvn3d_eval_utils_kpls.py:220-284): class 1 is the object.
    ``mesh_kps [n_kps(+1),3]``: object-frame keypoints of ``obj_id`` (centre last when ``use_ctr``)."""
    n_kps, n_pts, _ = pred_kp_of.shape
    pred_ctr = pcld - ctr_of[0]
    pred_kp = pcld.view(1, n_pts, 3) - pred_kp_of
    cls_msk = mask == 1
    if int(cls_msk.sum()) < 1:
        return [np.identity(4)[:3, :]]
    kpc = _vote_object(pred_ctr, pred_kp, cls_msk, 0.04, use_ctr, use_ctr_clus_flter)
    mk = torch.as_tensor(np.asarray(mesh_kps, np.float32), device=kpc.device)
    return [ops.best_fit_transform(mk, kpc).cpu().numpy()]


# ---------------------------------------------------------------------------------------------------- pose scoring
class MeshTable:
    """The meshes that ADD / ADD-S are computed over, resident on the GPU and indexed by class id.

    ``mesh_pts``: mapping ``cls_id -> [P,3]`` vertices in metres, what the reference's ``bs_utils.get_pointxyz(_cuda)``
    returns (YCB: ``models/<cls>/points.xyz``; LineMOD: the 2 000-vertex subsample the caller drew, the reference
    redraws it in every process).  Holds ``pts [sum P,3]`` float32, ``off [max id + 2]`` int32 (mesh ``c`` is rows
    ``off[c] .. off[c+1]``; ids without a mesh are empty, and scoring one gives NaN) and ``max_points``."""

    def __init__(self, mesh_pts, device=None):
        if not mesh_pts:
            raise ValueError("MeshTable needs at least one mesh")
        ids = sorted(int(c) for c in mesh_pts)
        if ids[0] < 0:
            raise ValueError("class ids must be >= 0, got %d" % ids[0])
        arrs = {int(c): np.asarray(torch.as_tensor(v).detach().cpu(), np.float32) for c, v in mesh_pts.items()}
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


class TorchEval:
    """The reference's ``TorchEval`` (pvn3d_eval_utils_kpls.py:326-505): per-class ADD / ADD-S lists over a test run
    and their AUCs.

    The constructor takes what the reference reads from its module-level ``config`` / ``bs_utils``: ``mesh_pts``
    (mapping ``cls_id -> [P,3]``, the scoring meshes; LineMOD: keyed by ``obj_id``), ``mesh_kps`` (mapping
    ``cls_id -> [n_kps(+1),3]``, see :func:`cal_frame_poses`), ``cls_radius`` (``config.ycb_r_lst``) and
    ``sym_cls_ids`` (``config.ycb_sym_cls_ids`` or ``config_lm.lm_sym_cls_ids``).

    :meth:`eval_pose_parallel` votes each frame with :func:`cal_frame_poses` / :func:`cal_frame_poses_lm` and then
    scores every object of the batch in one :func:`ffb6d_b200.ops.pose_add_adds` launch; the lists grow frame by
    frame, object by object, as the reference's ``executor.map`` makes them.  :meth:`cal_auc` and :meth:`cal_lm_add`
    return the dict the reference pickles plus the averages it prints; they print nothing and write no file.

    One deliberate difference: the reference's ``cal_auc`` / ``cal_lm_add`` append to ``cls_add_s_dis[0]`` on every
    call, so a second call counts the objects twice.  Here the ADD(-S) lists are rebuilt on each call; a single call
    gives the reference's result."""

    def __init__(self, mesh_pts, mesh_kps, cls_radius=None, sym_cls_ids=(), n_cls=22):
        self.n_cls = n_cls
        self.mesh_table = MeshTable(mesh_pts)
        self.mesh_kps = mesh_kps
        self.cls_radius = cls_radius
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
        reference."""
        bs = pred_kp_ofs.shape[0]
        masks = masks.long()
        ids_h = _ids_column(cls_ids.reshape(-1, 1)).reshape(bs, -1)
        cls, poses, where, per_frame = [], [], [], []
        if ds == "ycb":
            gt_kps_h = gt_kps.detach().cpu().numpy()
            for b in range(bs):
                pred_cls_ids, pred_poses, pred_kpcs = cal_frame_poses(
                    pclds[b], masks[b], pred_ctr_ofs[b], pred_kp_ofs[b], use_ctr, self.n_cls, use_ctr_clus_flter,
                    gt_kps[b], gt_ctrs[b], kp_type=kp_type, mesh_kps=self.mesh_kps, cls_radius=self.cls_radius)
                self.pred_id2pose_lst.append({cid: pose for cid, pose in zip(pred_cls_ids, pred_poses)})
                c, p, e = _frame_objects(ids_h[b], pred_poses, pred_cls_ids, gt_kps_h[b], pred_kpcs)
                per_frame.append((c, e))
                cls += c
                poses += p
                where += [b * RTs.shape[1] + i for i in range(len(c))]
        else:
            for b in range(bs):
                pose = cal_frame_poses_lm(pclds[b], masks[b], pred_ctr_ofs[b], pred_kp_ofs[b], use_ctr, self.n_cls,
                                          use_ctr_clus_flter, obj_id, mesh_kps=self.mesh_kps[obj_id])[0]
                per_frame.append(([int(obj_id)], None))
                cls.append(int(obj_id))
                poses.append(np.asarray(pose).astype(np.float32))
                where.append(b * RTs.shape[1])
        sel = torch.as_tensor(np.asarray(where, np.int64)).to(RTs.device)
        add, adds = _score(self.mesh_table, cls, poses, RTs.reshape(-1, 3, 4)[sel])
        k = 0
        for c, errs in per_frame:
            for j, cid in enumerate(c):
                if errs is not None:
                    self.pred_kp_errs[cid].append(errs[j])
                for i in (cid, 0):
                    self.cls_add_dis[i].append(add[k])
                    self.cls_adds_dis[i].append(adds[k])
                k += 1

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
