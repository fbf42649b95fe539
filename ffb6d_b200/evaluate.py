"""The reference's test run from decoded frames, one CUDA graph replay per batch (:class:`GraphedTestStep`, DESIGN.md
§4.29).

    step = GraphedTestStep(model.eval(), batches[0], dataset="ycb", cam_scale=10000.0, K=K, mesh_pts=mesh_pts,
                           mesh_kps=mesh_kps, cls_radius=ycb_r_lst, sym_cls_ids=ycb_sym_cls_ids, capacity=len(test_set))
    for batch in loader:                       # decoded frames and object tables, as CUDA tensors
        end_points, loss, info = step(batch)   # get_item, forward, loss, vote, ADD / ADD-S and the record
    res = step.summary()                       # TorchEval.cal_auc()'s dict, eval_epoch's means; one synchronise

One replay is one batch of ``train_ycb.py -eval_net -test -test_pose`` (``train_lm.py ... -test``): the eval
``get_item`` (:func:`ffb6d_b200.build_ffb6d_item`, depth completion for YCB only, no augmentation), ``model(item)``
under ``torch.no_grad()``, ``ffb6d_loss`` masked by ``valid`` with ``acc_rgbd``, the vote ``model_fn`` calls (YCB
every class, ``use_ctr=True``, ``use_ctr_clus_flter=True``; LineMOD ``mask == 1`` of ``obj_id``), the scoring and the
record of every object in a device table (:func:`ffb6d_b200.ops.eval_record`).  The losses and ``acc_rgbd`` are
summed on the device; the AUC tables are computed there at the end (:func:`ffb6d_b200.ops.eval_auc`).
"""
import numpy as np
import torch

from . import _lib, ops
from . import pose as _pose
from .estimate import N_SAMPLE_POINTS
from .graphed import _GraphedEvalBase
from .loss import ffb6d_loss
from .ops import _frame_intrinsics, _intrinsics_arg
from .schedule import _OBJECT_KEYS, build_ffb6d_item, check_dataset, check_frame_batch

_IMAGE_KEYS = ("dpt", "rgb", "labels", "nrm_map")
_INFO_KEYS = ("loss_rgbd_seg", "loss_kp_of", "loss_ctr_of", "loss_all", "acc_rgbd")
# the lists of the reference's TorchEval: config.n_classes
_LM_LIST_CLASSES = 22


class GraphedTestStep(_GraphedEvalBase):
    """One batch of the reference's test, captured in one CUDA graph and replayed per batch (see the module).

    :param model: an :class:`~ffb6d_b200.model.FFB6D` in eval mode
    :param example_batch: dict of CUDA tensors ``dpt`` uint16 ``[B,H,W]``, ``rgb`` uint8 ``[B,H,W,3]``, ``labels``
      uint8 ``[B,H,W]``, ``nrm_map`` ``[B,H,W,3]``, the object tables of :func:`ffb6d_b200.item.pose_gt_objects`
      (``RTs``, ``kp_3ds``, ``ctr_3ds``, ``cls_ids``, ``obj_cls``, ``obj_kps``, ``obj_ctr``) and optionally ``K``
      float64 ``[B,3,3]`` (one camera matrix per frame; it replaces ``K``).  Every tensor gets a static input buffer;
      later batches must have the same keys, shapes and dtypes.
    :param dataset: ``"ycb"`` or ``"linemod"``; :param cam_scale: raw depth units per metre; :param K: the camera
      matrix as :func:`ffb6d_b200.build_ffb6d_item` takes it
    :param mesh_pts, mesh_kps, cls_radius, sym_cls_ids: as :class:`ffb6d_b200.pose.TorchEval` takes them (LineMOD:
      keyed by ``obj_id``)
    :param n_points: points sampled per frame; :param seed: the sampling seed (baked in, as in
      :class:`~ffb6d_b200.estimate.GraphedPoseStep`)
    :param capacity: the most frames one test run records (``len(test_set)``); the table holds ``capacity * n_obj``
      object rows
    :param test_gt: vote from the labels and target offsets instead of the predictions (``-test_gt``)
    :param obj_id: the LineMOD object's class id (``config.cls_id``)
    :param normals: ``"input"``: the batch's ``nrm_map``; ``"device"``: the batch holds no ``nrm_map`` and the normals
      are computed from the depth (:func:`ffb6d_b200.build_ffb6d_item`)

    ``step(batch)`` copies the batch into the input buffers and replays; it returns ``(end_points, loss, info)``,
    graph-owned device tensors that the next replay overwrites, and does not synchronise.  :meth:`summary`
    synchronises once and returns the test's results; :meth:`reset` starts a new run.  What capture bakes into the
    model is compared before every replay, as :class:`~ffb6d_b200.graphed.GraphedEvalStep` does (DESIGN.md §4.21).

    Rejected with ``ValueError`` before any CUDA work: a model in training mode; a ``DistributedDataParallel`` /
    ``DataParallel`` wrapper; an ``FFB6DFusionNet``; ``FFB6D_CHECK_INDICES`` set; an unknown dataset, a LineMOD
    step without ``obj_id``, a capacity below 1 or above the table's limit; a batch whose keys, shapes, dtypes or
    devices differ from the example's.
    """

    _needs_image_branch = True

    def __init__(self, model, example_batch, *, dataset, cam_scale, K, mesh_pts, mesh_kps, cls_radius=None,
                 sym_cls_ids=(), n_points=N_SAMPLE_POINTS, capacity, test_gt=False, obj_id=None, seed=0, warmup=3,
                 normals="input"):
        name = type(self).__name__
        self._check_model(model)
        self.model = model
        self._check()
        check_dataset(dataset, name)
        lm = dataset == "linemod"
        if lm and (isinstance(obj_id, bool) or not isinstance(obj_id, (int, np.integer)) or obj_id < 1):
            raise ValueError("%s: a LineMOD test needs obj_id, the object's class id >= 1, got %r" % (name, obj_id))
        if isinstance(capacity, bool) or not isinstance(capacity, (int, np.integer)) or capacity < 1:
            raise ValueError("%s: capacity must be an int >= 1 (frames), got %r" % (name, capacity))
        check_frame_batch(example_batch, name, _IMAGE_KEYS + _OBJECT_KEYS, normals)
        self.normals = normals
        B, n_obj = example_batch["RTs"].shape[:2]
        if capacity * n_obj > _lib.EVAL_MAX_ROWS:
            raise ValueError("%s: capacity * n_obj = %d rows, at most %d" % (name, capacity * n_obj,
                                                                              _lib.EVAL_MAX_ROWS))
        dev = example_batch["dpt"].device
        self.dataset, self.cam_scale, self.n_points, self.seed = dataset, cam_scale, int(n_points), int(seed)
        self.test_gt, self.capacity, self._n_obj = bool(test_gt), int(capacity), int(n_obj)
        self.obj_id = int(obj_id) if lm else 0
        self._keys = set(example_batch)
        self._mesh = _pose.MeshTable(mesh_pts, dev)
        if lm:
            kp = mesh_kps[self.obj_id] if isinstance(mesh_kps, dict) else mesh_kps
            self._table = _pose._lm_table(kp, dev)
            self.n_cls = max(_LM_LIST_CLASSES, self.obj_id + 1)
        else:
            self.n_cls = int(model.n_cls)
            self._table = _pose.VoteTable({c: k for c, k in mesh_kps.items() if 0 <= int(c) < self.n_cls},
                                          self.n_cls, cls_radius, dev)
        self.sym_cls_ids = [int(c) for c in sym_cls_ids]
        sym = np.zeros(self.n_cls, np.uint8)
        sym[[c for c in self.sym_cls_ids if 0 <= c < self.n_cls]] = 1
        self._sym = torch.as_tensor(sym, device=dev)
        self._intr = None if "K" in example_batch else _intrinsics_arg(K, B, dev)[0]
        self._rows = torch.zeros((self.capacity * n_obj, _lib.EVAL_ROW_WORDS), dtype=torch.int32, device=dev)
        self._state = torch.zeros(4, dtype=torch.int64, device=dev)
        self._frame_poses = self._frame_flags = None
        if not lm:
            self._frame_poses = torch.zeros((self.capacity, self.n_cls, 3, 4), dtype=torch.float64, device=dev)
            self._frame_flags = torch.zeros((self.capacity, self.n_cls), dtype=torch.uint8, device=dev)
        self._sums = torch.zeros(len(_INFO_KEYS) + 1, dtype=torch.float64, device=dev)
        self._one = torch.ones(1, dtype=torch.float64, device=dev)
        super().__init__(model, example_batch, warmup)

    # ------------------------------------------------------------------------------------------ capture
    def _step(self):
        b = self._static
        intr = _frame_intrinsics(b["K"]) if "K" in b else self._intr
        item = build_ffb6d_item(b["dpt"], self.cam_scale, intr, b["rgb"], b["labels"], b.get("nrm_map"), b,
                                self.n_points, seed=self.seed, fill=self.dataset == "ycb", normals=self.normals)
        item["rgb"] = item["rgb"].float()                     # model_fn's cast
        with torch.no_grad():
            end_points = self.model(item)
            loss, info = ffb6d_loss(end_points, item, valid=item["valid"])
            self._sums += torch.cat([torch.stack([info[k] for k in _INFO_KEYS]).double(), self._one])
            pcld = item["cld_rgb_nrm"][:, :3, :].permute(0, 2, 1).contiguous()
            if self.test_gt:        # train_ycb.py:284-293, train_lm.py:306-317
                mask = item["labels"]
                ctr = item["ctr_targ_ofst"].unsqueeze(2).permute(0, 2, 1, 3)
                kp = item["kp_targ_ofst"].permute(0, 2, 1, 3)
            else:
                mask = torch.max(end_points["pred_rgbd_segs"], 1)[1]
                ctr, kp = end_points["pred_ctr_ofs"], end_points["pred_kp_ofs"]
            if self.dataset == "ycb":
                votes, ids, pred, add, adds = _pose._ycb_scores(self._mesh, self._table, pcld, mask, ctr, kp,
                                                                item["cls_ids"], item["RTs"], True, True)
                _pose._ycb_record(self._rows, self._state, votes, ids, pred, add, adds, item["kp_3ds"],
                                  valid=item["valid"], frame_poses=self._frame_poses, frame_flags=self._frame_flags)
            else:
                votes, pred, add, adds = _pose._lm_scores(self._mesh, self._table, self.obj_id, pcld, mask, ctr, kp,
                                                          item["RTs"], True, True)
                _pose._lm_record(self._rows, self._state, votes, self.obj_id, self._n_obj, pred, add, adds,
                                 valid=item["valid"])
        return end_points, loss, info

    def _warm_up(self, n):
        """The warm-up with what it recorded undone, so a capture in the middle of a run (after a baked value
        changed) leaves the run's table and sums as they were."""
        saved = (self._state.clone(), self._sums.clone())
        super()._warm_up(n)
        self._state.copy_(saved[0])
        self._sums.copy_(saved[1])

    # ------------------------------------------------------------------------------------------ a run
    def reset(self):
        """Start a new test run: the table and the sums are emptied on the device, the graph is kept."""
        self._state.zero_()
        self._sums.zero_()

    def summary(self, diameter=None):
        """The run's results, after one synchronisation.

        YCB: the dict of :meth:`ffb6d_b200.pose.TorchEval.cal_auc`; LineMOD: that of
        :meth:`~ffb6d_b200.pose.TorchEval.cal_lm_add` for ``obj_id`` with ``diameter`` (the object's diameter, mm).
        Both add ``mean_eval_dict`` (``eval_epoch``'s per-key means over the batches, ``acc_rgbd`` times 100, and
        ``loss_target``) and ``pred_id2pose_lst`` (YCB: each valid frame's ``{class id: pose}``; LineMOD: empty).
        Frames with ``valid == False`` are left out of every list.  Raises ``RuntimeError`` when a batch did not fit
        in ``capacity`` frames."""
        lm = self.dataset == "linemod"
        if lm and diameter is None:
            raise ValueError("%s.summary: a LineMOD summary needs the object's diameter (mm)" % type(self).__name__)
        lm_thr = diameter / 1000.0 * 0.1 if lm else 0.0
        auc, pct, kp = ops.eval_auc(self._rows, self._state, self.n_cls, self._sym, lm_thr)
        extra = () if lm else (self._frame_poses, self._frame_flags)
        state, auc, pct, kp, sums, rows, *frames = _pose._to_host(self._state, auc, pct, kp, self._sums, self._rows,
                                                                  *extra)
        if state[2]:
            raise RuntimeError("%s: a batch did not fit in the table of %d frames; it was not recorded (build the "
                               "step with a larger capacity)" % (type(self).__name__, self.capacity))
        n = self.n_cls
        add_dis, adds_dis, kp_errs = ([[] for _ in range(n)] for _ in range(3))
        _pose._append_rows(rows[:state[0]], add_dis, adds_dis, None if lm else kp_errs)
        add_s_dis = [[] for _ in range(n)]
        for c in ([self.obj_id] if lm else range(1, n)):
            add_s_dis[c] = list(adds_dis[c] if c in self.sym_cls_ids else add_dis[c])
            add_s_dis[0] += add_s_dis[c]
        nb = sums[-1]
        means = {k: sums[i] / nb * (100 if "acc" in k else 1) if nb else float("nan") for i, k in enumerate(_INFO_KEYS)}
        means["loss_target"] = means["loss_all"]
        pred_id2pose_lst = []
        if not lm:
            poses, flags = frames
            for f in range(int(state[1])):
                if flags[f, 0] & 2:
                    pred_id2pose_lst.append({c: poses[f, c] for c in np.flatnonzero(flags[f] & 1)})
        lst = lambda a: [float(x) for x in a]        # noqa: E731
        if lm:
            o = self.obj_id
            res = dict(add_dis_lst=add_dis, adds_dis_lst=adds_dis, add_auc_lst=[float(auc[0, o])],
                       adds_auc_lst=[float(auc[1, o])], add_s_auc_lst=[float(auc[2, o])], add=float(pct[0, o]),
                       adds=float(pct[1, o]))
        else:
            res = dict(add_dis_lst=add_dis, adds_dis_lst=adds_dis, add_auc_lst=lst(auc[0]), adds_auc_lst=lst(auc[1]),
                       add_s_auc_lst=lst(auc[2]), pred_kp_errs=kp_errs,
                       mean_kp_err=float(kp[0] / kp[1]) if kp[1] else float("nan"),
                       add_auc_mean=np.mean(auc[0, 1:]), adds_auc_mean=np.mean(auc[1, 1:]),
                       add_s_auc_mean=np.mean(auc[2, 1:]))
        res.update(mean_eval_dict=means, pred_id2pose_lst=pred_id2pose_lst)
        return res
