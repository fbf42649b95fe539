"""Object poses from decoded RGB-D frames: the inference ``get_item``, the ``FFB6D`` eval forward and the voting in
one call, eager (:func:`estimate_poses`) or replayed from one CUDA graph per batch (:class:`GraphedPoseStep`,
DESIGN.md §4.27).

    model = FFB6D(n_classes=22).cuda().eval()
    load_reference_checkpoint(model, "FFB6D_best.pth.tar")
    table = pose.VoteTable(mesh_kps, 22, cls_radius)
    step = GraphedPoseStep(model, frames, dataset="ycb", cam_scale=10000.0, K=K, mesh_kps=table)
    for frames in stream_of_batches:          # {"dpt": uint16 [B,H,W], "rgb": uint8 [B,H,W,3], "nrm_map": [B,H,W,3]}
        out = step(frames)                    # present, count, kps, poses, valid: device tensors

One estimate is what the reference's ``demo.py`` does per frame (demo.py:85-113): the dataset's ``get_item`` without
labels (:func:`ffb6d_b200.schedule.build_ffb6d_inputs`), ``rgb`` cast to float32 as ``model_fn`` casts it,
``model(item)`` in eval mode under ``torch.no_grad()``, ``torch.max(pred_rgbd_segs, 1)[1]`` as the mask,
``cld_rgb_nrm[:, :3]`` as the cloud, and the vote.  The dataset fixes the depth handling and the vote:

* ``"ycb"``: depth completion (``fill=True``); :func:`ffb6d_b200.pose.cal_batch_poses` with ``use_ctr=True`` and
  ``use_ctr_clus_flter=True`` over every class of the model;
* ``"linemod"``: the raw depth (``fill=False``); the two-class vote on ``mask == 1`` without refinement, as
  ``cal_frame_poses_lm`` (``n_cls = 2``, the object at row 1).

Normals are an input (``nrm_map``) by default: the reference computes them with the external ``normalSpeed`` (YCB from
the completed depth, see INTEGRATION.md).  With ``normals="device"`` the frames hold no ``nrm_map`` and the normals
are computed on the device from that same depth (:func:`ffb6d_b200.ops.depth_normal`, DESIGN.md §4.30).
"""
import torch

from . import pose as _pose
from .graphed import _GraphedEvalBase, _check_image_branch
from .ops import _frame_intrinsics, _intrinsics_arg
from .schedule import build_ffb6d_inputs, check_dataset, check_frame_batch

# the reference's config.n_sample_points (common.py:61)
N_SAMPLE_POINTS = 480 * 640 // 24

_FRAME_KEYS = ("dpt", "rgb", "nrm_map")


def vote_table(dataset, mesh_kps, n_cls, cls_radius=None, device=None):
    """The :class:`ffb6d_b200.pose.VoteTable` a dataset's vote reads: ``mesh_kps`` itself when it is one; for YCB
    the table of the mapping ``cls_id -> [n_kps+1,3]`` over ``n_cls`` classes with ``cls_radius``; for LineMOD the
    two-class table of the object's ``[n_kps+1,3]`` keypoints (class 1)."""
    if isinstance(mesh_kps, _pose.VoteTable):
        return mesh_kps
    if dataset == "ycb":
        return _pose.VoteTable(mesh_kps, n_cls, cls_radius, device)
    return _pose._lm_table(mesh_kps, device)


def forward_and_vote(model, item, dataset, mesh_kps, cls_radius=None):
    """The steps after the item: ``model(item)`` under ``torch.no_grad()``, ``torch.max(pred_rgbd_segs, 1)[1]`` as
    the mask, ``cld_rgb_nrm[:, :3]`` as the cloud and the dataset's vote (see the module).  The model is used in the
    mode it is in.  ``mesh_kps``: a :class:`~ffb6d_b200.pose.VoteTable`, or what :func:`vote_table` builds one from
    (``n_cls`` from the network's output).

    Returns ``(end_points, table, (present, count, kps, poses))`` with :func:`~ffb6d_b200.pose.cal_batch_poses`'
    shapes (LineMOD: two classes, the object at row 1)."""
    with torch.no_grad():
        end_points = model(item)
        segs = end_points["pred_rgbd_segs"]
        classes = torch.max(segs, 1)[1]
        pcld = item["cld_rgb_nrm"][:, :3, :].permute(0, 2, 1).contiguous()
        table = vote_table(dataset, mesh_kps, segs.shape[1], cls_radius, segs.device)
        ctr, kp = end_points["pred_ctr_ofs"], end_points["pred_kp_ofs"]
        if dataset == "ycb":
            votes = _pose.cal_batch_poses(pcld, classes, ctr, kp, True, table.n_cls, True, mesh_kps=table)
        else:
            votes = _pose._vote(table, pcld, classes == 1, ctr, kp, True, False, False)
    return end_points, table, votes


def _estimate(model, frames, dataset, cam_scale, intr, table, n_points, seed, normals):
    """One estimate from checked frames, with device intrinsics ``intr`` and a device vote table."""
    item = build_ffb6d_inputs(frames["dpt"], cam_scale, intr, frames["rgb"], frames.get("nrm_map"), n_points, seed=seed,
                              fill=dataset == "ycb", normals=normals)
    item["rgb"] = item["rgb"].to(torch.float32)             # model_fn's cast of the uint8 image
    _, _, (present, count, kps, poses) = forward_and_vote(model, item, dataset, table)
    return dict(present=present, count=count, kps=kps, poses=poses, valid=item["valid"])


def _prepare(model, frames, dataset, K, mesh_kps, cls_radius):
    """The device intrinsics (None with per-frame ``frames['K']``) and the device vote table of checked frames."""
    dev = frames["dpt"].device
    intr = None if "K" in frames else _intrinsics_arg(K, frames["dpt"].shape[0], dev)[0]
    table = vote_table(dataset, mesh_kps, getattr(getattr(model, "module", model), "n_cls", None), cls_radius, dev)
    return intr, table


def estimate_poses(model, frames, *, dataset, cam_scale, K, mesh_kps, cls_radius=None, n_points=N_SAMPLE_POINTS,
                   seed=0, normals="input"):
    """The object poses of a batch of decoded RGB-D frames, eager: the composition the module describes.

    :param model: an :class:`~ffb6d_b200.model.FFB6D`; it is switched to eval mode, as the reference's demo does
    :param frames: dict of CUDA tensors ``dpt`` uint16 ``[B,H,W]`` (raw depth), ``rgb`` uint8 ``[B,H,W,3]``,
      ``nrm_map`` float32 / float64 ``[B,H,W,3]`` and optionally ``K`` float64 ``[B,3,3]``, one camera matrix per
      frame (it replaces ``K``)
    :param dataset: ``"ycb"`` or ``"linemod"``; :param cam_scale: raw depth units per metre (YCB
      ``meta['factor_depth']``, LineMOD 1000)
    :param K: the camera matrix ``[3,3]`` / ``[B,3,3]``, or device intrinsics as
      :func:`ffb6d_b200.ops.backproject` takes them
    :param mesh_kps: a :class:`~ffb6d_b200.pose.VoteTable`; or YCB the mapping ``cls_id -> [n_kps+1,3]`` object-frame
      keypoints (centre last), LineMOD the ``[n_kps+1,3]`` keypoints of the object
    :param cls_radius: YCB ``config.ycb_r_lst``, for the centre-clustering refinement (None: no refinement)
    :param n_points: points sampled per frame, the reference's 12800 by default; :param seed: the sampling seed
    :param normals: ``"input"``: ``frames['nrm_map']`` is the normal map; ``"device"``: the frames hold no ``nrm_map``
      and :func:`ffb6d_b200.build_ffb6d_inputs` computes it from the depth
    :return: dict of CUDA tensors ``present [B,n_cls]`` bool, ``count [B,n_cls]`` int32, ``kps [B,n_cls,n_kps+1,3]``
      float32, ``poses [B,n_cls,3,4]`` float64 (rows as :func:`~ffb6d_b200.pose.cal_batch_poses` gives them;
      LineMOD ``n_cls = 2``, the object at row 1) and ``valid [B]`` bool (False: fewer than 400 valid depth pixels,
      where the reference's loader would skip the frame; its rows are computed all the same).

    With ``K`` as device intrinsics (or ``frames['K']``) and ``mesh_kps`` a ``VoteTable``, the call makes no host
    synchronisation; a host ``K`` or a mapping is first copied to the device, which synchronises."""
    check_dataset(dataset, "estimate_poses")
    _check_image_branch(model, "estimate_poses")
    check_frame_batch(frames, "estimate_poses", _FRAME_KEYS, normals)
    intr, table = _prepare(model, frames, dataset, K, mesh_kps, cls_radius)
    model.eval()
    if intr is None:
        intr = _frame_intrinsics(frames["K"])
    return _estimate(model, frames, dataset, cam_scale, intr, table, n_points, seed, normals)


class GraphedPoseStep(_GraphedEvalBase):
    """:func:`estimate_poses` captured in one CUDA graph and replayed per batch: the depth completion (YCB), the
    sampling, the 22 searches, the point features, the ``FFB6D`` eval forward, the argmax and the vote.

    :param example_frames: frames as :func:`estimate_poses` takes them; every tensor gets a static input buffer of
      its shape, dtype and device, and later frames must match them (the last, short batch of a test set is padded
      by the caller, or goes through :func:`estimate_poses`)
    :param warmup: eager estimates run on a side stream before the first capture

    Baked in at construction: ``dataset``, ``cam_scale``, ``n_points``, ``normals``, ``seed`` (so the same frame gives the same
    points on every replay, as :func:`estimate_poses` with that seed does), ``K`` (copied to the device once; with
    ``frames['K']`` the per-frame matrices are inputs instead) and the vote table (built from ``mesh_kps`` and
    ``cls_radius`` once, or the given :class:`~ffb6d_b200.pose.VoteTable`).

    Calling the step copies the frames into the input buffers on the current stream, compares what capture baked
    into the model (the rules of :class:`~ffb6d_b200.graphed.GraphedEvalStep`, DESIGN.md §4.21: weights changed in
    place or by ``load_state_dict`` need no new capture, a switched path flag or module does) and replays.  It
    returns :func:`estimate_poses`' dict: the graph's output tensors, which the next replay overwrites (clone what
    you keep).  ``captures`` counts the captures.

    Rejected with ``ValueError``: a model in training mode; a ``DistributedDataParallel`` / ``DataParallel``
    wrapper; an ``FFB6DFusionNet`` (no image branch); ``FFB6D_CHECK_INDICES`` set now or when the library loaded;
    frames whose keys, shapes, dtypes or devices differ from the example's.
    """

    _needs_image_branch = True

    def __init__(self, model, example_frames, *, dataset, cam_scale, K, mesh_kps, cls_radius=None,
                 n_points=N_SAMPLE_POINTS, seed=0, warmup=3, normals="input"):
        name = type(self).__name__
        check_dataset(dataset, name)
        self._check_model(model)
        check_frame_batch(example_frames, name, _FRAME_KEYS, normals)
        self._intr, self._table = _prepare(model, example_frames, dataset, K, mesh_kps, cls_radius)
        self.dataset, self.cam_scale, self.n_points, self.seed = dataset, cam_scale, int(n_points), int(seed)
        self.normals = normals
        self._keys = set(example_frames)
        super().__init__(model, example_frames, warmup)

    def _step(self):
        frames = self._static
        intr = _frame_intrinsics(frames["K"]) if "K" in frames else self._intr
        return _estimate(self.model, frames, self.dataset, self.cam_scale, intr, self._table, self.n_points,
                         self.seed, self.normals)
