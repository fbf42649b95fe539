"""ffb6d_b200 -- H100 (sm_90a) implementation of FFB6D's bidirectional-fusion hot path.

Public surface (same names and argument meaning as the reference, ethnhe/FFB6D):

* :func:`knn_search` -- ``DataProcessing.knn_search`` (models/RandLA/helper_tool.py:160-170)
* :func:`random_sample`, :func:`nearest_interpolation` -- ``FFB6D.random_sample`` /
  ``FFB6D.nearest_interpolation`` (models/ffb6d.py:159-194) and the RandLA twins
  (models/RandLA/RandLANet.py:87-117)
* :func:`gather_neighbour`, :func:`relative_pos_encoding` -- ``Building_block`` helpers
  (models/RandLA/RandLANet.py:216-234)
* :func:`grid_sub_sampling` -- ``DataProcessing.grid_sub_sampling`` (helper_tool.py:199-219)
* :func:`build_ffb6d_indices` -- the 22-call KNN schedule of the datasets
  (datasets/ycb/ycb_dataset.py:269-309) run on the GPU in one go.
* :func:`fill_missing` -- ``Basic_Utils.fill_missing`` (utils/basic_utils.py:467-487) as the YCB dataset calls it
  (datasets/ycb/ycb_dataset.py:204); :func:`build_ffb6d_indices_from_raw_depth` -- the depth half of its
  ``get_item`` from the raw depth PNG to the 22 index tensors.
* :func:`build_ffb6d_item` -- the datasets' whole ``get_item`` for a batch on the GPU (:func:`point_item` builds
  the sampled points' input and pose targets; :func:`pose_gt_objects` is the per-object half that stays on the host).
* :func:`rgb_add_noise`, :func:`add_real_back` -- the datasets' synthetic-frame augmentation
  (datasets/ycb/ycb_dataset.py:79-163, datasets/linemod/linemod_dataset.py:114-186) on the GPU; the scalar draws stay
  in the worker (:mod:`ffb6d_b200.augment`).  :func:`color_jitter` -- the datasets' ``trancolor``
  (torchvision ``ColorJitter``) on the GPU, from plans of :func:`ffb6d_b200.augment.draw_color_jitter`.
* :mod:`ffb6d_b200.pose` -- ``MeanShiftTorch``, ``best_fit_transform``, ``cal_batch_poses``, ``cal_frame_poses(_lm)``
  (utils/meanshift_pytorch.py:27-57, utils/pvn3d_eval_utils_kpls.py:28-160, 220-284): keypoint voting on the GPU;
  ``cal_add_cuda``, ``cal_adds_cuda``, ``cal_auc``, ``eval_metric(_lm)`` and ``TorchEval`` (utils/basic_utils.py:34-46,
  642-669, utils/pvn3d_eval_utils_kpls.py:162-195, 287-304, 326-505): the ADD / ADD-S scoring of a whole batch in
  one :func:`pose_add_adds` launch.
* :mod:`ffb6d_b200.loss` -- ``FocalLoss``, ``of_l1_loss``, ``OFLoss`` (models/loss.py:12-90) and
  :func:`~ffb6d_b200.loss.ffb6d_loss`, ``model_fn``'s loss block, masked by the batch's valid frames.
* :mod:`ffb6d_b200.cnn` -- the ResNet34-PSPNet image branch (models/cnn/extractors.py, models/cnn/pspnet.py) in
  torch, with :func:`psp_pool`, :func:`psp_bottleneck` and :func:`conv1x1_log_softmax` on the GPU for its PSP head
  and ``final`` at inference, and their adjoints (:func:`psp_bottleneck_bwd`, :func:`psp_pool_bwd`,
  :func:`log_softmax_bwd`, :func:`upsample_bilinear2d_bwd`) for deterministic training;
  ``ffb6d_b200.model.FFB6D`` is the whole network.
* :class:`GraphedTrainStep` (:mod:`ffb6d_b200.graphed`) -- a whole training step of ``FFB6DFusionNet`` / ``FFB6D``
  (forward, ``ffb6d_loss``, backward, optimizer update) captured in one CUDA graph and replayed per batch;
  :class:`GraphedEvalStep` -- the eval forward and its ``ffb6d_loss`` the same way, for validation and testing;
  :class:`GraphedFrameTrainStep` -- :func:`build_ffb6d_train_item` (the training ``get_item`` with its augmentation,
  from decoded frames) and the training step in one graph.
* :func:`farthest_point_sampling` -- ``fps_utils.farthest_point_sampling`` (utils/dataset_tools/fps/fps_utils.py:8-23)
  on the GPU, batched over clouds; :mod:`ffb6d_b200.objinfo` -- the object tables of
  utils/dataset_tools/gen_obj_info.py (box corners, radius, centre, keypoints) and their text files.
* :mod:`ffb6d_b200.vis` -- ``Basic_Utils.project_p3d`` / ``draw_p2ds`` / ``get_label_color`` (utils/basic_utils.py:
  268-295, 362-423) batched on the GPU, demo.py's ``cal_view_pred_pose`` for a whole batch and the trainers'
  ``view_labels``.
* :func:`estimate_poses` (:mod:`ffb6d_b200.estimate`) -- decoded RGB-D frames in, object poses out: the inference
  ``get_item`` (:func:`build_ffb6d_inputs`, no labels), the ``FFB6D`` eval forward and the voting, as the
  reference's ``demo.py`` composes them; :class:`GraphedPoseStep` -- all of it captured in one CUDA graph and
  replayed per batch.
* :class:`GraphedTestStep` (:mod:`ffb6d_b200.evaluate`) -- one batch of the reference's test (the eval ``get_item``,
  the forward, the loss, the vote, ADD / ADD-S and a device record of every object) replayed from one CUDA graph,
  and the AUC tables of the run computed on the GPU (:func:`eval_record`, :func:`eval_auc`).
* :func:`depth_normal` -- surface normals of millimetre depth maps on the GPU (DESIGN.md §4.30), the opt-in stand-in
  for the datasets' ``normalSpeed.depth_normal``; every item builder and graphed step from frames takes
  ``normals="device"`` to compute them from the depth the reference uses.
* :func:`render_rgbd` (:mod:`ffb6d_b200.render`) -- synthetic RGB-D frames of vertex-coloured meshes on the GPU, a
  z-buffer rasteriser (DESIGN.md §4.31) standing in for LineMOD's pre-rendered ``render`` pickles;
  :func:`build_ffb6d_train_item` and :class:`GraphedFrameTrainStep` take ``meshes=`` a
  :class:`~ffb6d_b200.render.RenderMeshTable` to render flagged frames of a batch.  A
  :class:`~ffb6d_b200.render.TexturedMeshTable` renders UV-mapped, mipmapped meshes through the same call (DESIGN.md
  §4.35), the renders of the dataset tool's pyrender path behind ``objinfo.textured_kp3ds``.
* :func:`fuse_rgbd` (:mod:`ffb6d_b200.fuse_frames`) -- LineMOD's ``fuse`` frames on the GPU: object crops of real
  frames pasted into a frame (DESIGN.md §4.34); :func:`build_ffb6d_train_item` and :class:`GraphedFrameTrainStep`
  take ``crops=`` a :class:`~ffb6d_b200.fuse_frames.FuseCropTable` to compose flagged frames of a batch.
* :func:`orb_detect` / :func:`orb_lift` -- ORB keypoints of ``cv2.ORB_create()``'s defaults on the GPU and their
  lift onto the mesh (DESIGN.md §4.32), the stages behind :func:`ffb6d_b200.objinfo.textured_kp3ds`.
* :func:`sift_detect` / :func:`sift_lift` -- SIFT keypoints of ``cv2.SIFT_create()``'s defaults on the GPU and
  their lift (DESIGN.md §4.33), behind ``textured_kp3ds(..., extractor="SIFT")``.
* :mod:`ffb6d_b200.modules` -- ``nn.Module`` twins of the fusion ``Conv2d`` and of RandLA's
  ``Att_pooling`` / ``Building_block`` / ``Dilated_res_block`` (reference parameter names).

Everything runs through libffb6d_b200.so (hand-written CUDA behind a C ABI, see
include/ffb6d_b200.h); there is no CPU fallback: touching any op loads the library and raises if
it is missing.  Only the plain-data helpers (:mod:`ffb6d_b200.tables`, :mod:`ffb6d_b200.synthetic`)
are importable without it -- that is what lets the CPU reference arm of ``bench.py`` run without
mapping the product library.
"""
import importlib

_OPS = ("knn_search", "random_sample", "nearest_interpolation", "gather_neighbour", "relative_pos_encoding",
        "choose_gather", "grid_sub_sampling", "KnnGrid", "backproject", "fusion_mlp", "fusion_mlp_pack",
        "PackedWeight", "fold_batchnorm", "att_pool", "sample_valid_pixels", "check_indices", "mean_shift_fit", "best_fit_transform",
        "fill_missing", "segment_plan", "segment_sum", "point_item", "rgb_add_noise", "add_real_back",
        "aug_noise_field", "color_jitter", "psp_pool", "psp_pack", "psp_bottleneck", "conv1x1_log_softmax",
        "psp_bottleneck_bwd", "psp_pool_bwd", "log_softmax_bwd", "upsample_bilinear2d_bwd", "upsample_bilinear2d",
        "farthest_point_sampling", "pose_add_adds", "vote_poses", "point_input", "rgb_noise_check_records",
        "color_jitter_check_plans", "eval_record", "eval_auc", "depth_normal", "orb_detect", "orb_lift",
        "sift_detect", "sift_lift")
_SCHEDULE = ("build_ffb6d_indices", "build_ffb6d_indices_from_depth", "build_ffb6d_indices_native",
             "build_ffb6d_indices_from_raw_depth", "build_ffb6d_item", "build_ffb6d_inputs", "build_ffb6d_train_item")
_TABLES = ("knn_schedule", "gather_schedule", "fusion_mlp_schedule")
_ITEM = ("pose_gt_objects",)
_GRAPHED = ("GraphedTrainStep", "GraphedEvalStep", "GraphedFrameTrainStep")
_ESTIMATE = ("estimate_poses", "GraphedPoseStep")
_EVALUATE = ("GraphedTestStep",)
_RENDER = ("render_rgbd",)
_FUSE = ("fuse_rgbd",)
_SUBMODULES = ("ops", "schedule", "tables", "synthetic", "pipeline", "randla", "modules", "fusion", "dist",
               "helper_tool", "model", "pose", "item", "augment", "loss", "cnn", "graphed", "objinfo", "vis", "estimate", "evaluate", "render",
               "fuse_frames",
               "_lib")

__all__ = list(_OPS + _SCHEDULE + _TABLES + _ITEM + _GRAPHED + _ESTIMATE + _EVALUATE + _RENDER + _FUSE) + ["randla", "modules", "fusion", "pose", "loss", "cnn", "objinfo", "vis", "estimate", "evaluate", "render", "fuse_frames", "DataProcessing"]


def __getattr__(name):   # PEP 562: the CUDA library is loaded by the first op that is touched
    if name in _OPS:
        return getattr(importlib.import_module(".ops", __name__), name)
    if name in _SCHEDULE:
        return getattr(importlib.import_module(".schedule", __name__), name)
    if name in _TABLES:
        return getattr(importlib.import_module(".tables", __name__), name)
    if name in _ITEM:
        return getattr(importlib.import_module(".item", __name__), name)
    if name in _GRAPHED:
        return getattr(importlib.import_module(".graphed", __name__), name)
    if name in _ESTIMATE:
        return getattr(importlib.import_module(".estimate", __name__), name)
    if name in _EVALUATE:
        return getattr(importlib.import_module(".evaluate", __name__), name)
    if name in _RENDER:
        return getattr(importlib.import_module(".render", __name__), name)
    if name in _FUSE:
        return getattr(importlib.import_module(".fuse_frames", __name__), name)
    if name == "DataProcessing":
        return importlib.import_module(".helper_tool", __name__).DataProcessing
    if name in _SUBMODULES:
        return importlib.import_module("." + name, __name__)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))


def __dir__():
    return sorted(set(globals()) | set(__all__))
