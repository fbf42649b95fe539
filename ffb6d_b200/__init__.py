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
* :mod:`ffb6d_b200.pose` -- ``MeanShiftTorch``, ``best_fit_transform``, ``cal_frame_poses(_lm)``
  (utils/meanshift_pytorch.py:27-57, utils/pvn3d_eval_utils_kpls.py:28-160, 220-284): keypoint voting on the GPU.
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
        "aug_noise_field", "color_jitter")
_SCHEDULE = ("build_ffb6d_indices", "build_ffb6d_indices_from_depth", "build_ffb6d_indices_native",
             "build_ffb6d_indices_from_raw_depth", "build_ffb6d_item")
_TABLES = ("knn_schedule", "gather_schedule", "fusion_mlp_schedule")
_ITEM = ("pose_gt_objects",)
_SUBMODULES = ("ops", "schedule", "tables", "synthetic", "pipeline", "randla", "modules", "fusion", "dist",
               "helper_tool", "model", "pose", "item", "augment", "_lib")

__all__ = list(_OPS + _SCHEDULE + _TABLES + _ITEM) + ["randla", "modules", "fusion", "pose", "DataProcessing"]


def __getattr__(name):   # PEP 562: the CUDA library is loaded by the first op that is touched
    if name in _OPS:
        return getattr(importlib.import_module(".ops", __name__), name)
    if name in _SCHEDULE:
        return getattr(importlib.import_module(".schedule", __name__), name)
    if name in _TABLES:
        return getattr(importlib.import_module(".tables", __name__), name)
    if name in _ITEM:
        return getattr(importlib.import_module(".item", __name__), name)
    if name == "DataProcessing":
        return importlib.import_module(".helper_tool", __name__).DataProcessing
    if name in _SUBMODULES:
        return importlib.import_module("." + name, __name__)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))


def __dir__():
    return sorted(set(globals()) | set(__all__))
