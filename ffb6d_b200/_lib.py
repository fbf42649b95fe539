"""ctypes binding of libffb6d_b200.so (the C ABI declared in include/ffb6d_b200.h).

There is no CPU fallback: if the shared library is missing or fails to load,
importing this module raises, and every op in :mod:`ffb6d_b200.ops` fails with
it.  Build it with ``python -c "import __graft_entry__ as g; g.build()"`` or
``make -C ffb6d_b200/csrc``.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libffb6d_b200.so")

OK = 0
ERR_INVALID = -1
ERR_CUDA = -2
ERR_WORKSPACE = -3
ERR_NO_DEVICE = -4
LAYOUT_NCS = 0
LAYOUT_NSC = 1
MAX_K = 64
FPS_MAX_CLUSTER = 8                              # FFB6D_FPS_MAX_* of include/ffb6d_b200.h
FPS_MAX_POINTS = FPS_MAX_CLUSTER * 14336
FPS_MAX_SAMPLES = FPS_MAX_POINTS
FPS_MAX_CLOUDS = 65535
POSE_EVAL_GT_TILE = 512                          # FFB6D_POSE_EVAL_* of include/ffb6d_b200.h
POSE_EVAL_PRED_TILE = 512
POSE_EVAL_MAX_OBJECTS = 65535
POSE_EVAL_MAX_POINTS = 1 << 20
POSE_EVAL_MAX_MESHES = (1 << 31) - 2
EVAL_ROW_WORDS = 20                              # FFB6D_EVAL_* of include/ffb6d_b200.h
EVAL_MAX_ROWS = 1 << 24
VOTE_MAX_POINTS =(1 << 24) - 1                  # FFB6D_VOTE_* of include/ffb6d_b200.h
VOTE_MAX_CLASSES = 1024
VOTE_MAX_KPS = 64
VOTE_MAX_SETS = 1 << 24
VOTE_MAX_SLOTS = (1 << 31) - 1
VIS_MAX_RADIUS = 64                              # FFB6D_VIS_* of include/ffb6d_b200.h
VIS_MAX_SIDE = 16384
VIS_MAX_SETS = 1 << 24
VIS_MAX_ROWS = 1 << 24
VIS_MAX_TABLE_ROWS = (1 << 31) - 1
VIS_MAX_FRAMES = 65535
NRM_MAX_KSIZE = 16                               # FFB6D_NRM_* of include/ffb6d_b200.h
NRM_MAX_FRAMES = 65535
NRM_MAX_HEIGHT = 65535 * 8 - 1
NRM_MAX_FRAME_PIXELS = (1 << 31) - 1
RND_MAX_FRAMES = 65535                           # FFB6D_RND_* of include/ffb6d_b200.h
RND_MAX_FRAME_PIXELS = (1 << 31) - 1
RND_MAX_SLOTS = 4096
RND_MAX_MESH_VERTS = (1 << 31) - 1
RND_MAX_FRAME_FACES = 1 << 32
RND_GUARD_BAND = 1 << 14
RND_BIG_FACE_PIXELS = 256
RND_QUEUE_CAP = 1 << 20
RND_MAX_TEX_SIDE = 16384
RND_MAX_TEX_LEVELS = 15
RND_MAX_UV = 1 << 16
FUSE_MAX_FRAMES = 65535                          # FFB6D_FUSE_* of include/ffb6d_b200.h
FUSE_MAX_FRAME_PIXELS = (1 << 31) - 1
FUSE_MAX_SLOTS = 1024
FUSE_MAX_CROPS = (1 << 31) - 1
ORB_MAX_FRAMES = 65535                           # FFB6D_ORB_* of include/ffb6d_b200.h
ORB_MIN_SIDE = 2
ORB_MAX_SIDE = 8192
ORB_LEVELS = 8
ORB_MAX_OBJECTS = 65535
SIFT_MAX_FRAMES = 65535                          # FFB6D_SIFT_* of include/ffb6d_b200.h
SIFT_MIN_SIDE = 4
SIFT_MAX_SIDE = 2048
SIFT_MAX_CAP = 1 << 26
SIFT_CHUNK = 16
SIFT_MAX_COPIES = 18


class FFB6DError(RuntimeError):
    """A libffb6d_b200 entry point returned a negative status."""

    def __init__(self, code, msg):
        super().__init__("libffb6d_b200 error %d: %s" % (code, msg))
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "%s not found: the CUDA library has not been built (run __graft_entry__.build() "
            "or `make -C ffb6d_b200/csrc`). There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i64, sz, ci, fp = C.c_void_p, C.c_int64, C.c_size_t, C.c_int, C.c_float
    sig = {
        "ffb6d_version": (ci, []),
        "ffb6d_last_error": (C.c_char_p, []),
        "ffb6d_device_count": (ci, []),
        "ffb6d_launch_count": (C.c_uint64, []),
        "ffb6d_knn_workspace_bytes": (sz, [i64, i64, i64, ci]),
        "ffb6d_knn_batch": (ci, [vp, vp, i64, i64, i64, ci, vp, ci, vp, sz, vp]),
        "ffb6d_knn_batch_algo": (ci, [vp, vp, i64, i64, i64, ci, vp, ci, vp, sz, ci, vp]),
        "ffb6d_knn_grid_bytes": (sz, [i64, i64]),
        "ffb6d_knn_grid_query_bytes": (sz, [i64, i64]),
        "ffb6d_knn_grid_build": (ci, [vp, i64, i64, ci, vp, sz, vp]),
        "ffb6d_knn_grid_query": (ci, [vp, vp, i64, i64, i64, ci, vp, ci, vp, sz, vp, sz, vp]),
        "ffb6d_knn_grid_query_organized": (ci, [vp, vp, i64, i64, i64, ci, vp, ci, vp, sz, vp, sz, i64, vp]),
        "ffb6d_build_indices_workspace_bytes": (sz, [i64, i64, i64, i64, ci]),
        "ffb6d_build_indices": (ci, [vp, vp, vp, vp, i64, i64, i64, i64, ci, vp, ci, vp, sz, vp]),
        "ffb6d_knn_grid_tune": (None, [fp, ci]),
        "ffb6d_knn_grid_tune_k1": (None, [fp]),
        "ffb6d_knn_batch_host": (ci, [vp, sz, sz, sz, vp, sz, sz, vp]),
        "ffb6d_knn_host": (ci, [vp, sz, sz, vp, sz, sz, vp]),
        "ffb6d_gather_max_fwd": (ci, [vp, vp, ci, i64, i64, i64, i64, ci, ci, vp, vp]),
        "ffb6d_check_indices": (ci, [vp, ci, i64, i64, vp]),
        "ffb6d_check_indices_enabled": (ci, []),
        "ffb6d_gather_kernel_name": (C.c_char_p, [i64, i64, i64, i64, ci, ci]),
        "ffb6d_gather_max_bwd": (ci, [vp, vp, ci, vp, i64, i64, i64, i64, ci, ci, vp, vp]),
        "ffb6d_gather_neighbour_fwd": (ci, [vp, vp, ci, i64, i64, i64, i64, ci, vp, vp]),
        "ffb6d_gather_neighbour_bwd": (ci, [vp, vp, ci, i64, i64, i64, i64, ci, vp, vp]),
        "ffb6d_relative_pos_encoding_fwd": (ci, [vp, vp, ci, i64, i64, ci, vp, vp]),
        "ffb6d_fusion_mlp_pack_bytes": (sz, [i64, i64]),
        "ffb6d_fusion_mlp_pack": (ci, [vp, i64, i64, vp, sz, vp]),
        "ffb6d_fusion_mlp_fwd_packed": (ci, [vp, i64, vp, i64, vp, vp, vp, i64, i64, i64, ci, fp, vp, vp]),
        "ffb6d_fusion_mlp_fwd_ex": (ci, [vp, i64, vp, i64, vp, vp, vp, i64, i64, i64, ci, fp, vp, vp, ci, i64, ci, vp, vp]),
        "ffb6d_bn_workspace_bytes": (sz, [i64, i64]),
        "ffb6d_bn_train_fwd": (ci, [vp, i64, i64, i64, vp, vp, fp, fp, vp, vp, ci, fp, vp, vp, vp, sz, vp]),
        "ffb6d_bn_train_bwd": (ci, [vp, vp, vp, i64, i64, i64, ci, fp, vp, vp, vp, vp, sz, vp]),
        "ffb6d_bn_sync_moments": (ci, [vp, i64, i64, i64, vp, vp, sz, vp]),
        "ffb6d_bn_sync_fwd": (ci, [vp, i64, i64, i64, vp, i64, vp, vp, fp, fp, vp, vp, ci, fp, vp, vp, vp, vp]),
        "ffb6d_bn_sync_bwd_sums": (ci, [vp, vp, vp, i64, i64, i64, ci, fp, vp, vp, vp, vp, sz, vp]),
        "ffb6d_bn_sync_bwd": (ci, [vp, vp, vp, i64, i64, i64, vp, i64, vp, ci, fp, vp, vp, sz, vp]),
        "ffb6d_act_bwd": (ci, [vp, vp, i64, ci, fp, vp, vp]),
        "ffb6d_fusion_mlp_wgrad": (ci, [vp, vp, i64, vp, i64, i64, i64, i64, vp, vp]),
        "ffb6d_segment_plan_bytes": (sz, [i64, i64, i64]),
        "ffb6d_segment_plan": (ci, [vp, ci, i64, i64, i64, vp, sz, vp]),
        "ffb6d_segment_sum": (ci, [vp, vp, sz, i64, i64, i64, i64, vp, vp]),
        "ffb6d_segment_csr_bytes": (sz, [i64, i64, i64]),
        "ffb6d_segment_csr": (ci, [vp, ci, i64, i64, i64, vp, sz, vp]),
        "ffb6d_segment_sum_csr": (ci, [vp, vp, sz, i64, i64, i64, i64, vp, vp]),
        "ffb6d_gather_max_bwd_det_workspace_bytes": (sz, [i64, i64, i64, i64, ci]),
        "ffb6d_gather_max_bwd_det": (ci, [vp, vp, ci, vp, i64, i64, i64, i64, ci, ci, vp, sz, vp, vp]),
        "ffb6d_gather_neighbour_bwd_det_workspace_bytes": (sz, [i64, i64, i64, ci]),
        "ffb6d_gather_neighbour_bwd_det": (ci, [vp, vp, ci, i64, i64, i64, i64, ci, vp, sz, vp, vp]),
        "ffb6d_fusion_mlp_wgrad_det_workspace_bytes": (sz, [i64, i64, i64, i64, i64]),
        "ffb6d_fusion_mlp_wgrad_det": (ci, [vp, vp, i64, vp, i64, i64, i64, i64, vp, sz, vp, vp]),
        "ffb6d_att_pool_bwd": (ci, [vp, i64, vp, i64, vp, vp, i64, i64, ci, vp, vp, vp, vp]),
        "ffb6d_lfa_att_pool_fused": (ci, [vp, vp, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, ci, i64, i64, fp, vp, vp]),
        "ffb6d_att_pool_fwd": (ci, [vp, i64, vp, i64, vp, i64, i64, ci, vp, vp]),
        "ffb6d_lfa_train_fwd": (ci, [vp, vp, ci, vp, vp, i64, i64, ci, i64, vp, vp]),
        "ffb6d_lfa_train_bwd_workspace_bytes": (sz, [i64, i64, ci, i64]),
        "ffb6d_lfa_train_bwd": (ci, [vp, vp, ci, vp, vp, vp, i64, i64, ci, i64, vp, vp, vp, vp, sz, vp]),
        "ffb6d_relative_pos_encoding_cm_fwd": (ci, [vp, vp, ci, i64, i64, ci, vp, vp]),
        "ffb6d_backproject": (ci, [vp, i64, i64, i64, vp, ci, vp, i64, vp, vp, vp, vp, vp]),
        "ffb6d_point_item": (ci, [vp, i64, i64, i64, vp, ci, vp, i64, vp, vp, vp, vp, vp, vp, i64, i64, vp, vp, vp, vp,
                                  vp]),
        "ffb6d_point_input": (ci, [vp, i64, i64, i64, vp, ci, vp, i64, vp, vp, vp, vp]),
        "ffb6d_sample_pixels_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_sample_pixels": (ci, [vp, i64, i64, i64, fp, i64, C.c_uint64, vp, vp, vp, sz, vp]),
        "ffb6d_sample_pixels_dseed": (ci, [vp, i64, i64, i64, fp, i64, vp, vp, vp, vp, sz, vp]),
        "ffb6d_fill_depth_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_fill_depth": (ci, [vp, i64, i64, i64, fp, vp, vp, vp, sz, vp]),
        "ffb6d_depth_normal": (ci, [vp, i64, i64, i64, vp, ci, ci, ci, ci, ci, vp, vp]),
        "ffb6d_depth_to_mm": (ci, [vp, i64, fp, vp, vp]),
        "ffb6d_render_workspace_bytes": (sz, [i64, i64, i64, i64, i64, i64]),
        "ffb6d_render_rgbd": (ci, [vp, vp, vp, vp, vp, i64, i64, i64, vp, vp, vp, i64, i64, vp, ci, i64, i64,
                                   C.c_double, vp, vp, vp, vp, vp, vp, sz, vp]),
        "ffb6d_render_texture_mips": (ci, [vp, vp, vp, i64, i64, vp]),
        "ffb6d_render_rgbd_textured": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, i64, i64,
                                            vp, ci, i64, i64, C.c_double, vp, vp, vp, vp, vp, vp, sz, vp]),
        "ffb6d_fuse_rgbd": (ci, [vp, vp, vp, vp, vp, i64, vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, vp, vp]),
        "ffb6d_orb_capacity": (i64, [i64, i64]),
        "ffb6d_orb_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_orb_detect": (ci, [vp, i64, i64, i64, vp, vp, vp, vp, i64, vp, sz, vp]),
        "ffb6d_orb_lift": (ci, [vp, vp, i64, vp, i64, i64, i64, vp, ci, vp, i64, vp, vp, vp]),
        "ffb6d_sift_capacity": (i64, [i64, i64]),
        "ffb6d_sift_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_sift_detect": (ci, [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, i64, vp, sz, vp]),
        "ffb6d_sift_lift": (ci, [vp, vp, i64, vp, i64, i64, i64, vp, ci, vp, i64, vp, vp, vp]),
        "ffb6d_mean_shift_workspace_bytes": (sz, [i64, i64]),
        "ffb6d_mean_shift_fit": (ci, [vp, vp, i64, i64, i64, fp, ci, vp, vp, vp, vp, vp, sz, vp]),
        "ffb6d_best_fit_transform": (ci, [vp, vp, i64, i64, vp, vp]),
        "ffb6d_vote_poses_workspace_bytes": (sz, [i64, i64, i64, i64]),
        "ffb6d_vote_poses": (ci, [vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, ci, ci, fp, ci, vp, vp, vp, vp, vp,
                                  sz, vp]),
        "ffb6d_rgb_add_noise": (ci, [vp, i64, i64, i64, vp, vp, C.c_uint64, vp, vp, vp, vp]),
        "ffb6d_rgb_add_noise_dseed": (ci, [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, vp]),
        "ffb6d_rgb_noise_check_records": (ci, [vp, i64]),
        "ffb6d_add_real_back": (ci, [vp, vp, vp, vp, vp, ci, vp, vp, ci, i64, i64, i64, vp, vp, vp]),
        "ffb6d_aug_noise_field": (ci, [C.c_uint64, i64, i64, i64, ci, vp, vp]),
        "ffb6d_color_jitter": (ci, [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp]),
        "ffb6d_color_jitter_check_plans": (ci, [vp, i64]),
        "ffb6d_loss_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_focal_loss_fwd": (ci, [vp, ci, vp, ci, vp, i64, i64, i64, fp, vp, ci, vp, vp, vp, vp, vp, sz, vp]),
        "ffb6d_focal_loss_bwd": (ci, [vp, ci, vp, ci, vp, i64, i64, i64, fp, vp, ci, vp, vp, vp, vp, vp]),
        "ffb6d_of_l1_loss_fwd": (ci, [vp, vp, vp, ci, vp, i64, i64, i64, vp, vp, vp, sz, vp]),
        "ffb6d_of_l1_loss_bwd": (ci, [vp, vp, vp, ci, vp, i64, i64, i64, vp, vp, vp, vp]),
        "ffb6d_psp_pool": (ci, [vp, i64, i64, i64, i64, vp, vp]),
        "ffb6d_psp_bottleneck_fwd": (ci, [vp, i64, i64, i64, i64, vp, vp, i64, vp, vp, vp]),
        "ffb6d_conv1x1_log_softmax_fwd": (ci, [vp, i64, i64, i64, vp, vp, i64, vp, vp]),
        "ffb6d_psp_bottleneck_bwd": (ci, [vp, vp, i64, i64, i64, i64, vp, vp, vp, vp]),
        "ffb6d_psp_pool_bwd": (ci, [vp, i64, i64, i64, i64, vp, vp]),
        "ffb6d_log_softmax_bwd": (ci, [vp, vp, i64, i64, i64, vp, vp]),
        "ffb6d_upsample_bilinear2d_bwd": (ci, [vp, i64, i64, i64, i64, i64, i64, vp, vp]),
        "ffb6d_upconv_taps_fwd": (ci, [vp, i64, i64, i64, i64, i64, i64, vp, vp, vp, vp, vp, vp]),
        "ffb6d_upconv_taps_bwd": (ci, [vp, i64, i64, i64, i64, i64, i64, vp, vp]),
        "ffb6d_prelu_fwd": (ci, [vp, i64, vp, vp, vp]),
        "ffb6d_bn_prelu_bwd": (ci, [vp, vp, vp, i64, i64, i64, vp, vp, vp, vp]),
        "ffb6d_farthest_point_sampling_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_farthest_point_sampling": (ci, [vp, vp, i64, i64, i64, vp, ci, vp, vp, sz, vp]),
        "ffb6d_pose_add_adds_workspace_bytes": (sz, [i64, i64]),
        "ffb6d_pose_add_adds": (ci, [vp, vp, i64, i64, vp, vp, vp, i64, vp, vp, vp, sz, vp]),
        "ffb6d_eval_record": (ci, [vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, vp, i64, vp, vp,
                                   vp, i64, vp]),
        "ffb6d_eval_auc_workspace_bytes": (sz, [i64, i64]),
        "ffb6d_eval_auc": (ci, [vp, vp, i64, i64, vp, C.c_double, vp, vp, vp, vp, sz, vp]),
        "ffb6d_project_p3d":(ci, [vp, ci, i64, vp, vp, vp, i64, i64, vp, vp, vp, ci, vp, vp]),
        "ffb6d_draw_p2ds_workspace_bytes": (sz, [i64, i64, i64]),
        "ffb6d_draw_p2ds": (ci, [vp, i64, i64, i64, vp, i64, i64, vp, vp, vp, vp, i64, vp, vp, ci, vp, sz, vp]),
        "ffb6d_grid_subsample_host": (ci, [vp, sz, vp, sz, vp, sz, fp, vp, vp, vp, C.POINTER(sz)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib, sorted(sig)


lib, SYMBOLS = _load()


def last_error():
    return lib.ffb6d_last_error().decode("utf-8", "replace")


def check(rc):
    if rc != OK:
        raise FFB6DError(rc, last_error())


def stream(device):
    """The current torch stream of ``device`` as the ``ffb6d_stream_t`` argument of an entry point."""
    return torch.cuda.current_stream(device).cuda_stream


def launch(fn, device, *args):
    """``fn(*args, stream(device))`` with ``device`` current: how every device entry point of the library is called
    (each takes its stream last).  Raises :class:`FFB6DError` on a failed status.  The stream is fetched inline, not
    through :func:`stream`: this runs once per launch, and an eager training step is host-bound."""
    with torch.cuda.device(device):
        check(fn(*args, torch.cuda.current_stream(device).cuda_stream))


def ptr(t):
    """The device pointer of ``t`` for an optional argument: None (NULL) for None."""
    return None if t is None else t.data_ptr()


def workspace(nbytes, device):
    """Scratch for an entry point whose ``*_bytes`` query answered ``nbytes``: at least 16 bytes, so never NULL even
    where the answer is 0, and enough for every entry point's minimum.  Pass the entry point ``nbytes`` itself."""
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def launch_count():
    return int(lib.ffb6d_launch_count())
