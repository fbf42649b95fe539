"""Host-side mirror of the reference's op surface for the fusion hot path.

Same function names, argument meaning and result shapes/dtypes as the reference
(ethnhe/FFB6D); every call goes through the C ABI of libffb6d_b200.so
(include/ffb6d_b200.h).  torch is used for device memory and streams only.
No op has a CPU implementation: numpy inputs are copied to the GPU by the
``*_host`` entry points, torch inputs must already be CUDA tensors.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, launch, ptr, workspace, LAYOUT_NCS, LAYOUT_NSC
from ._lib import stream as _stream   # noqa: F401  (the stream argument for direct lib.* calls: tests and tools)

import os as _os
_DEBUG_GRID = bool(_os.environ.get("FFB6D_DEBUG_GRID"))   # keep KNN workspaces for tools/grid_debug.py
_debug_ws = []
_I64 = (torch.int64,)
_IDX = (torch.int32, torch.int64)


def _need_cuda(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor, got %r" % (name, type(t)))
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: ffb6d_b200 has no CPU path" % name)


def _tensor(t, name, dtype=torch.float32, shape=None, device=None):
    """``t`` as a kernel reads it: a CUDA tensor of ``dtype``, of ``shape`` (a tuple) or of that many dimensions (an
    int) when given, on ``device`` when given; returned contiguous.  Raises ValueError otherwise (TypeError /
    RuntimeError for a non-tensor / a CPU tensor)."""
    _need_cuda(t, name)
    if isinstance(shape, int):
        bad_shape, want = t.dim() != shape, "with %d dims" % shape
    else:
        bad_shape, want = shape is not None and tuple(t.shape) != tuple(shape), tuple(shape or ())
    if t.dtype != dtype or bad_shape:
        raise ValueError("%s must be %s %s, got %s %s" % (name, dtype, want, t.dtype, tuple(t.shape)))
    if device is not None and t.device != device:
        raise ValueError("%s is on %s, expected %s" % (name, t.device, device))
    return t.contiguous()


def deterministic_backward(weight_grad=False):
    """Whether a backward should take its deterministic path, decided when the backward runs (as torch decides for
    its own ops).  ``torch.use_deterministic_algorithms(True)`` turns it on for every backward of this package that
    otherwise adds with atomics (gathers, neighbour gathers, layer weight gradients).  With ``weight_grad=True`` --
    the 1x1 layers, which stand in for cuDNN convolutions -- ``torch.backends.cudnn.deterministic`` does too: it is
    the flag the reference's ``--deterministic`` sets.  Like ``torch.gather``'s backward, the gathers do not follow
    ``cudnn.deterministic`` alone.  The deterministic paths write every output once, in a fixed order, and are
    bit-identical from run to run; the default paths are unchanged."""
    if torch.are_deterministic_algorithms_enabled():
        return True
    return bool(weight_grad) and bool(torch.backends.cudnn.deterministic)


def _idx_arg(idx, name):
    if idx.dtype not in _IDX:
        raise TypeError("%s must be int32 or int64, got %s" % (name, idx.dtype))
    return idx.contiguous(), int(idx.dtype == torch.int64)


# --------------------------------------------------------------------------- KNN
def knn_search(support_pts, query_pts, k, out_dtype=None, algo=0):
    """Exact KNN index build; mirrors ``DataProcessing.knn_search``
    (models/RandLA/helper_tool.py:160-170).

    :param support_pts: points you have, B*N1*3 (float32)
    :param query_pts: points you want the neighbour indices of, B*N2*3
    :param k: number of neighbours
    :return: neighbour indices B*N2*k, ascending distance.

    numpy in -> numpy int32 out, exactly as the reference (which casts the int64
    result of ``nearest_neighbors.knn_batch`` with ``.astype(np.int32)``); the call
    goes through ``ffb6d_knn_batch_host`` whose signature is that of the
    reference's ``cpp_knn_batch_omp`` (NN/knn_.h:14-16).
    CUDA tensors in -> CUDA tensor out (int32 unless ``out_dtype`` says int64), no
    host round trip.

    Deviations from the reference an integrator should know (DESIGN.md "tie contract"):
    * rows whose K+1 nearest contain EXACT fp32 distance ties (duplicated points, e.g. the datasets'
      ``np.pad(..., 'wrap')``, ycb_dataset.py:230) are ordered by ascending (distance, index); the
      reference's order there is its KD-tree's traversal order.  Distances per row are identical.
    * ``k`` must be in [1, 64] and points 3-D (the reference accepts any k and dim).
    """
    k = int(k)
    if isinstance(support_pts, np.ndarray) or isinstance(query_pts, np.ndarray):
        sup = np.ascontiguousarray(support_pts, dtype=np.float32)  # NN/knn.pyx:95-96
        qry = np.ascontiguousarray(query_pts, dtype=np.float32)
        if sup.ndim != 3 or qry.ndim != 3 or sup.shape[0] != qry.shape[0]:
            raise ValueError("knn_search expects [B,N1,3] and [B,N2,3], got %s and %s"
                             % (sup.shape, qry.shape))
        B, S, dim = sup.shape
        Q = qry.shape[1]
        indices = np.zeros((B, Q, k), dtype=np.int64)               # NN/knn.pyx:93
        check(lib.ffb6d_knn_batch_host(sup.ctypes.data, B, S, dim, qry.ctypes.data, Q, k,
                                       indices.ctypes.data))
        return indices.astype(np.int32)                             # helper_tool.py:170
    _need_cuda(support_pts, "support_pts")
    _need_cuda(query_pts, "query_pts")
    sup = support_pts.contiguous().float()
    qry = query_pts.contiguous().float()
    if sup.dim() != 3 or qry.dim() != 3 or sup.shape[0] != qry.shape[0] or sup.shape[2] != 3 \
            or qry.shape[2] != 3:
        raise ValueError("knn_search expects [B,N1,3] and [B,N2,3], got %s and %s"
                         % (tuple(sup.shape), tuple(qry.shape)))
    B, S, _ = sup.shape
    Q = qry.shape[1]
    dt = torch.int32 if out_dtype is None else out_dtype
    if dt not in _IDX:
        raise TypeError("out_dtype must be torch.int32 or torch.int64")
    out = torch.empty((B, Q, k), dtype=dt, device=sup.device)
    ws_bytes = int(lib.ffb6d_knn_workspace_bytes(B, S, Q, k)) if algo != 1 else 0
    ws = workspace(ws_bytes, sup.device)
    launch(lib.ffb6d_knn_batch_algo, sup.device, sup.data_ptr(), qry.data_ptr(), B, S, Q, k, out.data_ptr(),
           int(dt == torch.int64), ws.data_ptr(), ws_bytes, int(algo))
    if _DEBUG_GRID:
        _debug_ws.append((B, S, Q, k, ws if ws_bytes else None))
    return out


class KnnGrid:
    """Uniform-grid index of a support batch: build once, search many times
    (``ffb6d_knn_grid_build`` / ``ffb6d_knn_grid_query``).  The FFB6D schedule searches every
    pyramid level two to four times (datasets/ycb/ycb_dataset.py:275-308); sharing the grid
    removes the repeated builds.  Results are identical to :func:`knn_search`.

    :param support: ``[B, S, 3]`` float32 CUDA tensor
    :param k_hint: the neighbour count the grid will mostly be searched with (tunes the cell
      size only; any ``k`` may be queried)
    """

    def __init__(self, support, k_hint):
        _need_cuda(support, "support")
        sup = support.contiguous().float()
        if sup.dim() != 3 or sup.shape[2] != 3 or sup.shape[1] < 1:
            raise ValueError("KnnGrid expects a non-empty [B,S,3] support, got %s" % (tuple(sup.shape),))
        self.support = sup
        self.B, self.S = sup.shape[0], sup.shape[1]
        self.k_hint = int(k_hint)
        self.nbytes = int(lib.ffb6d_knn_grid_bytes(self.B, self.S))
        self.mem = torch.empty(self.nbytes, dtype=torch.uint8, device=sup.device)
        launch(lib.ffb6d_knn_grid_build, sup.device, sup.data_ptr(), self.B, self.S, self.k_hint, self.mem.data_ptr(),
               self.nbytes)

    def query(self, query_pts, k, out_dtype=None, query_width=0):
        """``query_pts [B,Q,3]`` -> ``[B,Q,k]`` neighbour indices into the support (int32 unless
        ``out_dtype`` is torch.int64).  Pass the support tensor itself for a self search.
        ``query_width``: the queries are the pixels of an image with rows of that many points (a
        performance hint for K = 1, results do not depend on it); 0 = no particular order."""
        _need_cuda(query_pts, "query_pts")
        qry = self.support if query_pts is self.support else query_pts.contiguous().float()
        if qry.dim() != 3 or qry.shape[0] != self.B or qry.shape[2] != 3:
            raise ValueError("query must be [B,Q,3] with B=%d, got %s" % (self.B, tuple(qry.shape)))
        k = int(k)
        Q = qry.shape[1]
        dt = torch.int32 if out_dtype is None else out_dtype
        if dt not in _IDX:
            raise TypeError("out_dtype must be torch.int32 or torch.int64")
        dev = self.support.device
        out = torch.empty((self.B, Q, k), dtype=dt, device=dev)
        sb = int(lib.ffb6d_knn_grid_query_bytes(self.B, Q))
        scratch = workspace(sb, dev)
        qw = int(query_width) if query_width and Q % int(query_width) == 0 else 0
        launch(lib.ffb6d_knn_grid_query_organized, dev, self.support.data_ptr(), qry.data_ptr(), self.B, self.S, Q, k,
               out.data_ptr(), int(dt == torch.int64), self.mem.data_ptr(), self.nbytes, scratch.data_ptr(), sb, qw)
        return out


def knn_uses_grid(B, S, Q, k):
    """True when :func:`knn_search` would answer this problem with the grid search (rather than
    the tiled scan it uses for small problems)."""
    return int(lib.ffb6d_knn_workspace_bytes(B, S, Q, int(k))) > 0


# --------------------------------------------------------------------------- gather + max
def _layout_of(f3):
    """f3: [B,C,S] view.  Returns (tensor, layout) with tensor dense in that layout."""
    B, Cc, S = f3.shape
    sb, sc, ss = f3.stride()
    if f3.is_contiguous():
        return f3, LAYOUT_NCS
    if S > 1 and Cc > 1 and sc == 1 and ss == Cc and (B == 1 or sb == Cc * S):
        return f3, LAYOUT_NSC          # channels_last view of an NCHW tensor
    return f3.contiguous(), LAYOUT_NCS


class _GatherMax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f3, idx):
        f3, layout = _layout_of(f3)
        idx_c, i64 = _idx_arg(idx, "index")
        B, Cc, S = f3.shape
        Q, K = idx_c.shape[1], idx_c.shape[2]
        if layout == LAYOUT_NCS:
            out = torch.empty((B, Cc, Q), dtype=torch.float32, device=f3.device)
        else:
            out = torch.empty((B, Q, Cc), dtype=torch.float32, device=f3.device).transpose(1, 2)
        launch(lib.ffb6d_gather_max_fwd, f3.device, f3.data_ptr(), idx_c.data_ptr(), i64, B, Cc, S, Q, K, layout,
               out.data_ptr())
        ctx.save_for_backward(f3, idx_c)
        ctx.layout = layout
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        f3, idx_c = ctx.saved_tensors
        return _gather_max_bwd(f3, idx_c, gout, ctx.layout), None


def _gather_max_bwd(f3, idx_c, gout, layout):
    """The gradient of :class:`_GatherMax` w.r.t. ``f3`` (in f3's layout): ``ffb6d_gather_max_bwd`` (fp32 atomics), or
    under :func:`deterministic_backward` a segment sum over the CSR of the index (``ffb6d_gather_max_bwd_det``)."""
    B, Cc, S = f3.shape
    Q, K = idx_c.shape[1], idx_c.shape[2]
    if layout == LAYOUT_NCS:
        g = gout.contiguous()
        gf = torch.empty((B, Cc, S), dtype=torch.float32, device=f3.device)
    else:
        g = gout.transpose(1, 2).contiguous().transpose(1, 2)   # dense [B,Q,C] storage
        gf = torch.empty((B, S, Cc), dtype=torch.float32, device=f3.device).transpose(1, 2)
    if deterministic_backward():
        if K == 1 and layout == LAYOUT_NCS and _counter_plan_fits(Q, S):
            return segment_sum(g, None, S, plan=SegmentPlan(idx_c.reshape(B, Q), S))
        _gather_max_bwd_det(f3, idx_c, g, layout, gf)
        return gf
    launch(lib.ffb6d_gather_max_bwd, f3.device, f3.data_ptr(), idx_c.data_ptr(), int(idx_c.dtype == torch.int64),
           g.data_ptr(), B, Cc, S, Q, K, layout, gf.data_ptr())
    return gf


def _counter_plan_fits(P, NA):
    """True when the (segment, 1024-entry tile) counters of :class:`SegmentPlan` take no more room than the
    linear :class:`SegmentCSR`: few segments, as in the p2r maps.  Both give the same CSR, so this choice changes
    speed only, never a result."""
    return NA * -(-P // 1024) <= P + NA


def _gather_max_bwd_det(f3, idx_c, g, layout, gf):
    """``ffb6d_gather_max_bwd_det`` into ``gf`` (the backward of :class:`_GatherMax` without atomics)."""
    B, Cc, S = f3.shape
    Q, K = idx_c.shape[1], idx_c.shape[2]
    nbytes = int(lib.ffb6d_gather_max_bwd_det_workspace_bytes(B, Cc, S, Q, K))
    ws = workspace(nbytes, f3.device)
    launch(lib.ffb6d_gather_max_bwd_det, f3.device, f3.data_ptr(), idx_c.data_ptr(), int(idx_c.dtype == torch.int64),
           g.data_ptr(), B, Cc, S, Q, K, layout, ws.data_ptr(), nbytes, gf.data_ptr())


def _gather_max(feature, idx3):
    """feature [B,C,S] or [B,C,S,1] f32 CUDA; idx3 [B,Q,K] -> [B,C,Q] (layout follows input)."""
    _need_cuda(feature, "feature")
    _need_cuda(idx3, "index")
    if feature.dtype != torch.float32:
        raise TypeError("feature must be float32 (the reference runs amp O0), got %s" % feature.dtype)
    if feature.dim() == 4:
        if feature.shape[3] != 1:
            raise ValueError("feature must be [B,C,N,1], got %s" % (tuple(feature.shape),))
        f3 = feature.squeeze(3)
    elif feature.dim() == 3:
        f3 = feature
    else:
        raise ValueError("feature must be [B,C,N] or [B,C,N,1], got %s" % (tuple(feature.shape),))
    if idx3.dim() != 3 or idx3.shape[0] != f3.shape[0]:
        raise ValueError("index must be [B,N',K] with the batch of feature, got %s"
                         % (tuple(idx3.shape),))
    if idx3.shape[2] < 1 or idx3.shape[2] > _lib.MAX_K:
        raise ValueError("neighbour count %d outside [1,%d]" % (idx3.shape[2], _lib.MAX_K))
    return _GatherMax.apply(f3, idx3)


def random_sample(feature, pool_idx):
    """Gather the K neighbours' features and max-pool over K; mirrors
    ``FFB6D.random_sample`` (models/ffb6d.py:159-177) and ``Network.random_sample``
    (models/RandLA/RandLANet.py:87-102).

    :param feature: [B, d, N, 1] (or [B, d, N]) input features
    :param pool_idx: [B, N', max_num] neighbour indices, N' the positions kept after pooling
    :return: pool_features = [B, d, N', 1]
    """
    return _gather_max(feature, pool_idx).unsqueeze(3)


def nearest_interpolation(feature, interp_idx):
    """Nearest-neighbour feature interpolation (K = 1 gather); mirrors
    ``FFB6D.nearest_interpolation`` (models/ffb6d.py:179-194) and the RandLA twin
    (models/RandLA/RandLANet.py:104-117).

    :param feature: [B, d, N, 1] input features
    :param interp_idx: [B, up_num_points, 1] nearest neighbour index
    :return: [B, d, up_num_points, 1] interpolated features
    """
    if feature.dim() != 4:
        raise ValueError("feature must be [B,C,N,1], got %s" % (tuple(feature.shape),))
    B, up = interp_idx.shape[0], interp_idx.shape[1]
    return _gather_max(feature, interp_idx.reshape(B, up, 1)).unsqueeze(3)


def choose_gather(rgb_emb, choose):
    """The final ``choose`` gather of ``FFB6D.forward`` (models/ffb6d.py:309-312):
    ``rgb_emb [B,C,H,W]`` (or [B,C,HW]), ``choose [B,1,N]`` -> ``[B,C,N]``."""
    B, Cc = rgb_emb.shape[0], rgb_emb.shape[1]
    f3 = rgb_emb.reshape(B, Cc, -1) if rgb_emb.dim() == 4 and rgb_emb.is_contiguous() else \
        rgb_emb.flatten(2)
    return _gather_max(f3, choose.reshape(B, -1, 1))


def check_indices(idx, S):
    """Raise :class:`ffb6d_b200._lib.FFB6DError` if any element of the CUDA index tensor ``idx`` lies
    outside ``[0, S)`` (``ffb6d_check_indices``; blocking).  The gather kernels trust their indices where
    ``torch.gather`` raises a device assert; set ``FFB6D_CHECK_INDICES=1`` to run this check in front of
    every gather (debugging aid, synchronises)."""
    _need_cuda(idx, "idx")
    idx_c, i64 = _idx_arg(idx, "idx")
    launch(lib.ffb6d_check_indices, idx_c.device, idx_c.data_ptr(), i64, idx_c.numel(), int(S))


# --------------------------------------------------------------------------- neighbour gather
class _GatherNeighbour(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pc, idx):
        pc = pc.contiguous()
        idx_c, i64 = _idx_arg(idx, "neighbor_idx")
        B, S, D = pc.shape
        N, K = idx_c.shape[1], idx_c.shape[2]
        out = torch.empty((B, N, K, D), dtype=torch.float32, device=pc.device)
        launch(lib.ffb6d_gather_neighbour_fwd, pc.device, pc.data_ptr(), idx_c.data_ptr(), i64, B, S, D, N, K,
               out.data_ptr())
        ctx.save_for_backward(idx_c)
        ctx.shape = (B, S, D)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        (idx_c,) = ctx.saved_tensors
        B, S, D = ctx.shape
        N, K = idx_c.shape[1], idx_c.shape[2]
        g = gout.contiguous()
        gpc = torch.empty((B, S, D), dtype=torch.float32, device=g.device)
        i64 = int(idx_c.dtype == torch.int64)
        if deterministic_backward():
            nbytes = int(lib.ffb6d_gather_neighbour_bwd_det_workspace_bytes(B, S, N, K))
            ws = workspace(nbytes, g.device)
            launch(lib.ffb6d_gather_neighbour_bwd_det, g.device, g.data_ptr(), idx_c.data_ptr(), i64, B, S, D, N, K,
                   ws.data_ptr(), nbytes, gpc.data_ptr())
            return gpc, None
        launch(lib.ffb6d_gather_neighbour_bwd, g.device, g.data_ptr(), idx_c.data_ptr(), i64, B, S, D, N, K,
               gpc.data_ptr())
        return gpc, None


def gather_neighbour(pc, neighbor_idx):
    """Gather the coordinates or features of neighbouring points; mirrors
    ``Building_block.gather_neighbour`` (models/RandLA/RandLANet.py:225-234).

    :param pc: [B, npoint, channel]
    :param neighbor_idx: [B, npoint, nsamples]
    :return: [B, npoint, nsamples, channel]
    """
    _need_cuda(pc, "pc")
    _need_cuda(neighbor_idx, "neighbor_idx")
    if pc.dtype != torch.float32:
        raise TypeError("pc must be float32, got %s" % pc.dtype)
    if pc.dim() != 3 or neighbor_idx.dim() != 3 or pc.shape[0] != neighbor_idx.shape[0]:
        raise ValueError("gather_neighbour expects pc [B,N,d] and idx [B,N,K], got %s, %s"
                         % (tuple(pc.shape), tuple(neighbor_idx.shape)))
    return _GatherNeighbour.apply(pc, neighbor_idx)


def relative_pos_encoding(xyz, neigh_idx, channel_major=False):
    """10-channel relative position encoding; mirrors
    ``Building_block.relative_pos_encoding`` (models/RandLA/RandLANet.py:216-223).
    Forward only (its inputs are coordinates and indices, neither requires grad in FFB6D).

    :param xyz: [B, N, 3]; :param neigh_idx: [B, N, K]; :return: [B, N, K, 10]
      (``channel_major=True``: [B, 10, N, K])
    """
    _need_cuda(xyz, "xyz")
    _need_cuda(neigh_idx, "neigh_idx")
    xyz = xyz.contiguous().float()
    idx_c, i64 = _idx_arg(neigh_idx, "neigh_idx")
    if xyz.dim() != 3 or xyz.shape[2] != 3 or idx_c.dim() != 3 or idx_c.shape[:2] != xyz.shape[:2]:
        raise ValueError("relative_pos_encoding expects xyz [B,N,3] and idx [B,N,K]")
    B, N, _ = xyz.shape
    K = idx_c.shape[2]
    if channel_major:    # [B,10,N,K]: what .permute((0,3,1,2)).contiguous() gives (RandLANet.py:197-198)
        out = torch.empty((B, 10, N, K), dtype=torch.float32, device=xyz.device)
        fn = lib.ffb6d_relative_pos_encoding_cm_fwd
    else:
        out = torch.empty((B, N, K, 10), dtype=torch.float32, device=xyz.device)
        fn = lib.ffb6d_relative_pos_encoding_fwd
    launch(fn, xyz.device, xyz.data_ptr(), idx_c.data_ptr(), i64, B, N, K, out.data_ptr())
    return out


# --------------------------------------------------------------------------- fusion 1x1 MLP
def fold_batchnorm(bn):
    """Eval-mode BatchNorm as a per-channel affine: ``scale = gamma / sqrt(var + eps)``,
    ``shift = beta - mean * scale`` (float32 tensors on the module's device)."""
    var, mean = bn.running_var.float(), bn.running_mean.float()
    gamma = bn.weight.float() if bn.weight is not None else torch.ones_like(var)
    beta = bn.bias.float() if bn.bias is not None else torch.zeros_like(var)
    scale = gamma / torch.sqrt(var + bn.eps)
    return scale.contiguous(), (beta - mean * scale).contiguous()


class PackedWeight:
    """``conv.weight`` of a 1x1 layer split into TF32 hi/lo tiles for :func:`fusion_mlp`
    (``ffb6d_fusion_mlp_pack``).  Build it once per layer at load time (inference)."""

    def __init__(self, weight):
        _need_cuda(weight, "weight")
        w = weight.detach().reshape(weight.shape[0], -1).contiguous().float()
        self.Co, self.Ci = int(w.shape[0]), int(w.shape[1])
        self.device = w.device
        nbytes = lib.ffb6d_fusion_mlp_pack_bytes(self.Co, self.Ci)
        self.data = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
        launch(lib.ffb6d_fusion_mlp_pack, w.device, w.data_ptr(), self.Co, self.Ci, self.data.data_ptr(), nbytes)


def fusion_mlp_pack(weight):
    """Prepare a layer's weights for repeated :func:`fusion_mlp` calls (returns a :class:`PackedWeight`)."""
    return PackedWeight(weight)


def fusion_mlp(x1, x2, weight, scale, shift, relu=True, negative_slope=None, add=None, add_idx=None,
               out_channels_last=False):
    """``relu(scale * conv1x1(cat(x1, x2, dim=1)) + shift)`` in one tensor-core kernel
    (``ffb6d_fusion_mlp_fwd_ex``): the fusion layers of FFB6D (models/ffb6d.py:55-80, 104-129 applied
    at :246-262, 282-298: ``torch.cat`` -> ``pt_utils.Conv2d(1x1, bias=False)`` -> BatchNorm -> ReLU)
    with frozen BatchNorm statistics.  Inference (no backward); :mod:`ffb6d_b200.modules` holds the
    training-mode layers.

    :param x1: ``[B, C1, N, 1]`` / ``[B, C1, H, W]`` / ``[B, C1, N]`` float32 CUDA, NCHW-contiguous
    :param x2: second input of the concat with the same trailing shape, or ``None``
    :param weight: ``[Co, C1+C2]`` or ``[Co, C1+C2, 1, 1]`` (``conv.weight``), or the
      :class:`PackedWeight` made from it by :func:`fusion_mlp_pack` (skips the per-call split)
    :param scale, shift: ``[Co]`` folded BatchNorm (:func:`fold_batchnorm`); pass ones / the conv
      bias for a layer without BatchNorm
    :param relu: apply ReLU; with ``negative_slope`` given, LeakyReLU(negative_slope) instead (RandLA's
      ``pt_utils.Conv2d``, models/RandLA/pytorch_utils.py:163-197)
    :param add, add_idx: ``add [B, NA, Co]`` (channels-last) and ``add_idx [B, P]`` / ``[B, P, 1]``: the
      epilogue adds ``add[b, add_idx[b, p], :]`` to the product before the affine (the gathered half of
      a restructured concat layer, see :func:`ffb6d_b200.fusion.p2r_fuse`)
    :param out_channels_last: store the result as ``[B, P, Co]`` (what ``add`` of a following call wants)
    :return: ``[B, Co, ...]`` with the trailing shape of ``x1`` (``[B, P, Co]`` if ``out_channels_last``)
    """
    _need_cuda(x1, "x1")
    if x1.dtype != torch.float32:
        raise TypeError("x1 must be float32")
    B, C1 = x1.shape[0], x1.shape[1]
    tail = tuple(x1.shape[2:])
    x1c = x1.contiguous()
    P = x1c.numel() // max(B * C1, 1)
    C2 = 0
    x2c = None
    if x2 is not None:
        _need_cuda(x2, "x2")
        if x2.dtype != torch.float32 or x2.shape[0] != B or tuple(x2.shape[2:]) != tail:
            raise ValueError("x2 must be float32 with the batch and trailing shape of x1")
        x2c = x2.contiguous()
        C2 = x2.shape[1]
    packed = weight if isinstance(weight, PackedWeight) else PackedWeight(weight)
    Co, Ci = packed.Co, packed.Ci
    if packed.device != x1.device:
        raise ValueError("packed weight lives on %s, inputs on %s" % (packed.device, x1.device))
    if Ci != C1 + C2:
        raise ValueError("weight has %d input channels, inputs have %d" % (Ci, C1 + C2))
    sc, sh = scale.contiguous().float(), shift.contiguous().float()
    if sc.numel() != Co or sh.numel() != Co:
        raise ValueError("scale/shift must have %d elements" % Co)
    addc, idxc, i64, NA = None, None, 0, 0
    if add is not None:
        _need_cuda(add, "add")
        if add_idx is None:
            raise ValueError("add needs add_idx")
        _need_cuda(add_idx, "add_idx")
        if add.dtype != torch.float32 or add.dim() != 3 or add.shape[0] != B or add.shape[2] != Co:
            raise ValueError("add must be float32 [B, NA, Co], got %s" % (tuple(add.shape),))
        addc = add.contiguous()
        NA = addc.shape[1]
        idxc, i64 = _idx_arg(add_idx.reshape(B, -1), "add_idx")
        if idxc.shape[1] != P:
            raise ValueError("add_idx must hold one index per position (%d), got %d" % (P, idxc.shape[1]))
    if out_channels_last:
        out = torch.empty((B, P, Co), dtype=torch.float32, device=x1.device)
    else:
        out = torch.empty((B, Co) + tail, dtype=torch.float32, device=x1.device)
    launch(lib.ffb6d_fusion_mlp_fwd_ex, x1.device, x1c.data_ptr(), C1, ptr(x2c), C2, packed.data.data_ptr(),
           sc.data_ptr(), sh.data_ptr(), B, Co, P, 2 if negative_slope is not None else int(bool(relu)),
           float(negative_slope or 0.0), ptr(addc), ptr(idxc), i64, NA, LAYOUT_NSC if out_channels_last else LAYOUT_NCS,
           out.data_ptr())
    return out


class SegmentPlan:
    """The pixels of every segment of a ``[B, P]`` index map, grouped per segment in ascending order
    (``ffb6d_segment_plan``): what :func:`segment_sum` reads.  Build it once per index map."""
    _bytes, _build, _sum = "ffb6d_segment_plan_bytes", "ffb6d_segment_plan", "ffb6d_segment_sum"

    def __init__(self, idx, n_segments):
        if not isinstance(idx, torch.Tensor):
            raise TypeError("idx must be a torch.Tensor, got %r" % type(idx))
        if idx.dtype not in _IDX:
            raise TypeError("idx must be int32 or int64, got %s" % idx.dtype)
        if idx.dim() not in (2, 3) or (idx.dim() == 3 and idx.shape[2] != 1) or idx.numel() == 0:
            raise ValueError("idx must be a non-empty [B, P] or [B, P, 1], got %s" % (tuple(idx.shape),))
        if int(n_segments) < 1:
            raise ValueError("n_segments must be >= 1, got %d" % int(n_segments))
        _need_cuda(idx, "idx")
        idx_c, i64 = _idx_arg(idx.reshape(idx.shape[0], -1), "idx")
        self.B, self.P, self.NA = int(idx_c.shape[0]), int(idx_c.shape[1]), int(n_segments)
        self.device = idx_c.device
        self.nbytes = int(getattr(lib, self._bytes)(self.B, self.P, self.NA))
        if self.nbytes == 0:
            raise ValueError("no segment plan for B=%d, P=%d, n_segments=%d" % (self.B, self.P, self.NA))
        self.data = workspace(self.nbytes, self.device)
        launch(getattr(lib, self._build), self.device, idx_c.data_ptr(), i64, self.B, self.P, self.NA,
               self.data.data_ptr(), self.nbytes)

    def csr(self):
        """``(offsets [B, n_segments+1], entries [B, P])`` int32 views of the plan; entries past
        ``offsets[b, -1]`` (positions with an out-of-range index) are unspecified."""
        words = self.data.view(torch.int32).view(self.B, -1)
        return words[:, :self.NA + 1], words[:, self.NA + 1:self.NA + 1 + self.P]


class SegmentCSR(SegmentPlan):
    """The same CSR as :class:`SegmentPlan`, built in work and memory linear in P + n_segments
    (``ffb6d_segment_csr``: counts, a device-wide scan, atomic placement, a sort per segment) where SegmentPlan
    keeps n_segments x ceil(P/1024) counters.  For index maps with many segments: the gathers of a training step."""
    _bytes, _build, _sum = "ffb6d_segment_csr_bytes", "ffb6d_segment_csr", "ffb6d_segment_sum_csr"


def segment_plan(idx, n_segments):
    """Plan the segment sum of the index map ``idx [B, P]`` / ``[B, P, 1]`` (int32 or int64 CUDA, values in
    ``[0, n_segments)``; others belong to no segment).  Returns a :class:`SegmentPlan`."""
    return SegmentPlan(idx, n_segments)


def segment_csr(idx, n_segments):
    """:func:`segment_plan` in work and memory linear in P + n_segments; returns a :class:`SegmentCSR`, which
    :func:`segment_sum` takes as its ``plan``."""
    return SegmentCSR(idx, n_segments)


def segment_sum(grad, idx, n_segments, plan=None):
    """``out[b, c, s] = sum of grad[b, c, p] over the pixels p with idx[b, p] = s`` (``ffb6d_segment_sum``): the
    backward of :func:`nearest_interpolation` with the same index, as a deterministic sum without atomics (fp64
    in ascending pixel order, one rounding to fp32; a segment no pixel maps to gets 0).

    :param grad: ``[B, C, P]`` or ``[B, C, h, w]`` (h * w = P) float32 CUDA
    :param idx: ``[B, P]`` or ``[B, P, 1]`` int32 / int64; ignored when ``plan`` is given
    :param plan: a :class:`SegmentPlan` or :class:`SegmentCSR` of ``idx`` (reuse it across calls with the same
      index map); without one, a SegmentPlan is built
    :return: ``[B, C, n_segments]`` float32"""
    if not isinstance(grad, torch.Tensor):
        raise TypeError("grad must be a torch.Tensor, got %r" % type(grad))
    if grad.dtype != torch.float32:
        raise TypeError("grad must be float32, got %s" % grad.dtype)
    if grad.dim() not in (3, 4) or grad.numel() == 0:
        raise ValueError("grad must be a non-empty [B, C, P] or [B, C, h, w], got %s" % (tuple(grad.shape),))
    _need_cuda(grad, "grad")
    B, Cc = int(grad.shape[0]), int(grad.shape[1])
    g = grad.contiguous().reshape(B, Cc, -1)
    if plan is None:
        plan = SegmentPlan(idx, n_segments)
    elif not isinstance(plan, SegmentPlan):
        raise TypeError("plan must be a SegmentPlan, got %r" % type(plan))
    if (plan.B, plan.P, plan.NA) != (B, g.shape[2], int(n_segments)):
        raise ValueError("plan is for B=%d, P=%d, n_segments=%d; grad has B=%d, P=%d and n_segments=%d"
                         % (plan.B, plan.P, plan.NA, B, g.shape[2], int(n_segments)))
    if plan.device != grad.device:
        raise ValueError("plan lives on %s, grad on %s" % (plan.device, grad.device))
    out = torch.empty((B, Cc, plan.NA), dtype=torch.float32, device=grad.device)
    launch(getattr(lib, plan._sum), grad.device, g.data_ptr(), plan.data.data_ptr(), plan.nbytes, B, Cc, plan.P, plan.NA,
           out.data_ptr())
    return out


def att_pool(f1, f2, att):
    """Attentive-pooling core of RandLA's ``Att_pooling`` (models/RandLA/RandLANet.py:245-248):
    ``sum_k cat(f1, f2) * softmax(att, dim=3)`` over the neighbour axis.

    :param f1: ``[B, C1, N, K]`` float32 CUDA; :param f2: ``[B, C2, N, K]`` or None
    :param att: ``[B, C1+C2, N, K]`` attention activations (output of the layer's ``fc``)
    :return: ``[B, C1+C2, N, 1]``
    """
    _need_cuda(f1, "f1")
    _need_cuda(att, "att")
    f1c = f1.contiguous()
    f2c = f2.contiguous() if f2 is not None else None
    B, C1, N, K = f1c.shape
    C2 = f2c.shape[1] if f2c is not None else 0
    a = att.contiguous()
    if tuple(a.shape) != (B, C1 + C2, N, K) or f1c.dtype != torch.float32 or a.dtype != torch.float32:
        raise ValueError("att must be float32 [B,C1+C2,N,K] matching f1/f2")
    out = torch.empty((B, C1 + C2, N, 1), dtype=torch.float32, device=f1.device)
    launch(lib.ffb6d_att_pool_fwd, f1.device, f1c.data_ptr(), C1, ptr(f2c), C2, a.data_ptr(), B, N, K, out.data_ptr())
    return out


def lfa_att_pool_fused(xyz, neigh_idx, feature, mlp1, mlp2, fc_weight, mlp_out, negative_slope=0.2):
    """One attentive pooling of RandLA's ``Building_block`` as ONE kernel (``ffb6d_lfa_att_pool_fused``): relative
    position encoding -> ``mlp1`` [-> ``mlp2``] -> concat with the gathered neighbour features -> ``fc`` -> softmax over
    K -> weighted sum -> output ``mlp`` (models/RandLA/RandLANet.py:196-250); inference, BatchNorm folded.

    :param xyz: ``[B,N,3]``; :param neigh_idx: ``[B,N,16]``; :param feature: ``[B,d/2,N,1]`` (or ``[B,d/2,N]``)
    :param mlp1, mlp2, mlp_out: ``(weight [Co,Ci], scale [Co], shift [Co])`` with BatchNorm folded; ``mlp2`` may be None
    :param fc_weight: ``[d,d]``; :return: ``[B,d_out,N,1]``"""
    _need_cuda(xyz, "xyz")
    _need_cuda(feature, "feature")
    xyz = xyz.contiguous().float()
    idx_c, i64 = _idx_arg(neigh_idx, "neigh_idx")
    B, N, K = idx_c.shape
    f = feature.reshape(B, feature.shape[1], N).contiguous().float()
    Dh = f.shape[1]

    def prep(layer):
        w, sc, sh = layer
        return w.reshape(w.shape[0], -1).contiguous().float(), sc.contiguous().float(), sh.contiguous().float()

    w1, s1, t1 = prep(mlp1)
    w2, s2, t2 = prep(mlp2) if mlp2 is not None else (None, None, None)
    wo, so, to = prep(mlp_out)
    wfc = fc_weight.reshape(fc_weight.shape[0], -1).contiguous().float()
    Do = wo.shape[0]
    if w1.shape != (Dh, 10) or wfc.shape != (2 * Dh, 2 * Dh) or wo.shape[1] != 2 * Dh or (w2 is not None and w2.shape != (Dh, Dh)):
        raise ValueError("layer shapes do not match d/2 = %d" % Dh)
    out = torch.empty((B, Do, N, 1), dtype=torch.float32, device=f.device)
    launch(lib.ffb6d_lfa_att_pool_fused, f.device, xyz.data_ptr(), idx_c.data_ptr(), i64, f.data_ptr(), w1.data_ptr(),
           s1.data_ptr(), t1.data_ptr(), ptr(w2), ptr(s2), ptr(t2), wfc.data_ptr(), wo.data_ptr(), so.data_ptr(),
           to.data_ptr(), B, N, K, Dh, Do, float(negative_slope), out.data_ptr())
    return out


def lfa_fusable(d_half, k):
    """True when :func:`lfa_att_pool_fused` (and the training kernels of :func:`lfa_train_fwd`) cover this width /
    neighbour count."""
    return int(k) == 16 and int(d_half) in (16, 32, 64)


def _lfa_train_args(feature, neigh_idx, f_xyz, w_fc):
    """Shapes first (so that a mismatch reads as one on any device), then the device: dense float32 CUDA tensors
    ``feature [B,Dh,N]``, ``idx [B,N,K]``, ``f_xyz [B,Dh,N,K]``, ``w_fc [2Dh,2Dh]``."""
    if feature.dim() == 4 and feature.shape[3] == 1:
        feature = feature.squeeze(3)
    if feature.dim() != 3:
        raise ValueError("feature must be [B,d/2,N,1] or [B,d/2,N], got %s" % (tuple(feature.shape),))
    B, Dh, N = feature.shape
    if neigh_idx.dim() != 3 or tuple(neigh_idx.shape[:2]) != (B, N):
        raise ValueError("neigh_idx must be [B,N,K] = [%d,%d,K], got %s" % (B, N, tuple(neigh_idx.shape)))
    K = neigh_idx.shape[2]
    if tuple(f_xyz.shape) != (B, Dh, N, K):
        raise ValueError("f_xyz must be [B,d/2,N,K] = %s, got %s" % ((B, Dh, N, K), tuple(f_xyz.shape)))
    w = w_fc.reshape(w_fc.shape[0], -1)
    if tuple(w.shape) != (2 * Dh, 2 * Dh):
        raise ValueError("w_fc must be [d,d] = [%d,%d], got %s" % (2 * Dh, 2 * Dh, tuple(w_fc.shape)))
    for t, name in ((feature, "feature"), (neigh_idx, "neigh_idx"), (f_xyz, "f_xyz"), (w_fc, "w_fc")):
        _need_cuda(t, name)
    for t, name in ((feature, "feature"), (f_xyz, "f_xyz"), (w_fc, "w_fc")):
        if t.dtype != torch.float32:
            raise TypeError("%s must be float32, got %s" % (name, t.dtype))
    idx_c, i64 = _idx_arg(neigh_idx, "neigh_idx")
    return feature.contiguous(), idx_c, i64, f_xyz.contiguous(), w.contiguous(), (B, N, K, Dh)


def lfa_train_fwd(feature, neigh_idx, f_xyz, w_fc):
    """The attentive pooling of a ``Building_block`` on its gathered neighbours, in training (``ffb6d_lfa_train_fwd``):
    ``f_agg = sum_k x_k * softmax_k(w_fc . x_k)`` with ``x_k = cat(feature[:, idx[n, k]], f_xyz[:, n, k])``
    (models/RandLA/RandLANet.py:200-212, 243-248), without materialising the gathered neighbours or the logits.

    :param feature: ``[B,d/2,N,1]`` (or ``[B,d/2,N]``); :param neigh_idx: ``[B,N,16]`` int32 / int64
    :param f_xyz: ``[B,d/2,N,16]``; :param w_fc: ``Att_pooling.fc.weight`` ``[d,d,1,1]`` (or ``[d,d]``)
    :return: ``f_agg [B,d,N,1]``.  K = 16 and d/2 in {16, 32, 64} (:func:`lfa_fusable`); other shapes raise."""
    f, idx_c, i64, fx, w, (B, N, K, Dh) = _lfa_train_args(feature, neigh_idx, f_xyz, w_fc)
    out = torch.empty((B, 2 * Dh, N, 1), dtype=torch.float32, device=f.device)
    launch(lib.ffb6d_lfa_train_fwd, f.device, f.data_ptr(), idx_c.data_ptr(), i64, fx.data_ptr(), w.data_ptr(), B, N, K,
           Dh, out.data_ptr())
    return out


def lfa_train_bwd(feature, neigh_idx, f_xyz, w_fc, grad_agg, need_feature=True):
    """Backward of :func:`lfa_train_fwd` (``ffb6d_lfa_train_bwd``), recomputing the gathered rows, the logits and the
    softmax from the inputs.  Returns ``(grad_feature [B,d/2,N,1] or None, grad_f_xyz [B,d/2,N,16], grad_w_fc [d,d])``.

    The feature half of the gradient comes out of the kernel per edge, ``[B,d/2,N*16]``, the gradient of the per-op
    path's K = 1 neighbour gather, and is scattered onto the points by that gather's own backward
    (:func:`_gather_max_bwd`): fp32 atomics by default, a segment sum under :func:`deterministic_backward`.  The edge
    buffer lives only for this call.  ``grad_w_fc`` is summed without atomics in a fixed order in both modes."""
    f, idx_c, i64, fx, w, (B, N, K, Dh) = _lfa_train_args(feature, neigh_idx, f_xyz, w_fc)
    if tuple(grad_agg.shape) not in ((B, 2 * Dh, N, 1), (B, 2 * Dh, N)):
        raise ValueError("grad_agg must be [B,d,N,1] = %s, got %s" % ((B, 2 * Dh, N, 1), tuple(grad_agg.shape)))
    g = grad_agg.contiguous().float()
    dev = f.device
    edge = torch.empty((B, Dh, N * K), dtype=torch.float32, device=dev)
    gx = torch.empty((B, Dh, N, K), dtype=torch.float32, device=dev)
    gw = torch.empty((2 * Dh, 2 * Dh), dtype=torch.float32, device=dev)
    nbytes = int(lib.ffb6d_lfa_train_bwd_workspace_bytes(B, N, K, Dh))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_lfa_train_bwd, dev, f.data_ptr(), idx_c.data_ptr(), i64, fx.data_ptr(), w.data_ptr(), g.data_ptr(),
           B, N, K, Dh, edge.data_ptr(), gx.data_ptr(), gw.data_ptr(), ws.data_ptr(), nbytes)
    del ws
    gf = None
    if need_feature:
        gf = _gather_max_bwd(f, idx_c.reshape(B, N * K, 1), edge, LAYOUT_NCS).unsqueeze(3)
    return gf, gx, gw.reshape(w_fc.shape)


# --------------------------------------------------------------------------- depth -> point sets
def backproject(depth, K, choose):
    """Depth map -> the point sets of the fusion schedule, on the GPU; replaces ``dpt_2_pcld`` +
    the ``choose`` sampling + the stride pyramids of the datasets
    (datasets/ycb/ycb_dataset.py:165-176, 237, 253-267), bit-identically (float64 math, one
    rounding to float32).

    :param depth: ``[B,H,W]`` float32 CUDA, metres, 0 at holes (``dpt_m`` of the datasets)
    :param K: camera matrix ``[3,3]`` (shared) or ``[B,3,3]``, anything ``np.asarray`` accepts
    :param choose: ``[B,1,N]`` or ``[B,N]`` int32/int64 flat pixel indices of the sampled points
    :return: ``(cld [B,N,3], {2: [B,HW/4,3], 4: [B,HW/16,3], 8: [B,HW/64,3]})`` float32
    """
    _need_cuda(depth, "depth")
    _need_cuda(choose, "choose")
    if depth.dim() != 3 or depth.dtype != torch.float32:
        raise ValueError("depth must be float32 [B,H,W], got %s %s" % (depth.dtype, tuple(depth.shape)))
    depth = depth.contiguous()
    intr_d, per_frame = _intrinsics_arg(K, depth.shape[0], depth.device)
    return _backproject(depth, intr_d, per_frame, choose)


def _intrinsics_arg(K, B, dev):
    """``K`` as :func:`backproject` takes it -> ``(float64 (fx, fy, cx, cy) [4] or [B,4] on dev, per_frame)``."""
    if isinstance(K, torch.Tensor) and K.is_cuda:
        # (fx, fy, cx, cy) already on the device: [4] shared or [B,4] (no host copy: graph-capturable)
        if K.dtype != torch.float64 or K.shape not in ((4,), (B, 4)):
            raise ValueError("device intrinsics must be float64 [4] or [B,4] = (fx, fy, cx, cy)")
        return K.contiguous(), int(K.dim() == 2)
    Kn = np.asarray(K, dtype=np.float64)
    if Kn.shape not in ((3, 3), (B, 3, 3)):
        raise ValueError("K must be [3,3] or [B,3,3], got %s" % (Kn.shape,))
    return intrinsics_to_device(Kn, dev), int(Kn.ndim == 3)


def _frame_intrinsics(K):
    """Per-frame camera matrices ``[B,3,3]`` float64 CUDA -> ``(fx, fy, cx, cy)`` ``[B,4]`` on the device."""
    return torch.stack((K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]), 1).contiguous()


def point_item(depth_m, K, choose, rgb, labels, nrm_map, obj_cls, obj_kps, obj_ctr):
    """The sampled points' input features and pose-training targets on the GPU (``ffb6d_point_item``): the half of
    the datasets' ``get_item`` that reads ``choose`` (datasets/ycb/ycb_dataset.py:237-247 and ``get_pose_gt_info``
    :348-386; datasets/linemod/linemod_dataset.py:284-293, 398-436), bit-identical to the reference.

    :param depth_m: ``[B,H,W]`` float32 CUDA, metres (``dpt_m``); :param K: camera matrix as :func:`backproject`
      takes it
    :param choose: ``[B,1,N]`` or ``[B,N]`` int32 / int64 CUDA flat pixel indices
    :param rgb: ``[B,H,W,3]`` uint8; :param labels: ``[B,H,W]`` uint8 label image
    :param nrm_map: ``[B,H,W,3]`` float32, or float64 (rounded once to float32, as the reference's concat + cast does)
    :param obj_cls: ``[B,n_obj]`` int32 class id per object slot (< 0: empty slot)
    :param obj_kps: ``[B,n_obj,n_kps,3]`` float64 posed keypoints; :param obj_ctr: ``[B,n_obj,3]`` float64 posed centres
      (the tables of :func:`ffb6d_b200.item.pose_gt_objects`)
    :return: ``(cld_rgb_nrm [B,9,N] f32, labels [B,N] i32, kp_targ_ofst [B,N,n_kps,3] f32, ctr_targ_ofst [B,N,3] f32)``
    """
    tensors = ((depth_m, "depth_m"), (choose, "choose"), (rgb, "rgb"), (labels, "labels"), (nrm_map, "nrm_map"),
               (obj_cls, "obj_cls"), (obj_kps, "obj_kps"), (obj_ctr, "obj_ctr"))
    B, H, W = _point_input_checks(tensors, depth_m, choose, rgb, nrm_map)
    if labels.dtype != torch.uint8 or tuple(labels.shape) != (B, H, W):
        raise ValueError("labels must be uint8 [B,H,W], got %s %s" % (labels.dtype, tuple(labels.shape)))
    if obj_cls.dtype != torch.int32 or obj_cls.dim() != 2 or obj_cls.shape[0] != B:
        raise ValueError("obj_cls must be int32 [B,n_obj], got %s %s" % (obj_cls.dtype, tuple(obj_cls.shape)))
    n_obj = obj_cls.shape[1]
    if obj_kps.dtype != torch.float64 or obj_kps.dim() != 4 or tuple(obj_kps.shape[:2]) != (B, n_obj) \
            or obj_kps.shape[3] != 3:
        raise ValueError("obj_kps must be float64 [B,n_obj,n_kps,3], got %s %s" % (obj_kps.dtype, tuple(obj_kps.shape)))
    n_kps = obj_kps.shape[2]
    if obj_ctr.dtype != torch.float64 or tuple(obj_ctr.shape) != (B, n_obj, 3):
        raise ValueError("obj_ctr must be float64 [B,n_obj,3], got %s %s" % (obj_ctr.dtype, tuple(obj_ctr.shape)))
    _same_cuda_device(tensors, depth_m)
    dev = depth_m.device
    intr_d, per_frame = _intrinsics_arg(K, B, dev)
    ch = choose.reshape(B, -1).to(torch.int32).contiguous()
    N = ch.shape[1]
    nrm = nrm_map.to(torch.float32).contiguous()
    cld_rgb_nrm = torch.empty((B, 9, N), dtype=torch.float32, device=dev)
    labels_pt = torch.empty((B, N), dtype=torch.int32, device=dev)
    kp_targ_ofst = torch.empty((B, N, n_kps, 3), dtype=torch.float32, device=dev)
    ctr_targ_ofst = torch.empty((B, N, 3), dtype=torch.float32, device=dev)
    args = [t.contiguous() for t in (depth_m, rgb, labels, obj_cls, obj_kps, obj_ctr)]
    depth_c, rgb_c, labels_c, cls_c, kps_c, ctr_c = args
    launch(lib.ffb6d_point_item, dev, depth_c.data_ptr(), B, H, W, intr_d.data_ptr(), per_frame, ch.data_ptr(), N,
           rgb_c.data_ptr(), labels_c.data_ptr(), nrm.data_ptr(), cls_c.data_ptr(), kps_c.data_ptr(), ctr_c.data_ptr(),
           n_obj, n_kps, cld_rgb_nrm.data_ptr(), labels_pt.data_ptr(), kp_targ_ofst.data_ptr(), ctr_targ_ofst.data_ptr())
    return cld_rgb_nrm, labels_pt, kp_targ_ofst, ctr_targ_ofst


def _point_input_checks(tensors, depth_m, choose, rgb, nrm_map):
    """The argument checks :func:`point_item` and :func:`point_input` share (types of all ``tensors``, then the
    depth map, ``choose``, ``rgb`` and ``nrm_map``); returns ``(B, H, W)``."""
    for t, name in tensors:
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor, got %r" % (name, type(t)))
    if depth_m.dim() != 3 or depth_m.dtype != torch.float32:
        raise ValueError("depth_m must be float32 [B,H,W], got %s %s" % (depth_m.dtype, tuple(depth_m.shape)))
    B, H, W = depth_m.shape
    if choose.dtype not in _IDX:
        raise ValueError("choose must be int32 or int64, got %s" % choose.dtype)
    if not (choose.dim() == 2 or (choose.dim() == 3 and choose.shape[1] == 1)) or choose.shape[0] != B:
        raise ValueError("choose must be [B,1,N] or [B,N], got %s" % (tuple(choose.shape),))
    if rgb.dtype != torch.uint8 or tuple(rgb.shape) != (B, H, W, 3):
        raise ValueError("rgb must be uint8 [B,H,W,3] = %s, got %s %s" % ((B, H, W, 3), rgb.dtype, tuple(rgb.shape)))
    if nrm_map.dtype not in (torch.float32, torch.float64) or tuple(nrm_map.shape) != (B, H, W, 3):
        raise ValueError("nrm_map must be float32 or float64 [B,H,W,3], got %s %s" % (nrm_map.dtype, tuple(nrm_map.shape)))
    return B, H, W


def _same_cuda_device(tensors, depth_m):
    for t, name in tensors:
        _need_cuda(t, name)
        if t.device != depth_m.device:
            raise ValueError("%s is on %s, depth_m on %s" % (name, t.device, depth_m.device))


def point_input(depth_m, K, choose, rgb, nrm_map):
    """The sampled points' network input on the GPU (``ffb6d_point_input``): ``cld_rgb_nrm [B,9,N]`` float32, the
    point of each ``choose`` pixel, its colour and its normal, bitwise ``point_item(...)[0]`` for the same
    arguments.  It needs no labels and no objects, so it serves frames whose pose is to be estimated.  Arguments
    and checks as :func:`point_item`."""
    tensors = ((depth_m, "depth_m"), (choose, "choose"), (rgb, "rgb"), (nrm_map, "nrm_map"))
    B, H, W = _point_input_checks(tensors, depth_m, choose, rgb, nrm_map)
    _same_cuda_device(tensors, depth_m)
    dev = depth_m.device
    intr_d, per_frame = _intrinsics_arg(K, B, dev)
    ch = choose.reshape(B, -1).to(torch.int32).contiguous()
    N = ch.shape[1]
    nrm = nrm_map.to(torch.float32).contiguous()
    cld_rgb_nrm = torch.empty((B, 9, N), dtype=torch.float32, device=dev)
    depth_c, rgb_c = depth_m.contiguous(), rgb.contiguous()
    launch(lib.ffb6d_point_input, dev, depth_c.data_ptr(), B, H, W, intr_d.data_ptr(), per_frame, ch.data_ptr(), N,
           rgb_c.data_ptr(), nrm.data_ptr(), cld_rgb_nrm.data_ptr())
    return cld_rgb_nrm


def _device_seed(seed, dev):
    """``seed`` when it is a one-element int64 / uint64 CUDA tensor on ``dev`` (read on the device by the ``_dseed``
    entry points, so a captured call takes a new seed per replay; its 64 bits are the seed), None for a host int."""
    if not isinstance(seed, torch.Tensor):
        return None
    if not seed.is_cuda or seed.device != dev or seed.dtype not in (torch.int64, torch.uint64) or seed.numel() != 1:
        raise ValueError("a tensor seed must be one int64 / uint64 element on %s, got %s %s on %s"
                         % (dev, seed.dtype, tuple(seed.shape), seed.device))
    return seed.contiguous()


def sample_valid_pixels(depth, n_points, seed=0, min_depth=1e-8, return_count=False):
    """The datasets' point sampling on the GPU (datasets/ycb/ycb_dataset.py:218-235): the valid pixels of each
    depth map (``depth > min_depth``) are compacted, ``n_points`` of them are drawn uniformly without replacement
    (all of them, repeated cyclically like ``np.pad(..., 'wrap')``, when fewer exist) and returned in uniformly
    random order.  Deterministic per ``seed``; the picks have the reference's distribution but do not replay
    numpy's random stream.

    :param depth: ``[B,H,W]`` float32 CUDA; :param seed: an int, or a one-element int64 / uint64 CUDA tensor read on
      the device (the same picks as the int of the same 64 bits)
    :return: ``choose [B,1,n_points]`` int32 flat pixel indices
      (what :func:`backproject` and the final ``choose`` gather take); with ``return_count`` also the number
      of valid pixels per frame ``[B]`` int32."""
    _need_cuda(depth, "depth")
    if depth.dim() != 3 or depth.dtype != torch.float32:
        raise ValueError("depth must be float32 [B,H,W]")
    depth = depth.contiguous()
    B, H, W = depth.shape
    dev = depth.device
    choose = torch.empty((B, 1, int(n_points)), dtype=torch.int32, device=dev)
    count = torch.empty((B,), dtype=torch.int32, device=dev)
    nbytes = int(lib.ffb6d_sample_pixels_workspace_bytes(B, H, W))
    ws = workspace(nbytes, dev)
    seed_d = _device_seed(seed, dev)
    if seed_d is None:
        launch(lib.ffb6d_sample_pixels, dev, depth.data_ptr(), B, H, W, float(min_depth), int(n_points),
               int(seed) & (2 ** 64 - 1), choose.data_ptr(), count.data_ptr(), ws.data_ptr(), nbytes)
    else:
        launch(lib.ffb6d_sample_pixels_dseed, dev, depth.data_ptr(), B, H, W, float(min_depth), int(n_points),
               seed_d.data_ptr(), choose.data_ptr(), count.data_ptr(), ws.data_ptr(), nbytes)
    return (choose, count) if return_count else choose


def fill_missing(dpt, cam_scale, scale_2_80m=1, fill_type='multiscale', extrapolate=False, show_process=False,
                 blur_type='bilateral'):
    """Depth completion of raw sensor depth on the GPU: ``Basic_Utils.fill_missing``
    (utils/basic_utils.py:467-487) as ``datasets/ycb/ycb_dataset.py:204`` calls it, i.e. ip_basic's
    ``fill_in_multiscale`` (utils/ip_basic/ip_basic/depth_map_utils_ycb.py:290-443) with ``max_depth=3.0``
    (``ffb6d_fill_depth``).  Every pixel the final bilateral blur leaves alone is bit-identical to the
    reference; the blurred ones differ from OpenCV's by at most 2e-6 m (exact weights instead of its table).

    :param dpt: ``[B,H,W]`` or ``[H,W]`` ``torch.uint16`` CUDA tensor, the depth PNG's raw values
    :param cam_scale: raw units per metre (``meta['factor_depth']``), used as float32 like the dataset's
    :param scale_2_80m, fill_type, extrapolate, blur_type: only the dataset's ``1``, ``'multiscale'``,
      ``False``, ``'bilateral'`` are implemented; anything else raises ``ValueError``
    :param show_process: accepted and ignored (the reference's ``fill_missing`` drops the process images too)
    :return: float32 completed depth in raw units, the shape of ``dpt``
    """
    return _fill_depth(dpt, cam_scale, scale_2_80m, fill_type, extrapolate, blur_type, want_m=False)[0]


def _fill_depth(dpt, cam_scale, scale_2_80m=1, fill_type='multiscale', extrapolate=False, blur_type='bilateral',
                want_raw=True, want_m=True):
    """:func:`fill_missing` returning ``(filled_raw, depth_m)`` (``None`` for an output not wanted)."""
    if fill_type != 'multiscale':
        raise ValueError("fill_type %r is not implemented: only 'multiscale' (the YCB dataset's)" % (fill_type,))
    if extrapolate is not False:
        raise ValueError("extrapolate=%r is not implemented: only False (the YCB dataset's)" % (extrapolate,))
    if blur_type != 'bilateral':
        raise ValueError("blur_type %r is not implemented: only 'bilateral' (the YCB dataset's)" % (blur_type,))
    if isinstance(scale_2_80m, bool) or scale_2_80m != 1:
        raise ValueError("scale_2_80m=%r is not implemented: only 1 (the YCB dataset's)" % (scale_2_80m,))
    cs = float(np.float32(cam_scale))
    if not (cs > 0.0 and np.isfinite(cs)):
        raise ValueError("cam_scale must be positive and finite, got %r" % (cam_scale,))
    if not isinstance(dpt, torch.Tensor):
        raise TypeError("dpt must be a torch.Tensor, got %r" % type(dpt))
    if dpt.dtype != torch.uint16 or dpt.dim() not in (2, 3) or dpt.numel() == 0:
        raise ValueError("dpt must be a non-empty torch.uint16 [B,H,W] or [H,W] tensor, got %s %s"
                         % (dpt.dtype, tuple(dpt.shape)))
    _need_cuda(dpt, "dpt")
    raw = dpt.contiguous()
    B, H, W = (1,) + tuple(raw.shape) if raw.dim() == 2 else tuple(raw.shape)
    dev = raw.device
    outs = [torch.empty(raw.shape, dtype=torch.float32, device=dev) if want else None for want in (want_raw, want_m)]
    nbytes = int(lib.ffb6d_fill_depth_workspace_bytes(B, H, W))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_fill_depth, dev, raw.data_ptr(), B, H, W, cs, ptr(outs[0]), ptr(outs[1]), ws.data_ptr(), nbytes)
    return tuple(outs)


def depth_normal(dpt_mm, K, k_size=5, distance_threshold=2000, difference_threshold=20, point_into_surface=False):
    """Surface normals of millimetre depth maps on the GPU (``ffb6d_depth_normal``, DESIGN.md §4.30): the batched
    ``normalSpeed.depth_normal(d, K[0][0], K[1][1], k_size, distance_threshold, difference_threshold,
    point_into_surface)`` of the datasets (datasets/ycb/ycb_dataset.py:207-210), computed by a specified estimator: the
    least-squares depth-gradient fit of OpenCV's LINEMOD with the camera's fx, fy.  Whether ``normalSpeed`` gives the
    same values is not known; the reference's trained checkpoints were trained on ``normalSpeed``'s.

    :param dpt_mm: ``[H,W]`` or ``[B,H,W]`` ``torch.uint16`` CUDA, depth in millimetres (0 = hole)
    :param K: camera matrix as :func:`backproject` takes it (host ``[3,3]`` / ``[B,3,3]``, or device float64
      ``(fx, fy, cx, cy)`` ``[4]`` / ``[B,4]``: no host copy, capturable); only fx and fy are read
    :param k_size: the neighbour offset r in pixels; :param distance_threshold: depths at or beyond it (mm) get a zero
      normal; :param difference_threshold: neighbours whose depth differs by this many mm or more are left out
    :param point_into_surface: negate the normals (they face the camera by default)
    :return: float32 ``[..., H, W, 3]``; ``(0, 0, 0)`` at holes, beyond ``distance_threshold`` and where the fit is
      degenerate
    """
    _need_cuda(dpt_mm, "dpt_mm")
    if dpt_mm.dtype != torch.uint16 or dpt_mm.dim() not in (2, 3):
        raise ValueError("dpt_mm must be torch.uint16 [H,W] or [B,H,W], got %s %s" % (dpt_mm.dtype, tuple(dpt_mm.shape)))
    for name, v in (("k_size", k_size), ("distance_threshold", distance_threshold),
                    ("difference_threshold", difference_threshold)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError("%s must be an int, got %r" % (name, v))
    d = dpt_mm.contiguous()
    B, H, W = (1,) + tuple(d.shape) if d.dim() == 2 else tuple(d.shape)
    dev = d.device
    intr_d, per_frame = _intrinsics_arg(K, B, dev)
    nrm = torch.empty(tuple(d.shape) + (3,), dtype=torch.float32, device=dev)
    launch(lib.ffb6d_depth_normal, dev, d.data_ptr(), B, H, W, intr_d.data_ptr(), per_frame, int(k_size),
           int(distance_threshold), int(difference_threshold), int(bool(point_into_surface)), nrm.data_ptr())
    return nrm


def orb_detect(rgb):
    """ORB keypoints of ``cv2.ORB_create()``'s defaults on the GPU (``ffb6d_orb_detect``, DESIGN.md §4.32): what
    ``ORB_create().detect`` returns for each frame's BGR image, bit for bit as a set (pinned through
    oracle/orb_oracle.py), in level then raster order.

    :param rgb: ``[B,H,W,3]`` (or ``[H,W,3]``) uint8 CUDA, RGB as :func:`ffb6d_b200.render.render_rgbd` returns it;
      ``2 <= H, W <= 8192``
    :return: ``(count [B] int32, pt [B,cap,2] float32 (x, y), octave [B,cap] int32, response [B,cap] float32)`` on
      the device (no synchronisation); frame b's keypoints are its first ``count[b]`` rows (later rows hold
      scratch).  ``cap`` (``ffb6d_orb_capacity``) bounds what the detector can keep, so nothing is ever clipped.
    """
    if not isinstance(rgb, torch.Tensor) or rgb.dtype != torch.uint8:
        raise ValueError("orb_detect: rgb must be a uint8 tensor, got %s" % getattr(rgb, "dtype", type(rgb).__name__))
    _need_cuda(rgb, "rgb")
    if rgb.dim() not in (3, 4) or rgb.shape[-1] != 3:
        raise ValueError("orb_detect: rgb must be [B,H,W,3] or [H,W,3], got %s" % (tuple(rgb.shape),))
    x = rgb.contiguous() if rgb.dim() == 4 else rgb.contiguous()[None]
    B, H, W = (int(n) for n in x.shape[:3])
    if not (_lib.ORB_MIN_SIDE <= H <= _lib.ORB_MAX_SIDE and _lib.ORB_MIN_SIDE <= W <= _lib.ORB_MAX_SIDE):
        raise ValueError("orb_detect: H and W must lie in [%d, %d], got %dx%d"
                         % (_lib.ORB_MIN_SIDE, _lib.ORB_MAX_SIDE, H, W))
    if B > _lib.ORB_MAX_FRAMES:
        raise ValueError("orb_detect: at most %d frames, got %d" % (_lib.ORB_MAX_FRAMES, B))
    cap = int(lib.ffb6d_orb_capacity(H, W))
    dev = x.device
    count = torch.zeros(B, dtype=torch.int32, device=dev)
    pt = torch.zeros((B, cap, 2), dtype=torch.float32, device=dev)
    octave = torch.zeros((B, cap), dtype=torch.int32, device=dev)
    response = torch.zeros((B, cap), dtype=torch.float32, device=dev)
    nbytes = int(lib.ffb6d_orb_workspace_bytes(B, H, W))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_orb_detect, dev, x.data_ptr(), B, H, W, count.data_ptr(), pt.data_ptr(), octave.data_ptr(),
           response.data_ptr(), cap, ws.data_ptr(), nbytes)
    return count, pt, octave, response


def orb_lift(count, pt, depth, K, RTs, views):
    """Lift the keypoints of :func:`orb_detect` into the object frame as the reference's textured keypoint tool does
    (``ffb6d_orb_lift``; rgbd_rnder_sift_kp3ds.py:138-155): the depth at ``(int(pt.y), int(pt.x))`` back-projected,
    points with a non-finite x or ``z <= 1e-8`` dropped, then ``(p - t) . R``.

    :param count, pt: as :func:`orb_detect` returns them for ``B = n_obj * views`` renders, object o's views being
      frames ``o * views ... o * views + views - 1``
    :param depth: ``[B,H,W]`` float32 CUDA metres (0 where nothing is drawn)
    :param K: camera as :func:`backproject` takes it; :param RTs: ``[B,3,4]`` or ``[B,4,4]`` object-to-camera poses
      (host arrays or CUDA tensors, taken as float64)
    :return: ``(cloud [n_obj, views * cap, 3] float32, n_points [n_obj] int32)`` on the device: each object's points,
      views in order, ready for ``farthest_point_sampling(cloud, n, n_points=n_points)``.
    """
    for t, name in ((count, "count"), (pt, "pt"), (depth, "depth")):
        _need_cuda(t, name)
    if count.dtype != torch.int32 or pt.dtype != torch.float32 or depth.dtype != torch.float32:
        raise ValueError("orb_lift: count must be int32, pt and depth float32")
    if depth.dim() != 3 or count.dim() != 1 or pt.dim() != 3 or pt.shape[-1] != 2:
        raise ValueError("orb_lift: need count [B], pt [B,cap,2] and depth [B,H,W]")
    B, H, W = (int(n) for n in depth.shape)
    cap = int(lib.ffb6d_orb_capacity(H, W))
    if tuple(count.shape) != (B,) or tuple(pt.shape) != (B, cap, 2):
        raise ValueError("orb_lift: count must be [%d] and pt [%d,%d,2] for %dx%d frames, got %s and %s"
                         % (B, B, cap, H, W, tuple(count.shape), tuple(pt.shape)))
    if isinstance(views, bool) or not isinstance(views, (int, np.integer)) or views < 1 or B % views:
        raise ValueError("orb_lift: views must be a positive int dividing B=%d, got %r" % (B, views))
    views = int(views)
    if B // views > _lib.ORB_MAX_OBJECTS or views * cap >= 1 << 31:
        raise ValueError("orb_lift: %d objects of %d views exceed the limits" % (B // views, views))
    dev = depth.device
    rt = RTs if isinstance(RTs, torch.Tensor) else torch.from_numpy(np.asarray(RTs, np.float64))
    if rt.dim() != 3 or rt.shape[0] != B or tuple(rt.shape[1:]) not in ((3, 4), (4, 4)):
        raise ValueError("orb_lift: RTs must be [B,3,4] or [B,4,4], got %s" % (tuple(rt.shape),))
    rt = rt[:, :3, :].to(device=dev, dtype=torch.float64).contiguous()
    intr, per_frame = _intrinsics_arg(K, B, dev)
    cloud = torch.zeros((B // views, views * cap, 3), dtype=torch.float32, device=dev)
    n_points = torch.zeros(B // views, dtype=torch.int32, device=dev)
    launch(lib.ffb6d_orb_lift, dev, count.contiguous().data_ptr(), pt.contiguous().data_ptr(), cap,
           depth.contiguous().data_ptr(), B, H, W, intr.data_ptr(), per_frame, rt.data_ptr(), views,
           cloud.data_ptr(), n_points.data_ptr())
    return cloud, n_points


def depth_to_mm(depth, divisor=10.0):
    """``(depth / divisor).astype(np.uint16)`` on the GPU (``ffb6d_depth_to_mm``): a float32 IEEE division, then a
    truncation, as numpy computes it for in-range values (out of range, where numpy's cast is undefined, it saturates).
    With ``divisor`` 10 this is the YCB dataset's millimetre map of the completed depth (ycb_dataset.py:207).

    :param depth: float32 CUDA tensor of any shape; :return: ``torch.uint16`` of the same shape"""
    _need_cuda(depth, "depth")
    if depth.dtype != torch.float32:
        raise ValueError("depth must be float32, got %s" % depth.dtype)
    src = depth.contiguous()
    out = torch.empty(src.shape, dtype=torch.uint16, device=src.device)
    launch(lib.ffb6d_depth_to_mm, src.device, src.data_ptr(), src.numel(), float(np.float32(divisor)), out.data_ptr())
    return out


def intrinsics_to_device(K, device, batch=None):
    """Camera matrix ``[3,3]`` / ``[B,3,3]`` -> float64 ``[4]`` / ``[B,4]`` (fx, fy, cx, cy) on the device."""
    Kn = np.asarray(K, dtype=np.float64)
    if Kn.ndim == 2:
        v = np.array([Kn[0, 0], Kn[1, 1], Kn[0, 2], Kn[1, 2]], np.float64)
    else:
        v = np.stack([Kn[:, 0, 0], Kn[:, 1, 1], Kn[:, 0, 2], Kn[:, 1, 2]], 1).copy()
    return torch.from_numpy(v).to(device)


def _backproject(depth, intr_d, per_frame, choose):
    B, H, W = depth.shape
    dev = depth.device
    ch = choose.reshape(B, -1)
    if ch.dtype != torch.int32 or not ch.is_contiguous():
        ch = ch.to(torch.int32).contiguous()
    N = ch.shape[1]
    cld = torch.empty((B, N, 3), dtype=torch.float32, device=dev)
    pyr = {s: torch.empty((B, (H // s) * (W // s), 3), dtype=torch.float32, device=dev) for s in (2, 4, 8)}
    launch(lib.ffb6d_backproject, dev, depth.data_ptr(), B, H, W, intr_d.data_ptr(), per_frame, ch.data_ptr(), N,
           cld.data_ptr(), pyr[2].data_ptr(), pyr[4].data_ptr(), pyr[8].data_ptr())
    return cld, pyr


# --------------------------------------------------------------------------- grid subsampling
def grid_sub_sampling(points, features=None, labels=None, grid_size=0.1, verbose=0):
    """Voxel-grid barycentre subsampling; mirrors ``DataProcessing.grid_sub_sampling``
    (models/RandLA/helper_tool.py:199-219) and the wrapper's argument checks
    (GS/cpp_subsampling/wrapper.cpp:96-190).

    :param points: (N, 3) float32 points
    :param features: optional (N, d) float32 features
    :param labels: optional (N,) or (N, ld) int32 labels
    :param grid_size: voxel size
    :return: sub-sampled points, then features and/or labels if given (numpy arrays).
      Rows are ordered by ascending voxel key (the reference's row order is that of a
      hash map and carries no meaning).
    """
    pts = np.ascontiguousarray(points, dtype=np.float32)
    if pts.ndim != 2 or pts.shape[1] != 3:
        raise RuntimeError("Wrong dimensions : points.shape is not (N, 3)")      # wrapper.cpp:133-141
    N = pts.shape[0]
    if N < 1:
        raise RuntimeError("Error")                                              # wrapper.cpp:225-229
    feats = None
    fdim = 0
    if features is not None:
        feats = np.ascontiguousarray(features, dtype=np.float32)
        if feats.ndim != 2 or feats.shape[0] != N:
            raise RuntimeError("Wrong dimensions : features.shape is not (N, d)")  # :143-159
        fdim = feats.shape[1]
    cls = None
    ldim = 0
    if labels is not None:
        cls = np.ascontiguousarray(labels, dtype=np.int32)
        if cls.ndim > 2 or cls.shape[0] != N:
            raise RuntimeError("Wrong dimensions : classes.shape is not (N,) or (N, d)")  # :161-177
        ldim = 1 if cls.ndim == 1 else cls.shape[1]
    sub_p = np.empty((N, 3), np.float32)
    sub_f = np.empty((N, max(fdim, 1)), np.float32)
    sub_c = np.empty((N, max(ldim, 1)), np.int32)
    M = C.c_size_t(0)
    check(lib.ffb6d_grid_subsample_host(
        pts.ctypes.data, N, feats.ctypes.data if feats is not None else None, fdim,
        cls.ctypes.data if cls is not None else None, ldim, float(grid_size),
        sub_p.ctypes.data, sub_f.ctypes.data, sub_c.ctypes.data, C.byref(M)))
    m = M.value
    out = [sub_p[:m].copy()]
    if feats is not None:
        out.append(sub_f[:m, :fdim].copy())
    if cls is not None:
        out.append(sub_c[:m, :ldim].copy())      # wrapper.cpp:240-243: classes come back [M, ld]
    return out[0] if len(out) == 1 else tuple(out)


# --------------------------------------------------------------------------- farthest point sampling
def _fps_host_ints(v, G, n, name):
    """A host start / count argument: an int or G ints, as int32 [G]; None for a CUDA tensor (checked on the device)."""
    if isinstance(v, torch.Tensor) and v.is_cuda:
        return None
    a = np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v)
    if a.dtype.kind not in "iu":
        raise TypeError("%s must hold integers, got %s" % (name, a.dtype))
    a = np.broadcast_to(a, (G,)) if a.ndim == 0 else a
    if a.shape != (G,):
        raise ValueError("%s must be an int or %d ints, got shape %s" % (name, G, a.shape))
    if n is not None and (np.any(a < 0) or np.any(a >= n)):
        raise ValueError("%s must lie in [0, %s), got %s" % (name, n, a))
    return a.astype(np.int32)


def farthest_point_sampling(pts, sn, init_center=False, start=None, return_index=False, n_points=None):
    """Farthest point sampling on the GPU; mirrors ``fps_utils.farthest_point_sampling`` (utils/dataset_tools/fps/
    fps_utils.py:8-23), whose selection it reproduces bit for bit (include/ffb6d_b200.h).

    :param pts: numpy ``[P,3]`` (copied to the current CUDA device as float32, as the reference converts it), or a
      float32 CUDA tensor ``[P,3]`` or ``[G,P,3]`` (G clouds in one launch)
    :param sn: number of points to select, ``1 <= sn <= FFB6D_FPS_MAX_SAMPLES``; ``sn > P`` repeats index 0
    :param init_center: start from the point farthest from the centre of the bounding box (deterministic)
    :param start: without ``init_center``, the first index of each cloud: an int, ``G`` ints, or an int32 CUDA tensor
      ``[G]`` (host values are range-checked here; a CUDA tensor's are checked by the kernel, which writes -1 into
      the rows of clouds whose start is out of range).  ``None`` draws it uniformly from torch's CUDA generator,
      where the reference uses ``rand()``
    :param n_points: cloud ``g`` is its first ``n_points[g]`` points (int, ``G`` ints or int32 CUDA tensor);
      ``None``: all ``P``
    :return: ``pts[idxs]`` (``[sn,3]`` / ``[G,sn,3]``, numpy for numpy input), and with ``return_index`` also the
      indices (int32)
    """
    as_numpy = not isinstance(pts, torch.Tensor)
    if as_numpy:
        x = np.ascontiguousarray(pts, np.float32)
        if x.ndim != 2 or x.shape[1] != 3:
            raise ValueError("pts must be [P,3], got shape %s" % (x.shape,))
    else:
        _need_cuda(pts, "pts")
        if pts.dtype != torch.float32:
            raise TypeError("pts must be float32, got %s" % pts.dtype)
        if pts.dim() not in (2, 3) or pts.shape[-1] != 3:
            raise ValueError("pts must be [P,3] or [G,P,3], got shape %s" % (tuple(pts.shape),))
        x = pts
    single = x.ndim == 2
    G, P = (1, x.shape[0]) if single else x.shape[:2]
    if isinstance(sn, bool) or not isinstance(sn, (int, np.integer)):
        raise TypeError("sn must be an int, got %r" % (sn,))
    sn = int(sn)
    if not 1 <= sn <= _lib.FPS_MAX_SAMPLES:
        raise ValueError("sn must lie in [1, %d], got %d" % (_lib.FPS_MAX_SAMPLES, sn))
    if not (1 <= G <= _lib.FPS_MAX_CLOUDS and 1 <= P <= _lib.FPS_MAX_POINTS):
        raise ValueError("need 1 <= G <= %d clouds of 1 <= P <= %d points, got G=%d, P=%d"
                         % (_lib.FPS_MAX_CLOUDS, _lib.FPS_MAX_POINTS, G, P))
    counts_h = st_h = None
    n_hi = P
    if n_points is not None:
        counts_h = _fps_host_ints(n_points, G, None, "n_points")
        if counts_h is None:
            if n_points.dtype != torch.int32 or tuple(n_points.shape) != (G,):
                raise ValueError("n_points must be an int32 CUDA tensor [%d]" % G)
        elif np.any(counts_h < 1) or np.any(counts_h > P):
            raise ValueError("n_points must lie in [1, %d], got %s" % (P, counts_h))
        else:
            n_hi = counts_h
    if not init_center and start is not None:
        st_h = _fps_host_ints(start, G, n_hi, "start")
        if st_h is None and (start.dtype != torch.int32 or tuple(start.shape) != (G,)):
            raise ValueError("start must be an int32 CUDA tensor [%d]" % G)

    x = torch.from_numpy(x).to(torch.device("cuda", torch.cuda.current_device())) if as_numpy else x
    x = (x[None] if single else x).contiguous()
    dev = x.device
    counts = None
    if n_points is not None:
        counts = torch.from_numpy(counts_h).to(dev) if counts_h is not None else n_points.to(dev).contiguous()
    st = None
    if not init_center:
        if start is None:
            n = counts.to(torch.float64) if counts is not None else torch.full((G,), float(P), dtype=torch.float64,
                                                                                device=dev)
            st = torch.minimum((torch.rand(G, dtype=torch.float64, device=dev) * n).floor(), n - 1).to(torch.int32)
        else:
            st = torch.from_numpy(st_h).to(dev) if st_h is not None else start.to(dev).contiguous()
    idx = torch.empty((G, sn), dtype=torch.int32, device=dev)
    nbytes = int(lib.ffb6d_farthest_point_sampling_workspace_bytes(G, P, sn))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_farthest_point_sampling, dev, x.data_ptr(), ptr(counts), G, P, sn, ptr(st), int(bool(init_center)),
           idx.data_ptr(), ws.data_ptr(), nbytes)
    sel = torch.gather(x, 1, idx.clamp(min=0).long()[..., None].expand(G, sn, 3))
    if single:
        sel, idx = sel[0], idx[0]
    if as_numpy:
        sel, idx = sel.cpu().numpy(), idx.cpu().numpy()
    return (sel, idx) if return_index else sel


def pose_add_adds(mesh_pts, mesh_off, obj_mesh, pred_RT, gt_RT, max_points):
    """ADD and ADD-S of ``M`` predicted poses in one launch: ``Basic_Utils.cal_add_cuda`` / ``cal_adds_cuda``
    (utils/basic_utils.py:651-669) for every object of a batch.

    ``mesh_pts [P,3]`` float32: the meshes stacked; ``mesh_off [n_meshes+1]`` int32: mesh ``c`` is rows
    ``mesh_off[c] .. mesh_off[c+1]``; ``obj_mesh [M]`` int32: each object's mesh; ``pred_RT``, ``gt_RT [M,3,4]``
    float32; ``max_points``: a bound on the size of every mesh scored (it sets the grid, so no sync is needed).
    All tensors on one CUDA device.  Returns ``(add [M], adds [M])`` float32 CUDA tensors.  An object whose pose or
    points are not finite, or whose mesh index, offsets or size is out of range on the device, gets NaN (see
    include/ffb6d_b200.h); capturable in a CUDA graph."""
    pts = _tensor(mesh_pts, "mesh_pts", torch.float32, 2)
    dev = pts.device
    if pts.shape[1] != 3:
        raise ValueError("mesh_pts must be [P,3], got %s" % (tuple(pts.shape),))
    off = _tensor(mesh_off, "mesh_off", torch.int32, 1, dev)
    om = _tensor(obj_mesh, "obj_mesh", torch.int32, 1, dev)
    M = om.shape[0]
    pr = _tensor(pred_RT, "pred_RT", torch.float32, (M, 3, 4), dev)
    gt = _tensor(gt_RT, "gt_RT", torch.float32, (M, 3, 4), dev)
    if isinstance(max_points, bool) or not isinstance(max_points, (int, np.integer)):
        raise TypeError("max_points must be an int, got %r" % (max_points,))
    if not 1 <= max_points <= _lib.POSE_EVAL_MAX_POINTS:
        raise ValueError("max_points must lie in [1, %d], got %d" % (_lib.POSE_EVAL_MAX_POINTS, max_points))
    if M > _lib.POSE_EVAL_MAX_OBJECTS:
        raise ValueError("at most %d objects per call, got %d" % (_lib.POSE_EVAL_MAX_OBJECTS, M))
    if off.shape[0] < 2 and M > 0:
        raise ValueError("mesh_off must hold n_meshes + 1 >= 2 offsets, got %d" % off.shape[0])
    if pts.shape[0] > 2 ** 31 - 1:
        raise ValueError("mesh_pts has %d rows, more than int32 offsets address" % pts.shape[0])
    add = torch.empty(M, dtype=torch.float32, device=dev)
    adds = torch.empty(M, dtype=torch.float32, device=dev)
    if M == 0:
        return add, adds
    nbytes = int(lib.ffb6d_pose_add_adds_workspace_bytes(M, int(max_points)))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_pose_add_adds, dev, pts.data_ptr(), off.data_ptr(), off.shape[0] - 1, int(max_points),
           om.data_ptr(), pr.data_ptr(), gt.data_ptr(), M, add.data_ptr(), adds.data_ptr(), ws.data_ptr(), nbytes)
    return add, adds


def _u8(t, name, shape, dev):
    if torch.is_tensor(t) and t.dtype == torch.bool:
        t = t.view(torch.uint8)
    return _tensor(t, name, torch.uint8, shape, dev)


def _written(*ts):
    for t in ts:
        if not t.is_contiguous():
            raise ValueError("the record table's tensors are written in place and must be contiguous")


def eval_record(rows, state, cls_ids, present, pred_RT, add, adds, kps=None, gt_kps=None, valid=None, obj_id=0,
                poses=None, frame_poses=None, frame_flags=None):
    """One batch of a test run into the device record table (``ffb6d_eval_record``, see include/ffb6d_b200.h):
    slot ``(b, j)`` becomes row ``state[0] + b * n_obj + j``, and ``state`` advances on the device.

    :param rows: ``[capacity, EVAL_ROW_WORDS]`` int32; :param state: ``[4]`` int64 (rows used, frames, overflow)
    :param cls_ids: ``[B, n_obj]`` int32 class ids (YCB; LineMOD reads only the shape)
    :param present: ``[B, n_cls]`` bool / uint8 from the vote; :param pred_RT: the scored float32 poses, ``[B, n_obj,
      3, 4]`` (YCB) or ``[B, 3, 4]`` (LineMOD); :param add, adds: their float32 scores, ``[B * n_obj]`` or ``[B]``
    :param kps: ``[B, n_cls, n_kps + 1, 3]`` float32 vote keypoints, :param gt_kps: ``[B, n_obj, n_kps, 3]`` float32
      (YCB)
    :param valid: ``[B]`` bool, or None; :param obj_id: 0 for YCB, the LineMOD object's id otherwise
    :param poses: ``[B, n_cls, 3, 4]`` float64, with ``frame_poses [F, n_cls, 3, 4]`` float64 and ``frame_flags
      [F, n_cls]`` uint8: the optional frame table.
    No host synchronisation; capturable in a CUDA graph."""
    rw = _tensor(rows, "rows", torch.int32, 2)
    dev = rw.device
    if rw.shape[1] != _lib.EVAL_ROW_WORDS:
        raise ValueError("rows must be [capacity, %d], got %s" % (_lib.EVAL_ROW_WORDS, tuple(rw.shape)))
    st = _tensor(state, "state", torch.int64, (4,), dev)
    _written(rows, state)
    ids = _tensor(cls_ids, "cls_ids", torch.int32, 2, dev)
    B, n_obj = ids.shape
    pres = _u8(present, "present", 2, dev)
    n_cls = pres.shape[1]
    if pres.shape[0] != B:
        raise ValueError("present must be [B=%d, n_cls], got %s" % (B, tuple(pres.shape)))
    if isinstance(obj_id, bool) or not isinstance(obj_id, (int, np.integer)) or obj_id < 0:
        raise ValueError("obj_id must be an int >= 0, got %r" % (obj_id,))
    lm = obj_id > 0
    pr = _tensor(pred_RT, "pred_RT", torch.float32, (B, 3, 4) if lm else (B, n_obj, 3, 4), dev)
    a = _tensor(add, "add", torch.float32, (B if lm else B * n_obj,), dev)
    s = _tensor(adds, "adds", torch.float32, (B if lm else B * n_obj,), dev)
    k = g = None
    R = n_kps = 0
    if not lm:
        if kps is None or gt_kps is None:
            raise ValueError("a YCB record needs kps and gt_kps")
        k = _tensor(kps, "kps", torch.float32, 4, dev)
        g = _tensor(gt_kps, "gt_kps", torch.float32, 4, dev)
        R, n_kps = k.shape[2], g.shape[2]
        if tuple(k.shape) != (B, n_cls, R, 3) or tuple(g.shape) != (B, n_obj, n_kps, 3) or R != n_kps + 1:
            raise ValueError("kps must be [B,n_cls,n_kps+1,3] and gt_kps [B,n_obj,n_kps,3] = [%d,%d,n_kps,3], got %s "
                             "and %s" % (B, n_obj, tuple(k.shape), tuple(g.shape)))
    v = None if valid is None else _u8(valid, "valid", (B,), dev)
    fp = ff = ps = None
    F_cap = 0
    if frame_poses is not None or frame_flags is not None:
        ff = _u8(frame_flags, "frame_flags", 2, dev)
        F_cap = ff.shape[0]
        fp = _tensor(frame_poses, "frame_poses", torch.float64, (F_cap, n_cls, 3, 4), dev)
        ps = _tensor(poses, "poses", torch.float64, (B, n_cls, 3, 4), dev)
        _written(frame_poses, frame_flags)
        if ff.shape[1] != n_cls:
            raise ValueError("frame_flags must be [F, n_cls=%d], got %s" % (n_cls, tuple(ff.shape)))
    launch(lib.ffb6d_eval_record, dev, ptr(ids), ptr(v), pres.data_ptr(), ptr(k), ptr(ps), ptr(g), pr.data_ptr(),
           a.data_ptr(), s.data_ptr(), B, n_obj, n_cls, R, n_kps, int(obj_id), rw.data_ptr(), rw.shape[0],
           st.data_ptr(), ptr(fp), ptr(ff), F_cap)


def eval_auc(rows, state, n_cls, sym=None, lm_thr=0.0, ws=None):
    """The summary of a record table (``ffb6d_eval_auc``): ``(auc [3, n_cls], pct [2, n_cls], kp [2])`` float64
    CUDA tensors -- the ADD, ADD-S and ADD(-S) AUCs per class in percent (class 0 over every object), the
    percentages of ADD and ADD-S below ``lm_thr`` and the keypoint-error sum and count over the first ``state[0]``
    rows.  ``sym``: ``[n_cls]`` bool / uint8 CUDA (ADD-S for ADD(-S)), or None.  ``ws``: a workspace of at least
    :func:`eval_auc_workspace_bytes` bytes, or None to allocate one.  No host synchronisation."""
    rw = _tensor(rows, "rows", torch.int32, 2)
    dev = rw.device
    if rw.shape[1] != _lib.EVAL_ROW_WORDS:
        raise ValueError("rows must be [capacity, %d], got %s" % (_lib.EVAL_ROW_WORDS, tuple(rw.shape)))
    st = _tensor(state, "state", torch.int64, (4,), dev)
    n_cls = int(n_cls)
    sy = None if sym is None else _u8(sym, "sym", (n_cls,), dev)
    auc = torch.empty((3, n_cls), dtype=torch.float64, device=dev)
    pct = torch.empty((2, n_cls), dtype=torch.float64, device=dev)
    kp = torch.empty(2, dtype=torch.float64, device=dev)
    nbytes = eval_auc_workspace_bytes(rw.shape[0], n_cls)
    if ws is None:
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
    off = -ws.data_ptr() % 256
    launch(lib.ffb6d_eval_auc, dev, rw.data_ptr(), st.data_ptr(), rw.shape[0], n_cls, ptr(sy), float(lm_thr),
           auc.data_ptr(), pct.data_ptr(), kp.data_ptr(), ws.data_ptr() + off, ws.numel() - off)
    return auc, pct, kp


def eval_auc_workspace_bytes(capacity, n_cls):
    """Bytes :func:`eval_auc` needs for a table of ``capacity`` rows; raises ``ValueError`` outside the limits."""
    nbytes = int(lib.ffb6d_eval_auc_workspace_bytes(int(capacity), int(n_cls)))
    if nbytes == 0:
        raise ValueError("eval_auc: need 1 <= capacity <= %d and 1 <= n_cls <= %d, got %d and %d"
                         % (_lib.EVAL_MAX_ROWS, _lib.VOTE_MAX_CLASSES, capacity, n_cls))
    return nbytes


def _set_table(start, count, enable, dev):
    st = _tensor(start, "start", torch.int32, 1, dev)
    S = st.shape[0]
    ct = _tensor(count, "count", torch.int32, (S,), dev)
    en = None
    if enable is not None:
        en = _tensor(enable.to(torch.uint8) if torch.is_tensor(enable) and enable.dtype == torch.bool else enable,
                     "enable", torch.uint8, (S,), dev)
    if S > _lib.VIS_MAX_SETS:
        raise ValueError("at most %d sets per call, got %d" % (_lib.VIS_MAX_SETS, S))
    return st, ct, en, S


def _max_rows(max_rows):
    if isinstance(max_rows, bool) or not isinstance(max_rows, (int, np.integer)):
        raise TypeError("max_rows must be an int, got %r" % (max_rows,))
    if not 1 <= max_rows <= _lib.VIS_MAX_ROWS:
        raise ValueError("max_rows must lie in [1, %d], got %d" % (_lib.VIS_MAX_ROWS, max_rows))
    return int(max_rows)


def project_p3d(pts, start, count, max_rows, K, cam_scale=1.0, pose=None, enable=None):
    """``Basic_Utils.project_p3d`` (utils/basic_utils.py:268-277) of ``S`` point sets in one launch, bitwise numpy's
    float64 arithmetic (include/ffb6d_b200.h, DESIGN.md §4.26).

    :param pts: ``[n_rows,3]`` float32 or float64 CUDA, the point table; set ``s`` is rows ``start[s] ..
      start[s] + count[s]`` (``start``, ``count`` ``[S]`` int32), drawn where ``enable[s]`` (``[S]`` bool/uint8, or
      None for all).  A set whose rows leave the table or exceed ``max_rows`` is empty.
    :param K: float64 ``[3,3]`` (every set) or ``[S,3,3]``; ``cam_scale``: a float or a float64 tensor ``[1]``
      (``[S]`` with a per-set ``K``).  Without ``pose``, float32 points are scaled in float32 (numpy's casting of a
      Python float).
    :param pose: float64 ``[S,3,4]`` or None: the demo's ``np.dot(mesh, R.T) + t`` in float64 first.
    :return: int32 ``[S,max_rows,2]``, ``(INT32_MIN, INT32_MIN)`` at padding rows.  Capturable in a CUDA graph."""
    _need_cuda(pts, "pts")
    p, dev = pts, pts.device
    if p.dtype not in (torch.float32, torch.float64) or p.dim() != 2 or p.shape[1] != 3:
        raise ValueError("pts must be float32 or float64 [n,3], got %s %s" % (p.dtype, tuple(p.shape)))
    p = p.contiguous()
    if p.shape[0] > _lib.VIS_MAX_TABLE_ROWS:
        raise ValueError("pts has %d rows, more than int32 starts address" % p.shape[0])
    st, ct, en, S = _set_table(start, count, enable, dev)
    max_rows = _max_rows(max_rows)
    k = _tensor(K, "K", torch.float64, K.dim() if torch.is_tensor(K) else 2, dev)
    per_set = k.dim() == 3
    if tuple(k.shape) != ((S, 3, 3) if per_set else (3, 3)):
        raise ValueError("K must be float64 [3,3] or [S,3,3] = [%d,3,3], got %s" % (S, tuple(k.shape)))
    if not torch.is_tensor(cam_scale):
        cam_scale = torch.full((S if per_set else 1,), float(cam_scale), dtype=torch.float64, device=dev)
    cs = _tensor(cam_scale, "cam_scale", torch.float64, (S if per_set else 1,), dev)
    ps = None if pose is None else _tensor(pose, "pose", torch.float64, (S, 3, 4), dev)
    out = torch.empty((S, max_rows, 2), dtype=torch.int32, device=dev)
    if S == 0:
        return out
    launch(lib.ffb6d_project_p3d, dev, p.data_ptr(), int(p.dtype == torch.float64), p.shape[0], st.data_ptr(),
           ct.data_ptr(), ptr(en), S, max_rows, ptr(ps), k.data_ptr(), cs.data_ptr(), int(per_set), out.data_ptr())
    return out


def draw_p2ds_workspace(img):
    """The scratch :func:`draw_p2ds` needs for ``img [B,H,W,3]``: ``B H W`` 8-byte keys (19.7 MB at 8 x 480 x 640).
    Pass it to every call on images of that size to keep them free of allocations."""
    B, H, W = (int(v) for v in img.shape[:3])
    return workspace(lib.ffb6d_draw_p2ds_workspace_bytes(B, H, W), img.device)


def draw_p2ds(img, p2ds, frame, start, count, n_rows, radius, colors, enable=None, ws=None):
    """``Basic_Utils.draw_p2ds`` (utils/basic_utils.py:283-295) of ``S`` sets in one call, in place: ``img [B,H,W,3]``
    uint8 CUDA gets, for every row ``r < count[s]`` of every enabled set ``s``, the filled ``cv2.circle`` of radius
    ``radius[s]`` at ``p2ds[s, r]`` clipped to ``[0,W] x [0,H]``, in frame ``frame[s]``; where circles overlap the last
    in (set, row) order wins.

    :param p2ds: int32 ``[S,max_rows,2]`` (what :func:`project_p3d` returns); ``frame``, ``radius`` ``[S]`` int32;
      ``start``, ``count``, ``enable`` and ``n_rows`` the set table of :func:`project_p3d` (a set that is empty there
      draws nothing); a frame out of ``[0,B)`` or a radius out of ``[0, 64]`` draws nothing.
    :param colors: uint8 ``[S,3]`` (one colour per set) or ``[S,max_rows,3]`` (one per row).
    :param ws: a :func:`draw_p2ds_workspace` of ``img``, or None to allocate one.
    :return: ``img``.  No host synchronisation: capturable in a CUDA graph."""
    im = _tensor(img, "img", torch.uint8, 4)
    if im.data_ptr() != img.data_ptr():
        raise ValueError("img must be contiguous: it is drawn in place")
    dev = im.device
    B, H, W, c3 = im.shape
    if c3 != 3:
        raise ValueError("img must be [B,H,W,3], got %s" % (tuple(im.shape),))
    if not (1 <= H <= _lib.VIS_MAX_SIDE and 1 <= W <= _lib.VIS_MAX_SIDE) or B > _lib.VIS_MAX_FRAMES:
        raise ValueError("img of %s: at most %d frames of 1 .. %d pixels a side" % (
            tuple(im.shape), _lib.VIS_MAX_FRAMES, _lib.VIS_MAX_SIDE))
    st, ct, en, S = _set_table(start, count, enable, dev)
    pt = _tensor(p2ds, "p2ds", torch.int32, 3, dev)
    max_rows = _max_rows(pt.shape[1])
    if tuple(pt.shape) != (S, max_rows, 2):
        raise ValueError("p2ds must be [S,max_rows,2] with S = %d, got %s" % (S, tuple(pt.shape)))
    fr = _tensor(frame, "frame", torch.int32, (S,), dev)
    rd = _tensor(radius, "radius", torch.int32, (S,), dev)
    col = _tensor(colors, "colors", torch.uint8, colors.dim() if torch.is_tensor(colors) else 2, dev)
    per_row = col.dim() == 3
    if tuple(col.shape) != ((S, max_rows, 3) if per_row else (S, 3)):
        raise ValueError("colors must be uint8 [S,3] or [S,max_rows,3], got %s" % (tuple(col.shape),))
    if not 0 <= int(n_rows) <= _lib.VIS_MAX_TABLE_ROWS:
        raise ValueError("n_rows must lie in [0, %d], got %d" % (_lib.VIS_MAX_TABLE_ROWS, int(n_rows)))
    nbytes = int(lib.ffb6d_draw_p2ds_workspace_bytes(B, H, W))
    if ws is None:
        ws = workspace(nbytes, dev)
    elif ws.device != dev or ws.numel() * ws.element_size() < nbytes:
        raise ValueError("ws holds %d bytes on %s, %d needed on %s" % (ws.numel() * ws.element_size(), ws.device,
                                                                      nbytes, dev))
    if B == 0 or S == 0:
        return img
    launch(lib.ffb6d_draw_p2ds, dev, im.data_ptr(), B, H, W, pt.data_ptr(), S, max_rows, fr.data_ptr(), st.data_ptr(),
           ct.data_ptr(), ptr(en), int(n_rows), rd.data_ptr(), col.data_ptr(), int(per_row), ws.data_ptr(),
           ws.numel() * ws.element_size())
    return img


def mean_shift_fit(votes, valid=None, bandwidth=0.05, max_iter=300, return_modes=False):
    """Gaussian mean shift of ``G`` independent vote sets in one persistent kernel: the batched form of
    ``MeanShiftTorch.fit`` (utils/meanshift_pytorch.py:33-57).

    :param votes: ``[G,N,3]`` float32 CUDA.
    :param valid: bool/uint8 mask of the points that vote, ``[N]`` (shared) or ``[G,N]``; ``None`` = all.
    :return: ``(centres [G,3] f32, labels [G,N] bool, iters [G] int32)`` and, with ``return_modes``, the converged
      position of every point ``[G,N,3]`` (the reference's ``ret_mid_res``)."""
    _need_cuda(votes, "votes")
    if votes.dim() != 3 or votes.shape[2] != 3 or votes.dtype != torch.float32:
        raise ValueError("votes must be float32 [G,N,3]")
    votes = votes.contiguous()
    G, N, _ = votes.shape
    dev = votes.device
    stride = 0
    vptr = None
    if valid is not None:
        _need_cuda(valid, "valid")
        if valid.dtype == torch.bool:
            valid = valid.to(torch.uint8)
        if valid.dtype != torch.uint8:
            raise ValueError("valid must be bool or uint8")
        valid = valid.contiguous()
        if tuple(valid.shape) == (N,):
            stride = 0
        elif tuple(valid.shape) == (G, N):
            stride = N
        else:
            raise ValueError("valid must be [N] or [G,N]")
        vptr = valid.data_ptr()
    centres = torch.empty((G, 3), dtype=torch.float32, device=dev)
    labels = torch.empty((G, N), dtype=torch.uint8, device=dev)
    iters = torch.empty((G,), dtype=torch.int32, device=dev)
    modes = torch.empty((G, N, 3), dtype=torch.float32, device=dev) if return_modes else None
    nbytes = int(lib.ffb6d_mean_shift_workspace_bytes(G, N))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_mean_shift_fit, dev, votes.data_ptr(), vptr, stride, G, N, float(bandwidth), int(max_iter),
           centres.data_ptr(), labels.data_ptr(), iters.data_ptr(), ptr(modes), ws.data_ptr(), nbytes)
    out = (centres, labels.bool(), iters)
    return out + (modes,) if return_modes else out


def vote_poses(pcld, mask, ctr_of, kp_of, mesh_kps, has_mesh, refine_thr=None, use_ctr=True, ctr_filter=True,
               bandwidth=0.04, max_iter=300):
    """The poses of every object of ``B`` frames in one call (``ffb6d_vote_poses``): the batched form of
    ``cal_frame_poses`` (utils/pvn3d_eval_utils_kpls.py:65-160), every vote set of a stage in one mean-shift launch.

    :param pcld: ``[B,N,3]`` float32 CUDA; ``mask`` ``[B,N]`` int64 predicted class ids in ``[0, n_cls)``;
      ``ctr_of`` ``[B,1,N,3]``, ``kp_of`` ``[B,n_kps,N,3]`` float32.
    :param mesh_kps: ``[n_cls,R,3]`` float32 object-frame keypoints, ``R = n_kps + use_ctr`` (centre last);
      ``has_mesh`` ``[n_cls]`` bool/uint8: the classes whose row is filled.
    :param refine_thr: ``[n_cls]`` float32 distances of the centre-clustering refinement, or None for none.
    :return: ``(present [B,n_cls] bool, count [B,n_cls] int32, kps [B,n_cls,R,3] float32, poses [B,n_cls,3,4]
      float64)`` CUDA tensors (see include/ffb6d_b200.h for the rows without a fit and the NaN rows).  No host
      synchronisation: capturable in a CUDA graph."""
    p = _tensor(pcld, "pcld", torch.float32, 3)
    dev = p.device
    B, N, _ = p.shape
    if p.shape[2] != 3:
        raise ValueError("pcld must be [B,N,3], got %s" % (tuple(p.shape),))
    m = _tensor(mask, "mask", torch.int64, (B, N), dev)
    c = _tensor(ctr_of, "ctr_of", torch.float32, (B, 1, N, 3), dev)
    k = _tensor(kp_of, "kp_of", torch.float32, 4, dev)
    n_kps = k.shape[1]
    if tuple(k.shape) != (B, n_kps, N, 3):
        raise ValueError("kp_of must be [B,n_kps,N,3] = [%d,n_kps,%d,3], got %s" % (B, N, tuple(k.shape)))
    mk = _tensor(mesh_kps, "mesh_kps", torch.float32, 3, dev)
    n_cls, R = mk.shape[0], n_kps + int(bool(use_ctr))
    if tuple(mk.shape) != (n_cls, R, 3):
        raise ValueError("mesh_kps must be [n_cls,%d,3], got %s" % (R, tuple(mk.shape)))
    hm = _tensor(has_mesh.to(torch.uint8) if torch.is_tensor(has_mesh) and has_mesh.dtype == torch.bool else has_mesh,
                 "has_mesh", torch.uint8, (n_cls,), dev)
    thr = None if refine_thr is None else _tensor(refine_thr, "refine_thr", torch.float32, (n_cls,), dev)
    present = torch.empty((B, n_cls), dtype=torch.uint8, device=dev)
    count = torch.empty((B, n_cls), dtype=torch.int32, device=dev)
    kps = torch.empty((B, n_cls, R, 3), dtype=torch.float32, device=dev)
    poses = torch.empty((B, n_cls, 3, 4), dtype=torch.float64, device=dev)
    nbytes = int(lib.ffb6d_vote_poses_workspace_bytes(B, N, n_cls, n_kps))
    ws = workspace(nbytes, dev)
    launch(lib.ffb6d_vote_poses, dev, p.data_ptr(), m.data_ptr(), c.data_ptr(), k.data_ptr(), mk.data_ptr(),
           hm.data_ptr(), ptr(thr), B, N, n_cls, n_kps, int(bool(use_ctr)), int(bool(ctr_filter)), float(bandwidth),
           int(max_iter), present.data_ptr(), count.data_ptr(), kps.data_ptr(), poses.data_ptr(), ws.data_ptr(),
           nbytes)
    return present.bool(), count, kps, poses


def best_fit_transform(A, B):
    """Least-squares rigid transform of point sets ``A -> B`` (pvn3d_eval_utils_kpls.py:28-59), batched.

    :param A, B: ``[G,M,3]`` (or ``[M,3]``) float32 CUDA; :return: ``[G,3,4]`` (or ``[3,4]``) float64 ``[R|t]``."""
    _need_cuda(A, "A")
    _need_cuda(B, "B")
    single = A.dim() == 2
    if single:
        A, B = A[None], B[None]
    if A.shape != B.shape or A.dim() != 3 or A.shape[2] != 3:
        raise ValueError("A and B must both be [G,M,3]")
    A = A.to(torch.float32).contiguous()
    B = B.to(torch.float32).contiguous()
    G, M, _ = A.shape
    T = torch.empty((G, 3, 4), dtype=torch.float64, device=A.device)
    launch(lib.ffb6d_best_fit_transform, A.device, A.data_ptr(), B.data_ptr(), G, M, T.data_ptr())
    return T[0] if single else T


def rgb_add_noise(rgb, plan, seed, noise=None, plan_dev=None):
    """The datasets' ``rgb_add_noise`` (datasets/ycb/ycb_dataset.py:107-143, linemod_dataset.py:142-164) for a batch
    on the GPU (``ffb6d_rgb_add_noise``).

    :param rgb: ``[B,H,W,3]`` uint8 CUDA, H, W >= 32 (the channel roles are the reference's: it feeds RGB data to
      ``COLOR_BGR2HSV``)
    :param plan: ``[B, REC_LEN]`` float64 numpy records of :func:`ffb6d_b200.augment.draw_rgb_noise`
    :param seed: key of the per-pixel normal draws (frame b of the batch, the record's pass); use one seed per batch.
      An int, or a one-element int64 / uint64 CUDA tensor read on the device (the same draws as the int of the same
      64 bits)
    :param noise: optional ``[2,B,H,W,3]`` float64 CUDA normals to use instead of the generator's (the first for
      ``gaussian_noise``, the second for YCB's ``normal(0, 7)``), e.g. to replay numpy's stream
    :param plan_dev: optional ``[B, REC_LEN]`` float64 CUDA copy of ``plan`` for the kernels to read (``plan`` is
      still what is checked); without it ``plan`` is copied to the device
    :return: ``[B,H,W,3]`` uint8
    """
    from . import augment as A
    _need_cuda(rgb, "rgb")
    if rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3:
        raise ValueError("rgb must be uint8 [B,H,W,3], got %s %s" % (rgb.dtype, tuple(rgb.shape)))
    B, H, W, _ = rgb.shape
    plan = np.ascontiguousarray(plan, dtype=np.float64)
    if plan.shape != (B, A.REC_LEN):
        raise ValueError("plan must be float64 [B, %d] = [%d, %d], got %s" % (A.REC_LEN, B, A.REC_LEN, plan.shape))
    dev = rgb.device
    seed_d = _device_seed(seed, dev)
    if seed_d is None and not (0 <= int(seed) < 1 << 64):
        raise ValueError("seed must fit 64 bits, got %r" % (seed,))
    if noise is not None:
        noise = _tensor(noise, "noise", torch.float64, (2, B, H, W, 3), dev)
    src = rgb.contiguous()
    if plan_dev is None:
        plan_d = torch.from_numpy(plan).to(dev)
    else:
        plan_d = _tensor(plan_dev, "plan_dev", torch.float64, (B, A.REC_LEN), dev)
    out = torch.empty_like(src)
    work = torch.empty_like(src)
    if seed_d is None:
        launch(lib.ffb6d_rgb_add_noise, dev, src.data_ptr(), B, H, W, plan.ctypes.data, plan_d.data_ptr(), int(seed),
               ptr(noise), out.data_ptr(), work.data_ptr())
    else:
        launch(lib.ffb6d_rgb_add_noise_dseed, dev, src.data_ptr(), B, H, W, plan.ctypes.data, plan_d.data_ptr(),
               seed_d.data_ptr(), ptr(noise), out.data_ptr(), work.data_ptr())
    return out


def rgb_noise_check_records(plan):
    """Check ``[B, REC_LEN]`` float64 host records as :func:`rgb_add_noise` checks them, without a launch
    (``ffb6d_rgb_noise_check_records``): raises :class:`~ffb6d_b200._lib.FFB6DError` with its message for a bad
    record."""
    from . import augment as A
    plan = np.ascontiguousarray(plan, dtype=np.float64)
    if plan.ndim != 2 or plan.shape[1] != A.REC_LEN:
        raise ValueError("plan must be float64 [B, %d], got %s" % (A.REC_LEN, plan.shape))
    check(lib.ffb6d_rgb_noise_check_records(plan.ctypes.data, plan.shape[0]))


def add_real_back(rgb, labels, dpt, back_rgb, back_labels, back_dpt, apply_rgb=None, dataset="ycb", active=None):
    """The datasets' ``add_real_back`` (datasets/ycb/ycb_dataset.py:145-163, linemod_dataset.py:166-186) for a batch
    on the GPU (``ffb6d_add_real_back``), after the worker has loaded the background frames.

    :param rgb: ``[B,H,W,3]`` uint8; :param labels: ``[B,H,W]`` uint8 (the frame's labels; 0 is background)
    :param dpt: ``[B,H,W]`` uint16 raw depth (YCB ``dpt_um``; LineMOD ``dpt_mm.astype(np.uint16)``)
    :param back_rgb: ``[B,H,W,3]`` uint8; :param back_labels: ``[B,H,W]`` or ``[B,H,W,3]`` uint8 (the background
      frame's label image, YCB, or mask, LineMOD); :param back_dpt: ``[B,H,W]`` uint16
    :param apply_rgb: LineMOD: per-frame bools, the ``rand() < 0.6`` draw (YCB always composes the colour image)
    :param dataset: ``'ycb'`` or ``'linemod'``; :param active: per-frame bools, frames that go through
      ``add_real_back`` at all (default: every frame); the others pass through unchanged.  When ``active`` and
      ``apply_rgb`` are both ``[B]`` CUDA tensors, the flags are combined on the device (no host copy)
    :return: ``(rgb [B,H,W,3] uint8, dpt [B,H,W] uint16)``; the composed depth is uint16 and feeds
      :func:`fill_missing` as it is
    """
    if dataset not in ("ycb", "linemod"):
        raise ValueError("dataset must be 'ycb' or 'linemod', got %r" % (dataset,))
    _need_cuda(rgb, "rgb")
    if rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3:
        raise ValueError("rgb must be uint8 [B,H,W,3], got %s %s" % (rgb.dtype, tuple(rgb.shape)))
    B, H, W, _ = rgb.shape
    dev = rgb.device
    labels = _tensor(labels, "labels", torch.uint8, (B, H, W), dev)
    dpt = _tensor(dpt, "dpt", torch.uint16, (B, H, W), dev)
    back_rgb = _tensor(back_rgb, "back_rgb", torch.uint8, (B, H, W, 3), dev)
    _need_cuda(back_labels, "back_labels")
    if back_labels.dim() == 3:
        back_labels = back_labels[..., None]
    ch = back_labels.shape[-1] if back_labels.dim() == 4 else 0
    back_labels = _tensor(back_labels, "back_labels", torch.uint8, (B, H, W, ch if ch in (1, 3) else -1), dev)
    back_dpt = _tensor(back_dpt, "back_dpt", torch.uint16, (B, H, W), dev)
    flags = (active, apply_rgb)
    if all(isinstance(f, torch.Tensor) and f.is_cuda for f in flags):      # combined on the device: capturable
        if any(tuple(f.shape) != (B,) or f.device != dev for f in flags):
            raise ValueError("apply_rgb and active must have one entry per frame (%d) on %s" % (B, dev))
        act, col = (f.to(torch.uint8) for f in flags)
        mode = act * (1 + 2 * col)
    else:
        act = np.ones(B, bool) if active is None else np.asarray(active, bool).reshape(-1)
        if dataset == "ycb":
            col = np.ones(B, bool) if apply_rgb is None else np.asarray(apply_rgb, bool).reshape(-1)
        else:
            if apply_rgb is None:
                raise ValueError("LineMOD needs apply_rgb (the frame's rand() < 0.6 draw)")
            col = np.asarray(apply_rgb, bool).reshape(-1)
        if act.shape != (B,) or col.shape != (B,):
            raise ValueError("apply_rgb and active must have one entry per frame (%d)" % B)
        mode = torch.from_numpy((act * (1 + 2 * col)).astype(np.uint8)).to(dev)
    src = rgb.contiguous()
    rgb_out = torch.empty_like(src)
    dpt_out = torch.empty_like(dpt)
    launch(lib.ffb6d_add_real_back, dev, src.data_ptr(), labels.data_ptr(), dpt.data_ptr(), back_rgb.data_ptr(),
           back_labels.data_ptr(), ch, back_dpt.data_ptr(), mode.data_ptr(), 0 if dataset == "ycb" else 1, B, H, W,
           rgb_out.data_ptr(), dpt_out.data_ptr())
    return rgb_out, dpt_out


def color_jitter(rgb, plan, active=None, plan_dev=None):
    """The datasets' ``trancolor`` (torchvision ``ColorJitter(0.2, 0.2, 0.2, 0.05)`` on the PIL image,
    datasets/ycb/ycb_dataset.py:190-193, linemod_dataset.py:220-223) for a batch on the GPU
    (``ffb6d_color_jitter``); bitwise what torchvision 0.26 with Pillow 12.2 computes.

    :param rgb: ``[B,H,W,3]`` uint8 CUDA
    :param plan: ``[B, JITTER_PLAN_LEN]`` float64 plans of :func:`ffb6d_b200.augment.draw_color_jitter`; every
      frame's plan is validated, an inactive frame's too
    :param active: per-frame bools (a sequence, or a tensor), frames to jitter (default: every frame); the others,
      e.g. frames the dataset does not jitter, pass through unchanged
    :param plan_dev: optional ``[B, JITTER_PLAN_LEN]`` float64 CUDA copy of ``plan`` for the kernels to read (``plan``
      is still what is checked); without it ``plan`` is copied to the device
    :return: ``[B,H,W,3]`` uint8
    """
    from . import augment as A
    _need_cuda(rgb, "rgb")
    if rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3:
        raise ValueError("rgb must be uint8 [B,H,W,3], got %s %s" % (rgb.dtype, tuple(rgb.shape)))
    B, H, W, _ = rgb.shape
    plan = np.ascontiguousarray(plan, dtype=np.float64)
    if plan.shape != (B, A.JITTER_PLAN_LEN):
        raise ValueError("plan must be float64 [B, %d] = [%d, %d], got %s"
                         % (A.JITTER_PLAN_LEN, B, A.JITTER_PLAN_LEN, plan.shape))
    dev = rgb.device
    if active is None:
        act = torch.ones(B, dtype=torch.uint8, device=dev)
    else:
        act = active if isinstance(active, torch.Tensor) else torch.from_numpy(np.asarray(active, bool))
        if tuple(act.shape) != (B,):
            raise ValueError("active must have one entry per frame (%d), got %s" % (B, tuple(act.shape)))
        act = act.to(device=dev, dtype=torch.uint8).contiguous()
    src = rgb.contiguous()
    out = torch.empty_like(src)
    if B * H * W == 0:
        return out
    if plan_dev is None:
        plan_d = torch.from_numpy(plan).to(dev)
    else:
        plan_d = _tensor(plan_dev, "plan_dev", torch.float64, (B, A.JITTER_PLAN_LEN), dev)
    work = torch.empty(B, dtype=torch.int64, device=dev)
    launch(lib.ffb6d_color_jitter, dev, src.data_ptr(), B, H, W, plan.ctypes.data, plan_d.data_ptr(), act.data_ptr(),
           out.data_ptr(), work.data_ptr())
    return out


def color_jitter_check_plans(plan):
    """Check ``[B, JITTER_PLAN_LEN]`` float64 host plans as :func:`color_jitter` checks them, without a launch
    (``ffb6d_color_jitter_check_plans``): raises :class:`~ffb6d_b200._lib.FFB6DError` with its message for a bad
    plan."""
    from . import augment as A
    plan = np.ascontiguousarray(plan, dtype=np.float64)
    if plan.ndim != 2 or plan.shape[1] != A.JITTER_PLAN_LEN:
        raise ValueError("plan must be float64 [B, %d], got %s" % (A.JITTER_PLAN_LEN, plan.shape))
    check(lib.ffb6d_color_jitter_check_plans(plan.ctypes.data, plan.shape[0]))


def aug_noise_field(seed, B, H, W, stage, device="cuda"):
    """The ``[B,H,W,3]`` float64 normals that :func:`rgb_add_noise` draws for ``(seed, frame, stage)``; stage
    ``2*pass`` is ``gaussian_noise``'s, ``2*pass + 1`` YCB's ``normal(0, 7)``'s (``ffb6d_aug_noise_field``)."""
    out = torch.empty((B, H, W, 3), dtype=torch.float64, device=device)
    _need_cuda(out, "out")
    launch(lib.ffb6d_aug_noise_field, out.device, int(seed), B, H, W, int(stage), out.data_ptr())
    return out


# --------------------------------------------------------------------------- training loss
def _loss_labels(labels, B, N, dev):
    _need_cuda(labels, "labels")
    lab, i64 = _idx_arg(labels, "labels")
    if lab.numel() != B * N or lab.device != dev:
        raise ValueError("labels must hold %d x %d values on %s, got %s on %s"
                         % (B, N, dev, tuple(labels.shape), labels.device))
    return lab.view(B, N), i64


def _loss_valid(valid, B, dev):
    """``valid`` as the kernels read it: None, or ``[B]`` uint8 on ``dev`` (a bool / integer tensor is converted on
    the device, without a host synchronisation)."""
    if valid is None:
        return None
    v = valid if isinstance(valid, torch.Tensor) else torch.as_tensor(np.asarray(valid, bool))
    if v.numel() != B:
        raise ValueError("valid must have one entry per frame (%d), got %s" % (B, tuple(v.shape)))
    return v.reshape(B).to(device=dev, dtype=torch.uint8).contiguous()


def _loss_workspace(B, N, n_kps, dev):
    nbytes = lib.ffb6d_loss_workspace_bytes(B, N, n_kps)
    if nbytes == 0:
        raise ValueError("loss: unsupported size B=%d N=%d n_kps=%d" % (B, N, n_kps))
    return workspace(nbytes, dev), nbytes


def focal_loss_fwd(logits, labels, valid=None, gamma=0.0, alpha=None, size_average=True, layout=0):
    """FocalLoss forward (models/loss.py:12-43) on ``logits [B,C,N]`` (``layout=0``) or ``[B,N,C]`` (``layout=1``)
    float32 CUDA, ``labels [B,N]`` int32 / int64, ``valid [B]`` or None, ``alpha [C]`` float32 CUDA or None
    (``ffb6d_focal_loss_fwd``, one call).  :return: ``(loss [], acc [], count [] int64, lse [B,N])``"""
    _need_cuda(logits, "logits")
    if logits.dim() != 3 or logits.dtype != torch.float32 or layout not in (0, 1):
        raise ValueError("logits must be float32 [B,C,N] (layout 0) or [B,N,C] (layout 1), got %s %s"
                         % (logits.dtype, tuple(logits.shape)))
    x = logits.contiguous()
    B, C, N = (x.shape[0], x.shape[2], x.shape[1]) if layout else x.shape
    dev = x.device
    lab, is64 = _loss_labels(labels, B, N, dev)
    v = _loss_valid(valid, B, dev)
    if alpha is not None:
        alpha = _tensor(alpha, "alpha", shape=1, device=dev)
        if alpha.numel() < C:
            raise ValueError("alpha must be a [>= C] float32 tensor on %s" % dev)
    ws, nbytes = _loss_workspace(B, N, 1, dev)
    out = torch.empty(2, dtype=torch.float32, device=dev)
    count = torch.empty((), dtype=torch.int64, device=dev)
    lse = torch.empty((B, N), dtype=torch.float32, device=dev)
    launch(lib.ffb6d_focal_loss_fwd, dev, x.data_ptr(), layout, lab.data_ptr(), is64, ptr(v), B, C, N, float(gamma),
           ptr(alpha), int(bool(size_average)), out.data_ptr(), out.data_ptr() + 4, count.data_ptr(), lse.data_ptr(),
           ws.data_ptr(), nbytes)
    return out[0], out[1], count, lse


def focal_loss_bwd(logits, labels, valid, gamma, alpha, size_average, lse, count, grad_loss, layout=0):
    """FocalLoss backward (``ffb6d_focal_loss_bwd``, one launch): the gradient of the logits, in their layout, from
    the forward's ``lse`` and ``count`` and the upstream gradient ``grad_loss`` (a one-element CUDA tensor)."""
    x = logits.contiguous()
    B, C, N = (x.shape[0], x.shape[2], x.shape[1]) if layout else x.shape
    dev = x.device
    lab, is64 = _loss_labels(labels, B, N, dev)
    v = _loss_valid(valid, B, dev)
    lse = _tensor(lse, "lse", shape=(B, N))
    g = grad_loss.to(torch.float32).reshape(1).contiguous()
    grad = torch.empty_like(x)
    launch(lib.ffb6d_focal_loss_bwd, dev, x.data_ptr(), layout, lab.data_ptr(), is64, ptr(v), B, C, N, float(gamma),
           ptr(alpha), int(bool(size_average)), lse.data_ptr(), count.data_ptr(), g.data_ptr(), grad.data_ptr())
    return grad


def _of_args(pred, targ, labels, valid):
    _need_cuda(pred, "pred_ofsts")
    if pred.dim() != 4 or pred.shape[3] != 3 or pred.dtype != torch.float32:
        raise ValueError("pred_ofsts must be float32 [B,n_kps,N,3], got %s %s" % (pred.dtype, tuple(pred.shape)))
    B, K, N, _ = pred.shape
    _need_cuda(targ, "kp_targ_ofst")
    if targ.numel() != B * N * K * 3 or targ.dtype != torch.float32 or targ.device != pred.device:
        raise ValueError("kp_targ_ofst must be float32 [B,N,n_kps,3] = [%d,%d,%d,3] on %s, got %s %s"
                         % (B, N, K, pred.device, targ.dtype, tuple(targ.shape)))
    lab, is64 = _loss_labels(labels, B, N, pred.device)
    return pred.contiguous(), targ.reshape(B, N, K, 3).contiguous(), lab, is64, _loss_valid(valid, B, pred.device)


def of_l1_loss_fwd(pred, targ, labels, valid=None):
    """of_l1_loss forward with ``normalize=True`` (models/loss.py:46-74; ``ffb6d_of_l1_loss_fwd``, one call):
    ``pred [B,n_kps,N,3]``, ``targ [B,N,n_kps,3]`` float32 CUDA.  :return: ``(loss [B,n_kps], count [B])``"""
    p, t, lab, is64, v = _of_args(pred, targ, labels, valid)
    B, K, N, _ = p.shape
    dev = p.device
    ws, nbytes = _loss_workspace(B, N, K, dev)
    out = torch.empty((B, K), dtype=torch.float32, device=dev)
    count = torch.empty(B, dtype=torch.float32, device=dev)
    launch(lib.ffb6d_of_l1_loss_fwd, dev, p.data_ptr(), t.data_ptr(), lab.data_ptr(), is64, ptr(v), B, K, N,
           out.data_ptr(), count.data_ptr(), ws.data_ptr(), nbytes)
    return out, count


def of_l1_loss_bwd(pred, targ, labels, valid, count, grad_out):
    """of_l1_loss backward (``ffb6d_of_l1_loss_bwd``, one launch): the gradient of ``pred`` for an upstream
    ``grad_out [B,n_kps]``, from the forward's ``count``."""
    p, t, lab, is64, v = _of_args(pred, targ, labels, valid)
    B, K, N, _ = p.shape
    dev = p.device
    count = _tensor(count, "count", shape=(B,))
    g = _tensor(grad_out.to(torch.float32), "grad_out", shape=(B, K))
    grad = torch.empty_like(p)
    launch(lib.ffb6d_of_l1_loss_bwd, dev, p.data_ptr(), t.data_ptr(), lab.data_ptr(), is64, ptr(v), B, K, N,
           count.data_ptr(), g.data_ptr(), grad.data_ptr())
    return grad


# --------------------------------------------------------------------------- PSP head of the image branch (eval)
PSP_SIZES = (1, 2, 3, 6)
_PSP_BINS = sum(s * s for s in PSP_SIZES)     # 50


def psp_pool(x):
    """``[AdaptiveAvgPool2d(s)(x) for s in (1, 2, 3, 6)]`` (the priors of PSPModule, models/cnn/pspnet.py:19-28) in
    one read of ``x [B,C,H,W]`` float32 CUDA (``ffb6d_psp_pool``).  :return: four ``[B,C,s,s]`` tensors, views of one
    buffer in the block order :func:`psp_bottleneck` reads."""
    xc = _tensor(x, "x", shape=4)
    B, C, H, W = xc.shape
    out = torch.empty(_PSP_BINS * B * C, dtype=torch.float32, device=xc.device)
    launch(lib.ffb6d_psp_pool, xc.device, xc.data_ptr(), B, C, H, W, out.data_ptr())
    views, off = [], 0
    for s in PSP_SIZES:
        views.append(out[off:off + B * C * s * s].view(B, C, s, s))
        off += B * C * s * s
    return views


class PSPWeights:
    """PSPModule's weights packed for :func:`psp_bottleneck`: with the bottleneck weight split by input block,
    ``W = [W_1|W_2|W_3|W_6|W_f]``, the stage convs ``C_s`` are folded into ``M_s = W_s C_s`` (computed in fp64, then
    packed), and ``W_f`` is packed as it is.  Build it once per weight version (inference)."""

    def __init__(self, stage_weights, weight, bias):
        _need_cuda(weight, "weight")
        w = weight.detach().reshape(weight.shape[0], -1)
        C = stage_weights[0].shape[0]
        if len(stage_weights) != len(PSP_SIZES) or w.shape[1] != (len(PSP_SIZES) + 1) * C:
            raise ValueError("PSPWeights: %d stage convs [C, C] and a [Co, %d C] bottleneck expected"
                             % (len(PSP_SIZES), len(PSP_SIZES) + 1))
        self.C, self.Co = int(C), int(w.shape[0])
        self.stages = [PackedWeight((w[:, i * C:(i + 1) * C].double() @ cs.detach().reshape(C, C).double()).float())
                       for i, cs in enumerate(stage_weights)]
        self.feat = PackedWeight(w[:, len(PSP_SIZES) * C:])
        self.bias = bias.detach().float().contiguous()
        self.one = torch.ones(self.Co, dtype=torch.float32, device=w.device)
        self.zero = torch.zeros(self.Co, dtype=torch.float32, device=w.device)
        self.device = w.device


def psp_pack(stage_weights, weight, bias):
    """:class:`PSPWeights` from the four stage convs' weights ``[C,C,1,1]``, the bottleneck's weight
    ``[Co,5C,1,1]`` and its bias ``[Co]``."""
    return PSPWeights(stage_weights, weight, bias)


def psp_bottleneck(x, pooled, weights):
    """``relu(bottleneck(cat(up_1(C_1 p_1), .., up_6(C_6 p_6), x)))`` of PSPModule (models/cnn/pspnet.py:24-31) without
    the upsampled priors or the concat: ``relu(W_f x + b + sum_s up_s(T_s))``, ``T_s = M_s p_s``.  The four ``T_s``
    are packed GEMMs on the 50 pooled columns (``ffb6d_fusion_mlp_fwd_ex``, channels-last into one table), the rest
    is ``ffb6d_psp_bottleneck_fwd``.  :param x: ``[B,C,H,W]`` float32 CUDA; :param pooled: :func:`psp_pool` of ``x``;
    :param weights: :class:`PSPWeights`.  :return: ``[B,Co,H,W]``"""
    xc = _tensor(x, "x", shape=4)
    B, C, H, W = xc.shape
    if C != weights.C or weights.device != xc.device:
        raise ValueError("psp weights take %d channels on %s, x has %d on %s" % (weights.C, weights.device, C, xc.device))
    Co = weights.Co
    table = torch.empty(_PSP_BINS * B * Co, dtype=torch.float32, device=xc.device)
    out = torch.empty((B, Co, H, W), dtype=torch.float32, device=xc.device)
    off = 0
    for s, p, pk in zip(PSP_SIZES, pooled, weights.stages):
        if tuple(p.shape) != (B, C, s, s) or not p.is_contiguous() or p.dtype != torch.float32:
            raise ValueError("pooled must be psp_pool(x)")
        launch(lib.ffb6d_fusion_mlp_fwd_ex, xc.device, p.data_ptr(), C, None, 0, pk.data.data_ptr(),
               weights.one.data_ptr(), weights.zero.data_ptr(), B, Co, s * s, 0, 0.0, None, None, 0, 0, LAYOUT_NSC,
               table.data_ptr() + 4 * off * Co)
        off += B * s * s
    launch(lib.ffb6d_psp_bottleneck_fwd, xc.device, xc.data_ptr(), B, C, H, W, weights.feat.data.data_ptr(),
           weights.bias.data_ptr(), Co, table.data_ptr(), out.data_ptr())
    return out


def conv1x1_log_softmax(x, weight, bias):
    """``log_softmax(conv1x1(x, weight, bias), dim=1)`` in one tensor-core kernel (``ffb6d_conv1x1_log_softmax_fwd``):
    PSPNet's ``final`` (models/cnn/pspnet.py:108-112).  :param x: ``[B,Ci,H,W]`` float32 CUDA; :param weight:
    ``[Co,Ci(,1,1)]`` or its :class:`PackedWeight`, Co <= 128; :param bias: ``[Co]``.  :return: ``[B,Co,H,W]``"""
    xc = _tensor(x, "x", shape=4)
    B, Ci, H, W = xc.shape
    packed = weight if isinstance(weight, PackedWeight) else PackedWeight(weight)
    if packed.Ci != Ci or packed.device != xc.device:
        raise ValueError("weight takes %d channels on %s, x has %d on %s" % (packed.Ci, packed.device, Ci, xc.device))
    b = bias.detach().float().contiguous()
    if b.numel() != packed.Co or b.device != xc.device:
        raise ValueError("bias must have %d elements on %s" % (packed.Co, xc.device))
    out = torch.empty((B, packed.Co, H, W), dtype=torch.float32, device=xc.device)
    launch(lib.ffb6d_conv1x1_log_softmax_fwd, xc.device, xc.data_ptr(), B, Ci, H * W, packed.data.data_ptr(),
           b.data_ptr(), packed.Co, out.data_ptr())
    return out


# --------------------------------------------------------------------------- PSP head of the image branch (training)
def psp_bottleneck_bwd(grad_out, out):
    """Backward of :func:`psp_bottleneck` (``ffb6d_psp_bottleneck_bwd``, one launch) from ``grad_out`` and the forward's
    ``out`` ``[B,Co,H,W]`` float32 CUDA.  :return: ``(grad_z [B,Co,H,W], grad_table [B*50, Co], grad_sum [B, Co])``:
    the gradient of the bottleneck's pre-ReLU sum (torch's ReLU backward on ``out``), that of the prior table in the
    forward's layout (block ``s`` is ``[B, s*s, Co]``, in the order of :data:`PSP_SIZES`), and the per-frame sums of
    ``grad_z`` (the bias gradient is their sum over the frames)."""
    o = _tensor(out, "out", shape=4)
    B, Co, H, W = o.shape
    g = _tensor(grad_out, "grad_out", shape=o.shape, device=o.device)
    gz = torch.empty_like(o)
    table = torch.empty((_PSP_BINS * B, Co), dtype=torch.float32, device=o.device)
    gsum = torch.empty((B, Co), dtype=torch.float32, device=o.device)
    launch(lib.ffb6d_psp_bottleneck_bwd, o.device, g.data_ptr(), o.data_ptr(), B, Co, H, W, gz.data_ptr(),
           table.data_ptr(), gsum.data_ptr())
    return gz, table, gsum


def psp_pool_bwd(grad_pooled, grad_x):
    """Adjoint of :func:`psp_pool` (``ffb6d_psp_pool_bwd``, one launch), accumulated: ``grad_x [B,C,H,W]`` float32 CUDA
    (contiguous; updated in place and returned) ``+= sum_s pool_s^T(grad_pooled[s])``.  :param grad_pooled: the four
    ``[B,C,s,s]`` gradients of :func:`psp_pool`'s outputs, or one flat buffer in its block order."""
    gx = _tensor(grad_x, "grad_x", shape=4)
    if gx.data_ptr() != grad_x.data_ptr():
        raise ValueError("grad_x must be contiguous (it is updated in place)")
    B, C, H, W = gx.shape
    if isinstance(grad_pooled, torch.Tensor):
        gp = _tensor(grad_pooled, "grad_pooled", shape=(_PSP_BINS * B * C,))
    else:
        parts = [_tensor(p, "grad_pooled[%d]" % i, shape=(B, C, s, s))
                 for i, (s, p) in enumerate(zip(PSP_SIZES, grad_pooled))]
        if len(parts) != len(PSP_SIZES):
            raise ValueError("grad_pooled must hold %d tensors" % len(PSP_SIZES))
        gp = torch.cat([p.reshape(-1) for p in parts])
    if gp.device != gx.device:
        raise ValueError("grad_pooled and grad_x must be on the same device")
    launch(lib.ffb6d_psp_pool_bwd, gx.device, gp.data_ptr(), B, C, H, W, gx.data_ptr())
    return grad_x


def log_softmax_bwd(grad_out, out):
    """Backward of ``log_softmax(dim=1)`` from its result ``out`` and ``grad_out`` ``[B,C,...]`` float32 CUDA
    (``ffb6d_log_softmax_bwd``, one launch): ``grad_out - exp(out) * grad_out.sum(1, keepdim=True)``."""
    _need_cuda(out, "out")
    if out.dtype != torch.float32 or out.dim() < 2:
        raise ValueError("out must be float32 [B,C,...], got %s %s" % (out.dtype, tuple(out.shape)))
    o = out.contiguous()
    g = _tensor(grad_out, "grad_out", shape=o.shape, device=o.device)
    B, C = o.shape[0], o.shape[1]
    gi = torch.empty_like(o)
    launch(lib.ffb6d_log_softmax_bwd, o.device, g.data_ptr(), o.data_ptr(), B, C, o.numel() // (B * C), gi.data_ptr())
    return gi


def upsample_bilinear2d_bwd(grad_out, input_size):
    """Backward of ``F.interpolate(x, mode="bilinear", align_corners=True)`` (``ffb6d_upsample_bilinear2d_bwd``, one
    launch): ``grad_out [B,C,Ho,Wo]`` float32 CUDA, ``input_size = (Hi, Wi)``.  :return: ``grad_in [B,C,Hi,Wi]``"""
    g = _tensor(grad_out, "grad_out", shape=4)
    B, C, Ho, Wo = g.shape
    Hi, Wi = (int(v) for v in input_size)
    gi = torch.empty((B, C, Hi, Wi), dtype=torch.float32, device=g.device)
    launch(lib.ffb6d_upsample_bilinear2d_bwd, g.device, g.data_ptr(), B, C, Hi, Wi, Ho, Wo, gi.data_ptr())
    return gi


class _UpsampleBilinear2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale_factor):
        ctx.in_size = tuple(x.shape[2:])
        return torch.nn.functional.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=True)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        return upsample_bilinear2d_bwd(grad.contiguous(), ctx.in_size), None


def upsample_bilinear2d(x, scale_factor=2):
    """``F.interpolate(x, scale_factor=scale_factor, mode="bilinear", align_corners=True)`` (``nn.Upsample`` of
    PSPUpsample, models/cnn/pspnet.py:36-48) with a deterministic backward: the forward is torch's, the backward
    :func:`upsample_bilinear2d_bwd`.  :param x: ``[B,C,H,W]`` float32 CUDA."""
    _tensor(x, "x", shape=4)
    return _UpsampleBilinear2d.apply(x, scale_factor)


# --------------------------------------------------------------------------- PSPUpsample at the input's resolution
def upconv_chunk(Ci, Co):
    """Output channels per chunk of :func:`upsample_conv3x3`: the chunk's tap table ``[B, 9 Cc, Hi, Wi]`` is at most
    the upsampled input ``[B, Ci, 2 Hi, 2 Wi]`` the torch path forms (``9 Cc <= 4 Ci``; one channel when ``Ci < 3``)."""
    return max(1, min(int(Co), 4 * int(Ci) // 9))


class UpConvWeights:
    """A 3x3 conv's weight ``[Co, Ci, 3, 3]`` stacked by tap and packed for :func:`upsample_conv3x3`, one
    :class:`PackedWeight` per chunk of :func:`upconv_chunk` output channels: chunk ``(co0, Cc)`` holds ``[9 Cc, Ci]``
    with row ``t Cc + j = W[co0 + j, :, ky, kx]``, ``t = 3 ky + kx``.  Build it once per weight version."""

    def __init__(self, weight):
        _need_cuda(weight, "weight")
        if weight.dim() != 4 or tuple(weight.shape[2:]) != (3, 3):
            raise ValueError("UpConvWeights: a [Co, Ci, 3, 3] weight expected, got %s" % (tuple(weight.shape),))
        w = weight.detach().float()
        self.Co, self.Ci = int(w.shape[0]), int(w.shape[1])
        self.device = w.device
        cc = upconv_chunk(self.Ci, self.Co)
        self.chunks = [(co0, min(cc, self.Co - co0)) for co0 in range(0, self.Co, cc)]
        self.packs = [PackedWeight(upconv_stack(w, co0, n)) for co0, n in self.chunks]


def upconv_stack(weight, co0, cc):
    """Rows ``t cc + j = weight[co0 + j, :, ky, kx]`` (``t = 3 ky + kx``) of a ``[Co, Ci, 3, 3]`` weight: ``[9 cc, Ci]``."""
    return weight[co0:co0 + cc].permute(2, 3, 0, 1).reshape(9 * cc, weight.shape[1])


def upconv_pack(weight):
    """:class:`UpConvWeights` of a 3x3 conv's weight ``[Co, Ci, 3, 3]``."""
    return UpConvWeights(weight)


def upconv_taps_fwd(table, out, co0, bias=None, scale=None, shift=None, alpha=None):
    """The epilogue of :func:`upsample_conv3x3` (``ffb6d_upconv_taps_fwd``, one launch): writes the chunk of output
    channels ``co0 .. co0 + Cc - 1`` of ``out [B, Co, 2 Hi, 2 Wi]`` from its tap table ``table [B, 9 Cc, Hi, Wi]``:
    ``act(affine(bias + sum of the nine shifted, upsampled planes))``; ``scale``/``shift`` ``[Co]`` the folded
    BatchNorm, ``alpha [1]`` PReLU's weight (each optional).  Returns ``out``."""
    t = _tensor(table, "table", shape=4)
    o = _tensor(out, "out", shape=4)
    if o.data_ptr() != out.data_ptr() or o.device != t.device:
        raise ValueError("out must be contiguous and on the table's device (it is written in place)")
    B, C9, Hi, Wi = t.shape
    Co = o.shape[1]
    if C9 % 9 or o.shape[0] != B or tuple(o.shape[2:]) != (2 * Hi, 2 * Wi):
        raise ValueError("table [B, 9 Cc, Hi, Wi] and out [B, Co, 2 Hi, 2 Wi] expected, got %s and %s"
                         % (tuple(t.shape), tuple(o.shape)))
    if (scale is None) != (shift is None):
        raise ValueError("scale and shift come together")
    b, sc, sh, a = (None if v is None else _tensor(v.detach().float().reshape(-1), name, shape=(n,), device=t.device)
                    for v, name, n in ((bias, "bias", Co), (scale, "scale", Co), (shift, "shift", Co),
                                       (alpha, "alpha", 1)))
    launch(lib.ffb6d_upconv_taps_fwd, t.device, t.data_ptr(), B, Co, int(co0), C9 // 9, Hi, Wi, ptr(b), ptr(sc), ptr(sh),
           ptr(a), o.data_ptr())
    return out


def upconv_taps_bwd(grad_z, co0, cc):
    """Adjoint of :func:`upconv_taps_fwd`'s tap sum (``ffb6d_upconv_taps_bwd``, one launch) for the chunk of ``cc``
    output channels from ``co0``: ``grad_z [B, Co, Ho, Wo]`` (Ho, Wo even) -> ``[B, 9 cc, Ho / 2, Wo / 2]``."""
    g = _tensor(grad_z, "grad_z", shape=4)
    B, Co, Ho, Wo = g.shape
    if Ho % 2 or Wo % 2:
        raise ValueError("grad_z must be [B, Co, 2 Hi, 2 Wi], got %s" % (tuple(g.shape),))
    gt = torch.empty((B, 9 * int(cc), Ho // 2, Wo // 2), dtype=torch.float32, device=g.device)
    launch(lib.ffb6d_upconv_taps_bwd, g.device, g.data_ptr(), B, Co, int(co0), int(cc), Ho // 2, Wo // 2, gt.data_ptr())
    return gt


def upsample_conv3x3(x, weights, bias=None, scale=None, shift=None, alpha=None, out=None):
    """``conv3x3(upsample_x2(x, align_corners=True)) + bias``, padding 1, without the upsampled map: per chunk of
    output channels the stacked GEMM at the input's resolution (``ffb6d_fusion_mlp_fwd_ex`` with the packed
    :class:`UpConvWeights`) and its tap epilogue (:func:`upconv_taps_fwd`), optionally followed by the folded BatchNorm
    ``scale``/``shift`` and PReLU ``alpha``.  :param x: ``[B, Ci, Hi, Wi]`` float32 CUDA.  :return: ``[B, Co, 2 Hi, 2 Wi]``"""
    xc = _tensor(x, "x", shape=4)
    B, Ci, Hi, Wi = xc.shape
    if not isinstance(weights, UpConvWeights):
        raise TypeError("weights must be ops.upconv_pack(conv.weight)")
    if Ci != weights.Ci or weights.device != xc.device:
        raise ValueError("the conv takes %d channels on %s, x has %d on %s" % (weights.Ci, weights.device, Ci, xc.device))
    if out is None:
        out = torch.empty((B, weights.Co, 2 * Hi, 2 * Wi), dtype=torch.float32, device=xc.device)
    for (co0, cc), pk in zip(weights.chunks, weights.packs):
        one, zero = torch.ones(9 * cc, device=xc.device), torch.zeros(9 * cc, device=xc.device)
        table = fusion_mlp(xc, None, pk, one, zero, relu=False)          # [B, 9 cc, Hi, Wi]
        upconv_taps_fwd(table, out, co0, bias, scale, shift, alpha)
        del table
    return out


def prelu_(y, alpha):
    """``nn.PReLU()`` with one weight, in place on ``y`` float32 CUDA (``ffb6d_prelu_fwd``); ``alpha [1]`` is read on
    the device, so the call can be captured in a CUDA graph.  Returns ``y``."""
    _need_cuda(y, "y")
    if y.dtype != torch.float32 or not y.is_contiguous():
        raise ValueError("y must be contiguous float32")
    a = _tensor(alpha.detach().float().reshape(-1), "alpha", shape=(1,), device=y.device)
    launch(lib.ffb6d_prelu_fwd, y.device, y.data_ptr(), y.numel(), a.data_ptr(), y.data_ptr())
    return y


def bn_prelu_bwd(z, grad_y, stats, alpha):
    """Backward of ``PReLU(u)``, ``u`` the training BatchNorm's output of ``z [B, C, ...]`` with the forward's
    ``stats [C, 4]`` (``ffb6d_bn_prelu_bwd``, one launch; ``u`` recomputed, not saved).  :return: ``(grad_u,
    grad_alpha [1])``; grad_alpha is the fp64 row sums added in a fixed order."""
    _need_cuda(z, "z")
    if z.dtype != torch.float32 or z.dim() < 2 or not z.is_contiguous():
        raise ValueError("z must be contiguous float32 [B, C, ...]")
    B, Cn = z.shape[0], z.shape[1]
    g = _tensor(grad_y, "grad_y", shape=z.shape)
    st = _tensor(stats, "stats", shape=(Cn, 4))
    a = _tensor(alpha.detach().float().reshape(-1), "alpha", shape=(1,), device=z.device)
    gu = torch.empty_like(z)
    part = torch.empty(B * Cn, dtype=torch.float64, device=z.device)
    launch(lib.ffb6d_bn_prelu_bwd, z.device, z.data_ptr(), g.data_ptr(), st.data_ptr(), B, Cn, z.numel() // (B * Cn),
           a.data_ptr(), gu.data_ptr(), part.data_ptr())
    return gu, part.sum().float().reshape(1)
