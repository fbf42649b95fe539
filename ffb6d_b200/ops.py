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
from ._lib import lib, check, LAYOUT_NCS, LAYOUT_NSC

import os as _os
_DEBUG_GRID = bool(_os.environ.get("FFB6D_DEBUG_GRID"))   # keep KNN workspaces for tools/grid_debug.py
_debug_ws = []
_I64 = (torch.int64,)
_IDX = (torch.int32, torch.int64)


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _need_cuda(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor, got %r" % (name, type(t)))
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: ffb6d_b200 has no CPU path" % name)


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
    with torch.cuda.device(sup.device):
        ws_bytes = int(lib.ffb6d_knn_workspace_bytes(B, S, Q, k)) if algo != 1 else 0
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=sup.device) if ws_bytes else None
        check(lib.ffb6d_knn_batch_algo(sup.data_ptr(), qry.data_ptr(), B, S, Q, k, out.data_ptr(),
                                       int(dt == torch.int64), ws.data_ptr() if ws is not None else None,
                                       ws_bytes, int(algo), _stream(sup.device)))
    if _DEBUG_GRID:
        _debug_ws.append((B, S, Q, k, ws))
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
        with torch.cuda.device(sup.device):
            self.nbytes = int(lib.ffb6d_knn_grid_bytes(self.B, self.S))
            self.mem = torch.empty(self.nbytes, dtype=torch.uint8, device=sup.device)
            check(lib.ffb6d_knn_grid_build(sup.data_ptr(), self.B, self.S, self.k_hint,
                                           self.mem.data_ptr(), self.nbytes, _stream(sup.device)))

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
        with torch.cuda.device(dev):
            sb = int(lib.ffb6d_knn_grid_query_bytes(self.B, Q))
            scratch = torch.empty(max(sb, 1), dtype=torch.uint8, device=dev)
            qw = int(query_width) if query_width and Q % int(query_width) == 0 else 0
            check(lib.ffb6d_knn_grid_query_organized(self.support.data_ptr(), qry.data_ptr(), self.B, self.S, Q, k,
                                                     out.data_ptr(), int(dt == torch.int64), self.mem.data_ptr(),
                                                     self.nbytes, scratch.data_ptr(), sb, qw, _stream(dev)))
        return out


def knn_uses_grid(B, S, Q, k):
    """True when :func:`knn_search` would answer this problem with the grid search (rather than
    the tiled scan it uses for small problems)."""
    return int(lib.ffb6d_knn_workspace_bytes(B, S, Q, int(k))) > 0


def subset_nn_from_knn(support, query_pts, knn_idx):
    """``cld_interp_idx{i}`` read off ``cld_nei_idx{i}`` (``ffb6d_knn_subset_nn``): the nearest point of ``support``
    for every query, when ``support [B,S,3]`` is the first S rows of ``query_pts [B,Q,3]`` (cloud level i+1 is a row
    prefix of level i, datasets/ycb/ycb_dataset.py:278) and ``knn_idx [B,Q,K]`` is the K-neighbour self search of
    ``query_pts`` (:275-277).  The first entry of a row that is < S is the answer (rows are ordered by (distance,
    index) over all of ``query_pts``); the ~0.75**K of the rows without one get a full scan.  Returns ``[B,Q,1]`` in
    the dtype of ``knn_idx``; identical to ``knn_search(support, query_pts, 1)``."""
    _need_cuda(support, "support")
    _need_cuda(query_pts, "query_pts")
    _need_cuda(knn_idx, "knn_idx")
    sup, qry = support.contiguous().float(), query_pts.contiguous().float()
    if sup.dim() != 3 or qry.dim() != 3 or sup.shape[2] != 3 or qry.shape[2] != 3 or sup.shape[0] != qry.shape[0]:
        raise ValueError("expected support [B,S,3] and query [B,Q,3]")
    B, S, Q = sup.shape[0], sup.shape[1], qry.shape[1]
    if knn_idx.dim() != 3 or knn_idx.shape[0] != B or knn_idx.shape[1] != Q or knn_idx.dtype not in _IDX:
        raise ValueError("knn_idx must be an int32 / int64 [B,Q,K] tensor, got %s %s" % (tuple(knn_idx.shape), knn_idx.dtype))
    if S < 1 or S > Q:
        raise ValueError("the support (%d rows) must be a non-empty row prefix of the %d queries" % (S, Q))
    knn = knn_idx.contiguous()
    out = torch.empty((B, Q, 1), dtype=knn.dtype, device=sup.device)
    with torch.cuda.device(sup.device):
        sb = int(lib.ffb6d_knn_grid_query_bytes(B, Q))
        scratch = torch.empty(max(sb, 1), dtype=torch.uint8, device=sup.device)
        check(lib.ffb6d_knn_subset_nn(sup.data_ptr(), qry.data_ptr(), B, S, Q, knn.data_ptr(), int(knn.shape[2]),
                                      out.data_ptr(), int(knn.dtype == torch.int64), scratch.data_ptr(), sb, _stream(sup.device)))
    return out


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
        with torch.cuda.device(f3.device):
            check(lib.ffb6d_gather_max_fwd(f3.data_ptr(), idx_c.data_ptr(), i64, B, Cc, S, Q, K,
                                           layout, out.data_ptr(), _stream(f3.device)))
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
    with torch.cuda.device(f3.device):
        check(lib.ffb6d_gather_max_bwd(f3.data_ptr(), idx_c.data_ptr(),
                                       int(idx_c.dtype == torch.int64), g.data_ptr(), B, Cc, S,
                                       Q, K, layout, gf.data_ptr(), _stream(f3.device)))
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
    dev = f3.device
    with torch.cuda.device(dev):
        nbytes = int(lib.ffb6d_gather_max_bwd_det_workspace_bytes(B, Cc, S, Q, K))
        ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
        check(lib.ffb6d_gather_max_bwd_det(f3.data_ptr(), idx_c.data_ptr(), int(idx_c.dtype == torch.int64),
                                           g.data_ptr(), B, Cc, S, Q, K, layout, ws.data_ptr(), nbytes,
                                           gf.data_ptr(), _stream(dev)))


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
    with torch.cuda.device(idx_c.device):
        check(lib.ffb6d_check_indices(idx_c.data_ptr(), i64, idx_c.numel(), int(S), _stream(idx_c.device)))


# --------------------------------------------------------------------------- neighbour gather
class _GatherNeighbour(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pc, idx):
        pc = pc.contiguous()
        idx_c, i64 = _idx_arg(idx, "neighbor_idx")
        B, S, D = pc.shape
        N, K = idx_c.shape[1], idx_c.shape[2]
        out = torch.empty((B, N, K, D), dtype=torch.float32, device=pc.device)
        with torch.cuda.device(pc.device):
            check(lib.ffb6d_gather_neighbour_fwd(pc.data_ptr(), idx_c.data_ptr(), i64, B, S, D, N, K,
                                                 out.data_ptr(), _stream(pc.device)))
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
        if deterministic_backward():
            with torch.cuda.device(g.device):
                nbytes = int(lib.ffb6d_gather_neighbour_bwd_det_workspace_bytes(B, S, N, K))
                ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=g.device)
                check(lib.ffb6d_gather_neighbour_bwd_det(g.data_ptr(), idx_c.data_ptr(), int(idx_c.dtype == torch.int64),
                                                         B, S, D, N, K, ws.data_ptr(), nbytes, gpc.data_ptr(),
                                                         _stream(g.device)))
            return gpc, None
        with torch.cuda.device(g.device):
            check(lib.ffb6d_gather_neighbour_bwd(g.data_ptr(), idx_c.data_ptr(),
                                                 int(idx_c.dtype == torch.int64), B, S, D, N, K,
                                                 gpc.data_ptr(), _stream(g.device)))
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
        with torch.cuda.device(xyz.device):
            check(lib.ffb6d_relative_pos_encoding_cm_fwd(xyz.data_ptr(), idx_c.data_ptr(), i64, B, N, K,
                                                         out.data_ptr(), _stream(xyz.device)))
        return out
    out = torch.empty((B, N, K, 10), dtype=torch.float32, device=xyz.device)
    with torch.cuda.device(xyz.device):
        check(lib.ffb6d_relative_pos_encoding_fwd(xyz.data_ptr(), idx_c.data_ptr(), i64, B, N, K,
                                                  out.data_ptr(), _stream(xyz.device)))
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
        with torch.cuda.device(w.device):
            check(lib.ffb6d_fusion_mlp_pack(w.data_ptr(), self.Co, self.Ci, self.data.data_ptr(), nbytes,
                                            _stream(w.device)))


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
    with torch.cuda.device(x1.device):
        check(lib.ffb6d_fusion_mlp_fwd_ex(
            x1c.data_ptr(), C1, x2c.data_ptr() if x2c is not None else None, C2, packed.data.data_ptr(),
            sc.data_ptr(), sh.data_ptr(), B, Co, P, 2 if negative_slope is not None else int(bool(relu)),
            float(negative_slope or 0.0), addc.data_ptr() if addc is not None else None,
            idxc.data_ptr() if idxc is not None else None, i64, NA,
            LAYOUT_NSC if out_channels_last else LAYOUT_NCS, out.data_ptr(), _stream(x1.device)))
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
        self.data = torch.empty(self.nbytes, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            check(getattr(lib, self._build)(idx_c.data_ptr(), i64, self.B, self.P, self.NA, self.data.data_ptr(),
                                            self.nbytes, _stream(self.device)))

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
    with torch.cuda.device(grad.device):
        check(getattr(lib, plan._sum)(g.data_ptr(), plan.data.data_ptr(), plan.nbytes, B, Cc, plan.P, plan.NA,
                                      out.data_ptr(), _stream(grad.device)))
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
    with torch.cuda.device(f1.device):
        check(lib.ffb6d_att_pool_fwd(f1c.data_ptr(), C1, f2c.data_ptr() if f2c is not None else None, C2,
                                     a.data_ptr(), B, N, K, out.data_ptr(), _stream(f1.device)))
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
    with torch.cuda.device(f.device):
        check(lib.ffb6d_lfa_att_pool_fused(
            xyz.data_ptr(), idx_c.data_ptr(), i64, f.data_ptr(), w1.data_ptr(), s1.data_ptr(), t1.data_ptr(),
            w2.data_ptr() if w2 is not None else None, s2.data_ptr() if w2 is not None else None,
            t2.data_ptr() if w2 is not None else None, wfc.data_ptr(), wo.data_ptr(), so.data_ptr(), to.data_ptr(),
            B, N, K, Dh, Do, float(negative_slope), out.data_ptr(), _stream(f.device)))
    return out


def lfa_fusable(d_half, k):
    """True when :func:`lfa_att_pool_fused` covers this width / neighbour count."""
    return int(k) == 16 and int(d_half) in (16, 32, 64)


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
    if Kn.shape == (3, 3):
        intr = np.array([Kn[0, 0], Kn[1, 1], Kn[0, 2], Kn[1, 2]], np.float64)
        per_frame = 0
    elif Kn.shape == (B, 3, 3):
        intr = np.stack([Kn[:, 0, 0], Kn[:, 1, 1], Kn[:, 0, 2], Kn[:, 1, 2]], 1).copy()
        per_frame = 1
    else:
        raise ValueError("K must be [3,3] or [B,3,3], got %s" % (Kn.shape,))
    return torch.from_numpy(intr).to(dev), per_frame


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
    if labels.dtype != torch.uint8 or tuple(labels.shape) != (B, H, W):
        raise ValueError("labels must be uint8 [B,H,W], got %s %s" % (labels.dtype, tuple(labels.shape)))
    if nrm_map.dtype not in (torch.float32, torch.float64) or tuple(nrm_map.shape) != (B, H, W, 3):
        raise ValueError("nrm_map must be float32 or float64 [B,H,W,3], got %s %s" % (nrm_map.dtype, tuple(nrm_map.shape)))
    if obj_cls.dtype != torch.int32 or obj_cls.dim() != 2 or obj_cls.shape[0] != B:
        raise ValueError("obj_cls must be int32 [B,n_obj], got %s %s" % (obj_cls.dtype, tuple(obj_cls.shape)))
    n_obj = obj_cls.shape[1]
    if obj_kps.dtype != torch.float64 or obj_kps.dim() != 4 or tuple(obj_kps.shape[:2]) != (B, n_obj) \
            or obj_kps.shape[3] != 3:
        raise ValueError("obj_kps must be float64 [B,n_obj,n_kps,3], got %s %s" % (obj_kps.dtype, tuple(obj_kps.shape)))
    n_kps = obj_kps.shape[2]
    if obj_ctr.dtype != torch.float64 or tuple(obj_ctr.shape) != (B, n_obj, 3):
        raise ValueError("obj_ctr must be float64 [B,n_obj,3], got %s %s" % (obj_ctr.dtype, tuple(obj_ctr.shape)))
    for t, name in tensors:
        _need_cuda(t, name)
        if t.device != depth_m.device:
            raise ValueError("%s is on %s, depth_m on %s" % (name, t.device, depth_m.device))
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
    with torch.cuda.device(dev):
        check(lib.ffb6d_point_item(depth_c.data_ptr(), B, H, W, intr_d.data_ptr(), per_frame, ch.data_ptr(), N,
                                   rgb_c.data_ptr(), labels_c.data_ptr(), nrm.data_ptr(), cls_c.data_ptr(),
                                   kps_c.data_ptr(), ctr_c.data_ptr(), n_obj, n_kps, cld_rgb_nrm.data_ptr(),
                                   labels_pt.data_ptr(), kp_targ_ofst.data_ptr(), ctr_targ_ofst.data_ptr(),
                                   _stream(dev)))
    return cld_rgb_nrm, labels_pt, kp_targ_ofst, ctr_targ_ofst


def sample_valid_pixels(depth, n_points, seed=0, min_depth=1e-8, return_count=False):
    """The datasets' point sampling on the GPU (datasets/ycb/ycb_dataset.py:218-235): the valid pixels of each
    depth map (``depth > min_depth``) are compacted, ``n_points`` of them are drawn uniformly without replacement
    (all of them, repeated cyclically like ``np.pad(..., 'wrap')``, when fewer exist) and returned in uniformly
    random order.  Deterministic per ``seed``; the picks have the reference's distribution but do not replay
    numpy's random stream.

    :param depth: ``[B,H,W]`` float32 CUDA; :return: ``choose [B,1,n_points]`` int32 flat pixel indices
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
    with torch.cuda.device(dev):
        nbytes = int(lib.ffb6d_sample_pixels_workspace_bytes(B, H, W))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        check(lib.ffb6d_sample_pixels(depth.data_ptr(), B, H, W, float(min_depth), int(n_points), int(seed) & (2 ** 64 - 1),
                                      choose.data_ptr(), count.data_ptr(), ws.data_ptr(), nbytes, _stream(dev)))
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
    with torch.cuda.device(dev):
        nbytes = int(lib.ffb6d_fill_depth_workspace_bytes(B, H, W))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        check(lib.ffb6d_fill_depth(raw.data_ptr(), B, H, W, cs, *(o.data_ptr() if o is not None else None for o in outs),
                                   ws.data_ptr(), nbytes, _stream(dev)))
    return tuple(outs)


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
    with torch.cuda.device(dev):
        check(lib.ffb6d_backproject(depth.data_ptr(), B, H, W, intr_d.data_ptr(), per_frame, ch.data_ptr(), N,
                                    cld.data_ptr(), pyr[2].data_ptr(), pyr[4].data_ptr(), pyr[8].data_ptr(),
                                    _stream(dev)))
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
    with torch.cuda.device(dev):
        nbytes = int(lib.ffb6d_mean_shift_workspace_bytes(G, N))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        check(lib.ffb6d_mean_shift_fit(votes.data_ptr(), vptr, stride, G, N, float(bandwidth), int(max_iter),
                                       centres.data_ptr(), labels.data_ptr(), iters.data_ptr(),
                                       modes.data_ptr() if modes is not None else None, ws.data_ptr(), nbytes, _stream(dev)))
    out = (centres, labels.bool(), iters)
    return out + (modes,) if return_modes else out


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
    with torch.cuda.device(A.device):
        check(lib.ffb6d_best_fit_transform(A.data_ptr(), B.data_ptr(), G, M, T.data_ptr(), _stream(A.device)))
    return T[0] if single else T


def _aug_image(t, name, shape=None, dtype=torch.uint8):
    _need_cuda(t, name)
    if t.dtype != dtype or (shape is not None and tuple(t.shape) != tuple(shape)):
        raise ValueError("%s must be %s %s, got %s %s" % (name, dtype, shape, t.dtype, tuple(t.shape)))
    return t.contiguous()


def rgb_add_noise(rgb, plan, seed, noise=None):
    """The datasets' ``rgb_add_noise`` (datasets/ycb/ycb_dataset.py:107-143, linemod_dataset.py:142-164) for a batch
    on the GPU (``ffb6d_rgb_add_noise``).

    :param rgb: ``[B,H,W,3]`` uint8 CUDA, H, W >= 32 (the channel roles are the reference's: it feeds RGB data to
      ``COLOR_BGR2HSV``)
    :param plan: ``[B, REC_LEN]`` float64 numpy records of :func:`ffb6d_b200.augment.draw_rgb_noise`
    :param seed: key of the per-pixel normal draws (frame b of the batch, the record's pass); use one seed per batch
    :param noise: optional ``[2,B,H,W,3]`` float64 CUDA normals to use instead of the generator's (the first for
      ``gaussian_noise``, the second for YCB's ``normal(0, 7)``), e.g. to replay numpy's stream
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
    if not (0 <= int(seed) < 1 << 64):
        raise ValueError("seed must fit 64 bits, got %r" % (seed,))
    dev = rgb.device
    if noise is not None:
        noise = _aug_image(noise, "noise", (2, B, H, W, 3), torch.float64)
        if noise.device != dev:
            raise ValueError("noise is on %s, rgb on %s" % (noise.device, dev))
    src = rgb.contiguous()
    plan_d = torch.from_numpy(plan).to(dev)
    out = torch.empty_like(src)
    work = torch.empty_like(src)
    with torch.cuda.device(dev):
        check(lib.ffb6d_rgb_add_noise(src.data_ptr(), B, H, W, plan.ctypes.data, plan_d.data_ptr(), int(seed),
                                      None if noise is None else noise.data_ptr(), out.data_ptr(), work.data_ptr(),
                                      _stream(dev)))
    return out


def add_real_back(rgb, labels, dpt, back_rgb, back_labels, back_dpt, apply_rgb=None, dataset="ycb", active=None):
    """The datasets' ``add_real_back`` (datasets/ycb/ycb_dataset.py:145-163, linemod_dataset.py:166-186) for a batch
    on the GPU (``ffb6d_add_real_back``), after the worker has loaded the background frames.

    :param rgb: ``[B,H,W,3]`` uint8; :param labels: ``[B,H,W]`` uint8 (the frame's labels; 0 is background)
    :param dpt: ``[B,H,W]`` uint16 raw depth (YCB ``dpt_um``; LineMOD ``dpt_mm.astype(np.uint16)``)
    :param back_rgb: ``[B,H,W,3]`` uint8; :param back_labels: ``[B,H,W]`` or ``[B,H,W,3]`` uint8 (the background
      frame's label image, YCB, or mask, LineMOD); :param back_dpt: ``[B,H,W]`` uint16
    :param apply_rgb: LineMOD: per-frame bools, the ``rand() < 0.6`` draw (YCB always composes the colour image)
    :param dataset: ``'ycb'`` or ``'linemod'``; :param active: per-frame bools, frames that go through
      ``add_real_back`` at all (default: every frame); the others pass through unchanged
    :return: ``(rgb [B,H,W,3] uint8, dpt [B,H,W] uint16)``; the composed depth is uint16 and feeds
      :func:`fill_missing` as it is
    """
    if dataset not in ("ycb", "linemod"):
        raise ValueError("dataset must be 'ycb' or 'linemod', got %r" % (dataset,))
    _need_cuda(rgb, "rgb")
    if rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3:
        raise ValueError("rgb must be uint8 [B,H,W,3], got %s %s" % (rgb.dtype, tuple(rgb.shape)))
    B, H, W, _ = rgb.shape
    labels = _aug_image(labels, "labels", (B, H, W))
    dpt = _aug_image(dpt, "dpt", (B, H, W), torch.uint16)
    back_rgb = _aug_image(back_rgb, "back_rgb", (B, H, W, 3))
    _need_cuda(back_labels, "back_labels")
    if back_labels.dim() == 3:
        back_labels = back_labels[..., None]
    ch = back_labels.shape[-1] if back_labels.dim() == 4 else 0
    back_labels = _aug_image(back_labels, "back_labels", (B, H, W, ch if ch in (1, 3) else -1))
    back_dpt = _aug_image(back_dpt, "back_dpt", (B, H, W), torch.uint16)
    for t, name in ((labels, "labels"), (dpt, "dpt"), (back_rgb, "back_rgb"), (back_labels, "back_labels"),
                    (back_dpt, "back_dpt")):
        if t.device != rgb.device:
            raise ValueError("%s is on %s, rgb on %s" % (name, t.device, rgb.device))
    act = np.ones(B, bool) if active is None else np.asarray(active, bool).reshape(-1)
    if dataset == "ycb":
        col = np.ones(B, bool) if apply_rgb is None else np.asarray(apply_rgb, bool).reshape(-1)
    else:
        if apply_rgb is None:
            raise ValueError("LineMOD needs apply_rgb (the frame's rand() < 0.6 draw)")
        col = np.asarray(apply_rgb, bool).reshape(-1)
    if act.shape != (B,) or col.shape != (B,):
        raise ValueError("apply_rgb and active must have one entry per frame (%d)" % B)
    dev = rgb.device
    mode = torch.from_numpy((act * (1 + 2 * col)).astype(np.uint8)).to(dev)
    src = rgb.contiguous()
    rgb_out = torch.empty_like(src)
    dpt_out = torch.empty_like(dpt)
    with torch.cuda.device(dev):
        check(lib.ffb6d_add_real_back(src.data_ptr(), labels.data_ptr(), dpt.data_ptr(), back_rgb.data_ptr(),
                                      back_labels.data_ptr(), ch, back_dpt.data_ptr(), mode.data_ptr(),
                                      0 if dataset == "ycb" else 1, B, H, W, rgb_out.data_ptr(), dpt_out.data_ptr(),
                                      _stream(dev)))
    return rgb_out, dpt_out


def color_jitter(rgb, plan, active=None):
    """The datasets' ``trancolor`` (torchvision ``ColorJitter(0.2, 0.2, 0.2, 0.05)`` on the PIL image,
    datasets/ycb/ycb_dataset.py:190-193, linemod_dataset.py:220-223) for a batch on the GPU
    (``ffb6d_color_jitter``); bitwise what torchvision 0.26 with Pillow 12.2 computes.

    :param rgb: ``[B,H,W,3]`` uint8 CUDA
    :param plan: ``[B, JITTER_PLAN_LEN]`` float64 plans of :func:`ffb6d_b200.augment.draw_color_jitter`; every
      frame's plan is validated, an inactive frame's too
    :param active: per-frame bools (a sequence, or a tensor), frames to jitter (default: every frame); the others,
      e.g. frames the dataset does not jitter, pass through unchanged
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
    plan_d = torch.from_numpy(plan).to(dev)
    work = torch.empty(B, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(lib.ffb6d_color_jitter(src.data_ptr(), B, H, W, plan.ctypes.data, plan_d.data_ptr(), act.data_ptr(),
                                     out.data_ptr(), work.data_ptr(), _stream(dev)))
    return out


def aug_noise_field(seed, B, H, W, stage, device="cuda"):
    """The ``[B,H,W,3]`` float64 normals that :func:`rgb_add_noise` draws for ``(seed, frame, stage)``; stage
    ``2*pass`` is ``gaussian_noise``'s, ``2*pass + 1`` YCB's ``normal(0, 7)``'s (``ffb6d_aug_noise_field``)."""
    out = torch.empty((B, H, W, 3), dtype=torch.float64, device=device)
    _need_cuda(out, "out")
    with torch.cuda.device(out.device):
        check(lib.ffb6d_aug_noise_field(int(seed), B, H, W, int(stage), out.data_ptr(), _stream(out.device)))
    return out
