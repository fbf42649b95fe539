"""``nn.Module`` twins of the reference's 1x1 layers and RandLA blocks, on this package's kernels, with
the reference's parameter names -- a maintainer can import-swap them and load published checkpoints.

* :class:`Conv2d` -- ``pt_utils.Conv2d`` of the fusion layers (models/pytorch_utils.py:168-201:
  ``conv`` -> ``normlayer.bn`` -> ``activation``; BatchNorm2d defaults eps 1e-5, momentum 0.1, ReLU).
* :class:`RandLAConv2d` -- RandLA's flavour (models/RandLA/pytorch_utils.py:163-197: ``conv`` -> ``bn.bn``
  -> ``activation``; eps 1e-6, momentum 0.99, LeakyReLU(0.2)).
* :class:`Att_pooling`, :class:`Building_block`, :class:`Dilated_res_block` -- models/RandLA/RandLANet.py:170-250.

Both modes run on the CUDA library:

* ``eval()``: one fused tensor-core kernel per layer (``ffb6d_fusion_mlp_fwd_ex``: concat + conv + folded
  BatchNorm + activation).
* ``train()``: batch-statistics BatchNorm and autograd -- forward = GEMM (wgmma) + ``ffb6d_bn_train_fwd``
  (running statistics updated like ``nn.BatchNorm2d``); backward = ``ffb6d_bn_train_bwd``, weight gradient
  ``ffb6d_fusion_mlp_wgrad`` (wgmma, split-K), input gradient = the forward GEMM with the transposed
  weight; neighbour gathers and attentive pooling have their own backward kernels.  Under
  ``torch.use_deterministic_algorithms(True)`` (or, for the weight gradients only, ``torch.backends.cudnn.deterministic``)
  the backwards that add with atomics take their run-to-run deterministic paths (:func:`ops.deterministic_backward`).
  After ``nn.SyncBatchNorm.convert_sync_batchnorm(model)`` a training-mode layer under an initialised process group
  of more than one rank normalises with the statistics of every rank's batch, as ``nn.SyncBatchNorm`` does
  (``ffb6d_bn_sync_*``, one all-gather per layer and direction; :meth:`_ConvBase._bn_sync`).

A layer accepts its input as one tensor or as the two halves of a concat (``layer(x1, x2)`` ==
``layer(torch.cat((x1, x2), 1))`` without materialising the concat, models/ffb6d.py:251-262).
:meth:`Conv2d.forward_interp` takes the second half as point features and the pixel -> point index of the
fusion's nearest interpolation, and never builds the interpolated map.
"""
import math

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F_

from . import dist as dist_, fusion, ops
from ._lib import lib, check

_ACT_NONE, _ACT_RELU, _ACT_LEAKY = 0, 1, 2


def _act_code(activation):
    if activation is None:
        return _ACT_NONE, 0.0
    if isinstance(activation, nn.ReLU):
        return _ACT_RELU, 0.0
    if isinstance(activation, nn.LeakyReLU):
        return _ACT_LEAKY, float(activation.negative_slope)
    raise ValueError("activation must be None, nn.ReLU or nn.LeakyReLU, got %r" % (activation,))


_const_cache = {}


def _ones_zeros(n, device):
    key = (n, device)
    if key not in _const_cache:
        _const_cache[key] = (torch.ones(n, device=device), torch.zeros(n, device=device))
    return _const_cache[key]


def _gemm(x1, x2, w2d):
    """z = W . cat(x1, x2), no affine, no activation (wgmma kernel)."""
    one, zero = _ones_zeros(w2d.shape[0], x1.device)
    return ops.fusion_mlp(x1, x2, w2d, one, zero, relu=False)


def _bn_act_fwd(z, B, Co, P, gamma, beta, running_mean, running_var, eps, momentum, act, slope, has_bn, sync=None):
    """y = act(BatchNorm with batch statistics(z)) (``ffb6d_bn_train_fwd``, also updates the running statistics) or,
    without BatchNorm, y = act(z).  Returns ``(y, stats, count)``; ``stats`` [Co, 4] and ``count`` are what
    :func:`_bn_act_bwd` reads.  With ``sync = (group, world)`` the statistics are those of the batches of every rank of
    ``group`` (torch's SyncBatchNorm): this rank's moments (``ffb6d_bn_sync_moments``), an all-gather, the rank-ordered
    combination (``ffb6d_bn_sync_fwd``); ``count`` [1] fp64 is then the global count, else None."""
    if not has_bn:
        if act == _ACT_RELU:
            return torch.relu(z), None, None
        return (F_.leaky_relu(z, slope) if act == _ACT_LEAKY else z), None, None
    stats = torch.empty((Co, 4), dtype=torch.float32, device=z.device)
    y = torch.empty_like(z)
    nbytes = int(lib.ffb6d_bn_workspace_bytes(Co, P))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=z.device)
    gamma_p = gamma.data_ptr() if gamma is not None else None
    beta_p = beta.data_ptr() if beta is not None else None
    rm_p = running_mean.data_ptr() if running_mean is not None else None
    rv_p = running_var.data_ptr() if running_var is not None else None
    with torch.cuda.device(z.device):
        if sync is None:
            check(lib.ffb6d_bn_train_fwd(
                z.data_ptr(), B, Co, P, gamma_p, beta_p, float(eps), float(momentum), rm_p, rv_p, int(act), float(slope),
                stats.data_ptr(), y.data_ptr(), ws.data_ptr(), nbytes, ops._stream(z.device)))
            return y, stats, None
        group, world = sync
        row = torch.empty(2 * Co + 1, dtype=torch.float64, device=z.device)
        check(lib.ffb6d_bn_sync_moments(z.data_ptr(), B, Co, P, row.data_ptr(), ws.data_ptr(), nbytes,
                                        ops._stream(z.device)))
        rows = dist_.all_gather_rows(row, group, world)
        count = torch.empty(1, dtype=torch.float64, device=z.device)
        check(lib.ffb6d_bn_sync_fwd(
            z.data_ptr(), B, Co, P, rows.data_ptr(), world, gamma_p, beta_p, float(eps), float(momentum), rm_p, rv_p,
            int(act), float(slope), stats.data_ptr(), count.data_ptr(), y.data_ptr(), ops._stream(z.device)))
    return y, stats, count


def _bn_act_bwd(z, gy, stats, B, Co, P, act, slope, has_bn, sync=None, count=None):
    """Backward of :func:`_bn_act_fwd`: ``(dz, dgamma, dbeta)``; dgamma / dbeta are None without BatchNorm.  With
    ``sync`` (and the forward's ``count``) dz uses the sums of every rank (``ffb6d_bn_sync_bwd_sums``, an all-gather,
    ``ffb6d_bn_sync_bwd``); dgamma / dbeta stay this rank's, for the gradient all-reduce of DDP to add."""
    dev = z.device
    with torch.cuda.device(dev):
        if has_bn:
            dz = torch.empty_like(z)
            ggamma = torch.empty(Co, dtype=torch.float32, device=dev)
            gbeta = torch.empty(Co, dtype=torch.float32, device=dev)
            nbytes = int(lib.ffb6d_bn_workspace_bytes(Co, P))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            if sync is None:
                check(lib.ffb6d_bn_train_bwd(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, Co, P, act, slope,
                                             ggamma.data_ptr(), gbeta.data_ptr(), dz.data_ptr(), ws.data_ptr(), nbytes,
                                             ops._stream(dev)))
                return dz, ggamma, gbeta
            group, world = sync
            row = torch.empty(2 * Co, dtype=torch.float64, device=dev)
            check(lib.ffb6d_bn_sync_bwd_sums(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, Co, P, act, slope,
                                             row.data_ptr(), ggamma.data_ptr(), gbeta.data_ptr(), ws.data_ptr(), nbytes,
                                             ops._stream(dev)))
            rows = dist_.all_gather_rows(row, group, world)
            check(lib.ffb6d_bn_sync_bwd(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, Co, P, rows.data_ptr(), world,
                                        count.data_ptr(), act, slope, dz.data_ptr(), ws.data_ptr(), nbytes,
                                        ops._stream(dev)))
            return dz, ggamma, gbeta
        if act != _ACT_NONE:
            dz = torch.empty_like(z)
            check(lib.ffb6d_act_bwd(z.data_ptr(), gy.data_ptr(), z.numel(), act, slope, dz.data_ptr(), ops._stream(dev)))
            return dz, None, None
    return gy, None, None


def _wgrad(dz, x1, x2, B, Co, P):
    """dW [Co, C1+C2] = sum over frames of dz [B, Co, P] . cat(x1, x2)^T (``ffb6d_fusion_mlp_wgrad``; under
    :func:`ffb6d_b200.ops.deterministic_backward` ``ffb6d_fusion_mlp_wgrad_det``, the splits added in a fixed order)."""
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    gw = torch.empty((Co, C1 + C2), dtype=torch.float32, device=dz.device)
    with torch.cuda.device(dz.device):
        if ops.deterministic_backward(weight_grad=True):
            nbytes = int(lib.ffb6d_fusion_mlp_wgrad_det_workspace_bytes(C1, C2, B, Co, P))
            ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dz.device)
            check(lib.ffb6d_fusion_mlp_wgrad_det(dz.data_ptr(), x1.data_ptr(), C1,
                                                 x2.data_ptr() if x2 is not None else None, C2, B, Co, P, ws.data_ptr(),
                                                 nbytes, gw.data_ptr(), ops._stream(dz.device)))
            return gw
        check(lib.ffb6d_fusion_mlp_wgrad(dz.data_ptr(), x1.data_ptr(), C1, x2.data_ptr() if x2 is not None else None,
                                         C2, B, Co, P, gw.data_ptr(), ops._stream(dz.device)))
    return gw


class _ConvBnActTrain(torch.autograd.Function):
    """conv1x1(cat(x1, x2)) -> [BatchNorm with batch statistics] -> activation, with its backward."""

    @staticmethod
    def forward(ctx, x1, x2, weight, bias, gamma, beta, running_mean, running_var, eps, momentum, act, slope, has_bn,
                sync=None):
        x1 = x1.contiguous()
        x2 = x2.contiguous() if x2 is not None else None
        B, C1 = x1.shape[0], x1.shape[1]
        C2 = x2.shape[1] if x2 is not None else 0
        w2d = weight.reshape(weight.shape[0], -1).contiguous()
        Co = w2d.shape[0]
        if bias is not None:     # conv bias (only without BatchNorm): the GEMM epilogue's shift
            one, _ = _ones_zeros(Co, x1.device)
            z = ops.fusion_mlp(x1, x2, w2d, one, bias, relu=False)
        else:
            z = _gemm(x1, x2, w2d)
        P = z.numel() // (B * Co)
        y, stats, count = _bn_act_fwd(z, B, Co, P, gamma, beta, running_mean, running_var, eps, momentum, act, slope,
                                      has_bn, sync)
        ctx.sync = sync
        ctx.save_for_backward(x1, x2, w2d, z, stats, gamma, count)
        ctx.meta = (B, C1, C2, Co, P, int(act), float(slope), bool(has_bn), bias is not None, tuple(weight.shape))
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy):
        x1, x2, w2d, z, stats, gamma, count = ctx.saved_tensors
        B, C1, C2, Co, P, act, slope, has_bn, has_bias, wshape = ctx.meta
        dz, ggamma, gbeta = _bn_act_bwd(z, gy.contiguous(), stats, B, Co, P, act, slope, has_bn, ctx.sync, count)
        gw = gbias = None
        if ctx.needs_input_grad[2]:
            gw = _wgrad(dz, x1, x2, B, Co, P).reshape(wshape)
        if has_bias:
            gbias = dz.reshape(B, Co, -1).sum(dim=(0, 2))
        # input gradients: dX = W^T . dz, one GEMM per half of the concat
        gx1 = gx2 = None
        if ctx.needs_input_grad[0]:
            gx1 = _gemm(dz, None, w2d[:, :C1].t().contiguous()).reshape(x1.shape)
        if x2 is not None and ctx.needs_input_grad[1]:
            gx2 = _gemm(dz, None, w2d[:, C1:].t().contiguous()).reshape(x2.shape)
        if gamma is None:
            ggamma = None
        return gx1, gx2, gw, gbias, ggamma, gbeta, None, None, None, None, None, None, None, None


class _InterpConvBnActTrain(torch.autograd.Function):
    """conv1x1(cat(x1, nearest_interpolation(p, idx))) -> [BatchNorm with batch statistics] -> activation without
    the interpolated map (SURVEY.md §8f-3): with W = [W1 | W2] split at C1,

        forward   Z = W2 . p (on the N' points, channels-last)      z = W1 . x1 + Z[idx]      y = act(BN(z))
        backward  dW1 = dz . x1^T    dx1 = W1^T . dz    dZ = segment_sum(dz, idx)    dW2 = dZ . p^T    dp = W2^T . dZ

    dZ is the transpose of the gather: for every point, the sum of dz over the pixels that map to it, in fp64 in
    ascending pixel order (``ffb6d_segment_sum``), so the gradients are bit-identical from run to run."""

    @staticmethod
    def forward(ctx, x1, p, idx, weight, bias, gamma, beta, running_mean, running_var, eps, momentum, act, slope, has_bn,
                sync=None):
        x1, p = x1.contiguous(), p.contiguous()
        B, C1 = x1.shape[0], x1.shape[1]
        C2, NA = p.shape[1], p.shape[2]
        w2d = weight.reshape(weight.shape[0], -1)
        Co = w2d.shape[0]
        w1, w2 = w2d[:, :C1].contiguous(), w2d[:, C1:].contiguous()
        one, zero = _ones_zeros(Co, x1.device)
        zp = ops.fusion_mlp(p, None, w2, one, zero, relu=False, out_channels_last=True)          # [B, N', Co]
        z = ops.fusion_mlp(x1, None, w1, one, bias if bias is not None else zero, relu=False, add=zp, add_idx=idx)
        P = z.numel() // (B * Co)
        y, stats, count = _bn_act_fwd(z, B, Co, P, gamma, beta, running_mean, running_var, eps, momentum, act, slope,
                                      has_bn, sync)
        ctx.sync = sync
        # dZ feeds dW2 and dp only: without either, the backward needs no plan
        ctx.plan = ops.segment_plan(idx, NA) if (ctx.needs_input_grad[1] or ctx.needs_input_grad[3]) else None
        ctx.save_for_backward(x1, p, w1, w2, z, stats, gamma, count)
        ctx.meta = (B, C1, C2, Co, P, NA, int(act), float(slope), bool(has_bn), bias is not None, tuple(weight.shape))
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy):
        x1, p, w1, w2, z, stats, gamma, count = ctx.saved_tensors
        B, C1, C2, Co, P, NA, act, slope, has_bn, has_bias, wshape = ctx.meta
        dz, ggamma, gbeta = _bn_act_bwd(z, gy.contiguous(), stats, B, Co, P, act, slope, has_bn, ctx.sync, count)
        dz = dz.reshape(B, Co, P)
        dzp = ops.segment_sum(dz, None, NA, plan=ctx.plan) if ctx.plan is not None else None     # [B, Co, N']
        gx1 = gp = gw = gbias = None
        if ctx.needs_input_grad[3]:
            gw = torch.cat((_wgrad(dz, x1.reshape(B, C1, P), None, B, Co, P),
                            _wgrad(dzp, p.reshape(B, C2, NA), None, B, Co, NA)), 1).reshape(wshape)
        if has_bias:
            gbias = dz.sum(dim=(0, 2))
        if ctx.needs_input_grad[0]:
            gx1 = _gemm(dz, None, w1.t().contiguous()).reshape(x1.shape)
        if ctx.needs_input_grad[1]:
            gp = _gemm(dzp, None, w2.t().contiguous()).reshape(p.shape)
        if gamma is None:
            ggamma = None
        return gx1, gp, None, gw, gbias, ggamma, gbeta, None, None, None, None, None, None, None, None


class _BNWrap(nn.Sequential):
    """The reference's ``_BNBase``: a Sequential holding one BatchNorm2d named ``bn``."""

    def __init__(self, channels, eps, momentum, dims=2):
        super().__init__()
        self.add_module("bn", (nn.BatchNorm2d if dims == 2 else nn.BatchNorm1d)(channels, eps=eps, momentum=momentum))
        nn.init.constant_(self[0].weight, 1.0)
        nn.init.constant_(self[0].bias, 0)


class _ConvBase(nn.Module):
    _bn_name = "normlayer"
    _bn_eps, _bn_momentum = 1e-5, 0.1

    _dims = 2

    def __init__(self, in_size, out_size, kernel_size=(1, 1), activation=None, bn=False, init=nn.init.kaiming_normal_,
                 bias=True, name=""):
        super().__init__()
        ks = (kernel_size,) if isinstance(kernel_size, int) else tuple(kernel_size)
        if any(k != 1 for k in ks):
            raise ValueError("only the 1x1 layers of the fusion / RandLA path are implemented here")
        bias = bias and (not bn)
        # holds the parameters under the reference's names; the arithmetic runs in the CUDA library
        conv_unit = (nn.Conv2d(in_size, out_size, kernel_size=(1, 1), bias=bias) if self._dims == 2
                     else nn.Conv1d(in_size, out_size, kernel_size=1, bias=bias))
        init(conv_unit.weight)
        if bias:
            nn.init.constant_(conv_unit.bias, 0)
        self._names = (name + "conv", name + self._bn_name)
        self.add_module(name + "conv", conv_unit)
        self.has_bn = bool(bn)
        if bn:
            self.add_module(name + self._bn_name, _BNWrap(out_size, self._bn_eps, self._bn_momentum, self._dims))
        if activation is not None:
            self.add_module(name + "activation", activation)
        self.act, self.slope = _act_code(activation)
        self._packed = None      # (weight version, PackedWeight, scale, shift) of the eval path
        self._split = None       # ((weight version, C1), fusion.SplitFuse) of forward_interp's eval path

    @property
    def _conv(self):
        return getattr(self, self._names[0])

    @property
    def _bn(self):
        return getattr(self, self._names[1]).bn if self.has_bn else None

    def _eval_version(self):
        conv, bn = self._conv, self._bn
        return (conv.weight._version, conv.weight.data_ptr(), bn.weight._version if bn is not None else 0,
                bn.running_mean._version if bn is not None else 0)

    def _eval_affine(self):
        """The folded BatchNorm (or the conv bias) as the GEMM epilogue's per-channel (scale, shift)."""
        conv, bn = self._conv, self._bn
        if bn is not None:
            return ops.fold_batchnorm(bn)
        scale = torch.ones(conv.weight.shape[0], device=conv.weight.device)
        return scale, (conv.bias.detach().float() if conv.bias is not None else torch.zeros_like(scale))

    def _eval_pack(self):
        ver = self._eval_version()
        if self._packed is None or self._packed[0] != ver:
            scale, shift = self._eval_affine()
            self._packed = (ver, ops.fusion_mlp_pack(self._conv.weight.detach()), scale, shift)
        return self._packed[1:]

    def _bn_sync(self):
        """``(process group, world size)`` when the training-mode BatchNorm normalises with the statistics of every
        rank, decided as ``nn.SyncBatchNorm.forward`` does: the layer is training, its BatchNorm is an
        ``nn.SyncBatchNorm``, torch.distributed is initialised, and the group (``process_group``, or WORLD) has more
        than one rank.  None otherwise: the layer's own batch, today's kernels."""
        bn = self._bn
        if not (self.training and isinstance(bn, nn.SyncBatchNorm) and dist.is_available() and dist.is_initialized()):
            return None
        group = bn.process_group if bn.process_group is not None else dist.group.WORLD
        world = dist.get_world_size(group)
        return (group, world) if world > 1 else None

    def _train_momentum(self, x, sync=None):
        """Training-mode BatchNorm bookkeeping before a forward, as nn.BatchNorm2d does it: rejects one value per
        channel (unless synchronised over several ranks, as nn.SyncBatchNorm), counts the batch, returns the momentum
        to update the running statistics with."""
        bn = self._bn
        if sync is None and x.shape[0] * math.prod(x.shape[2:]) == 1:     # as torch's BatchNorm in training
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (torch.Size((x.shape[0], bn.num_features) + tuple(x.shape[2:])),))
        if bn.track_running_stats and bn.num_batches_tracked is not None:
            bn.num_batches_tracked += 1
        momentum = bn.momentum
        if momentum is None:     # cumulative moving average, as nn.BatchNorm2d(momentum=None)
            momentum = 1.0 / float(bn.num_batches_tracked) if bn.num_batches_tracked is not None else 0.0
        return momentum

    def _frozen_bn_act(self, z):
        """Eval-mode BatchNorm and the activation as differentiable elementwise torch ops."""
        bn = self._bn
        y = F_.batch_norm(z, bn.running_mean, bn.running_var, bn.weight, bn.bias, False, 0.0, bn.eps)
        if self.act == _ACT_RELU:
            return torch.relu(y)
        return F_.leaky_relu(y, self.slope) if self.act == _ACT_LEAKY else y

    def forward(self, x, x2=None):
        if self._dims == 1:     # [B, C, N] layers run as [B, C, N, 1]
            return self._forward(x.unsqueeze(3), x2.unsqueeze(3) if x2 is not None else None).squeeze(3)
        return self._forward(x, x2)

    def _forward(self, x, x2=None):
        conv, bn = self._conv, self._bn
        need_grad = torch.is_grad_enabled() and (x.requires_grad or conv.weight.requires_grad or
                                                 (x2 is not None and x2.requires_grad))
        if self.training and bn is not None:
            sync = self._bn_sync()
            momentum = self._train_momentum(x, sync)
            return _ConvBnActTrain.apply(x, x2, conv.weight, None, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                         bn.eps, momentum, self.act, self.slope, True, sync)
        if need_grad and bn is None:
            return _ConvBnActTrain.apply(x, x2, conv.weight, conv.bias, None, None, None, None, 0.0, 0.0, self.act,
                                         self.slope, False)
        if need_grad:
            # eval-mode BatchNorm under autograd (fine-tuning with frozen statistics): GEMM with its backward,
            # then the per-channel affine and the activation as differentiable elementwise torch ops
            z = _ConvBnActTrain.apply(x, x2, conv.weight, None, None, None, None, None, 0.0, 0.0, _ACT_NONE, 0.0, False)
            return self._frozen_bn_act(z)
        packed, scale, shift = self._eval_pack()
        return ops.fusion_mlp(x, x2, packed, scale, shift, relu=(self.act == _ACT_RELU),
                              negative_slope=self.slope if self.act == _ACT_LEAKY else None)


class Conv2d(_ConvBase):
    """``pt_utils.Conv2d`` of FFB6D's fusion layers (models/pytorch_utils.py:168-201), 1x1 only.
    State-dict keys: ``conv.weight``, ``normlayer.bn.{weight,bias,running_mean,running_var,num_batches_tracked}``."""

    def __init__(self, in_size, out_size, kernel_size=(1, 1), stride=(1, 1), padding=(0, 0), dilation=(1, 1),
                 activation=nn.ReLU(inplace=True), bn=False, init=nn.init.kaiming_normal_, bias=True, preact=False, name=""):
        if preact or tuple(stride) != (1, 1) or tuple(padding) != (0, 0) or tuple(dilation) != (1, 1):
            raise ValueError("only plain 1x1 layers (no preact / stride / padding / dilation) are implemented here")
        super().__init__(in_size, out_size, kernel_size, activation, bn, init, bias, name)

    def forward_interp(self, x1, p, interp_idx):
        """``self(x1, nearest_interpolation(p, interp_idx).view(B, -1, h, w))`` without building the interpolated
        map (the pixel branch of FFB6D's fusion, models/ffb6d.py:246-253, 282-289, restructured as in SURVEY.md
        §8f-3): ``W . cat(x1, p[idx]) = W1 . x1 + (W2 . p)[idx]``.  The same three modes as ``forward``:

        * eval without autograd: :func:`ffb6d_b200.fusion.p2r_fuse` with the halves packed once per weight version;
        * training: batch-statistics BatchNorm (running statistics and ``num_batches_tracked`` updated as
          ``forward`` does), backward through the deterministic segment sum (``ffb6d_segment_sum``);
        * eval under autograd: the restructured GEMM with its backward, then the frozen BatchNorm and the
          activation as torch ops.

        :param x1: ``[B, C1, h, w]``; :param p: ``[B, C2, N', 1]`` with C1 + C2 the layer's input width
        :param interp_idx: ``[B, h*w, 1]`` (or ``[B, h*w]``) int32 / int64, values in ``[0, N')``
        :return: ``[B, Co, h, w]``"""
        conv, bn = self._conv, self._bn
        ops._need_cuda(x1, "x1")
        ops._need_cuda(p, "p")
        ops._need_cuda(interp_idx, "interp_idx")
        if x1.dim() != 4 or p.dim() != 4 or p.shape[3] != 1 or p.shape[0] != x1.shape[0]:
            raise ValueError("forward_interp expects x1 [B,C1,h,w] and p [B,C2,N',1], got %s and %s"
                             % (tuple(x1.shape), tuple(p.shape)))
        B, C1, h, w = x1.shape
        if C1 + p.shape[1] != conv.weight.shape[1]:
            raise ValueError("the layer takes %d input channels, x1 and p have %d + %d"
                             % (conv.weight.shape[1], C1, p.shape[1]))
        if interp_idx.shape[0] != B or interp_idx.numel() != B * h * w:
            raise ValueError("interp_idx must be [B, h*w, 1] = [%d, %d, 1], got %s" % (B, h * w, tuple(interp_idx.shape)))
        idx = interp_idx.reshape(B, h * w)
        need_grad = torch.is_grad_enabled() and (x1.requires_grad or p.requires_grad or conv.weight.requires_grad)
        if self.training and bn is not None:
            sync = self._bn_sync()
            momentum = self._train_momentum(x1, sync)
            return _InterpConvBnActTrain.apply(x1, p, idx, conv.weight, None, bn.weight, bn.bias, bn.running_mean,
                                               bn.running_var, bn.eps, momentum, self.act, self.slope, True, sync)
        if need_grad and bn is None:
            return _InterpConvBnActTrain.apply(x1, p, idx, conv.weight, conv.bias, None, None, None, None, 0.0, 0.0,
                                               self.act, self.slope, False)
        if need_grad:
            z = _InterpConvBnActTrain.apply(x1, p, idx, conv.weight, None, None, None, None, None, 0.0, 0.0, _ACT_NONE,
                                            0.0, False)
            return self._frozen_bn_act(z)
        key = (self._eval_version(), C1)
        if self._split is None or self._split[0] != key:
            scale, shift = self._eval_affine()
            self._split = (key, fusion.SplitFuse.from_weight(
                conv.weight, scale, shift, C1, relu=(self.act == _ACT_RELU),
                negative_slope=self.slope if self.act == _ACT_LEAKY else None))
        return fusion.p2r_fuse(x1, p, idx, self._split[1])


class RandLAConv2d(_ConvBase):
    """RandLA's ``pt_utils.Conv2d`` (models/RandLA/pytorch_utils.py:163-197), 1x1 only.
    State-dict keys: ``conv.weight``, ``bn.bn.{weight,bias,running_mean,running_var,num_batches_tracked}``."""
    _bn_name = "bn"
    _bn_eps, _bn_momentum = 1e-6, 0.99

    def __init__(self, in_size, out_size, *, kernel_size=(1, 1), stride=(1, 1), padding=(0, 0),
                 activation=nn.LeakyReLU(negative_slope=0.2, inplace=True), bn=False, init=nn.init.kaiming_normal_,
                 bias=True, preact=False, name="", instance_norm=False):
        if preact or instance_norm or tuple(stride) != (1, 1) or tuple(padding) != (0, 0):
            raise ValueError("only plain 1x1 layers are implemented here")
        super().__init__(in_size, out_size, kernel_size, activation, bn, init, bias, name)


class Conv1d(_ConvBase):
    """``pt_utils.Conv1d`` of FFB6D's prediction heads (models/pytorch_utils.py:132-165), kernel size 1: input
    ``[B, C, N]``.  State-dict keys as :class:`Conv2d` (``conv.weight`` is ``[Co, Ci, 1]``)."""
    _dims = 1

    def __init__(self, in_size, out_size, kernel_size=1, stride=1, padding=0, dilation=1,
                 activation=nn.ReLU(inplace=True), bn=False, init=nn.init.kaiming_normal_, bias=True, preact=False, name=""):
        if preact or stride != 1 or padding != 0 or dilation != 1:
            raise ValueError("only plain kernel-size-1 layers are implemented here")
        super().__init__(in_size, out_size, kernel_size, activation, bn, init, bias, name)


class RandLAConv1d(_ConvBase):
    """RandLA's ``pt_utils.Conv1d`` (``fc0`` of the network, models/RandLA/RandLANet.py:16), kernel size 1."""
    _dims = 1
    _bn_name = "bn"
    _bn_eps, _bn_momentum = 1e-6, 0.99

    def __init__(self, in_size, out_size, *, kernel_size=1, stride=1, padding=0,
                 activation=nn.LeakyReLU(negative_slope=0.2, inplace=True), bn=False, init=nn.init.kaiming_normal_,
                 bias=True, preact=False, name="", instance_norm=False):
        if preact or instance_norm or stride != 1 or padding != 0:
            raise ValueError("only plain kernel-size-1 layers are implemented here")
        super().__init__(in_size, out_size, kernel_size, activation, bn, init, bias, name)


# ----------------------------------------------------------------------------------------- RandLA blocks
class _AttPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f1, f2, att):
        out = ops.att_pool(f1, f2, att)
        ctx.save_for_backward(f1.contiguous(), f2.contiguous() if f2 is not None else None, att.contiguous())
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        f1, f2, att = ctx.saved_tensors
        B, C1, N, K = f1.shape
        C2 = f2.shape[1] if f2 is not None else 0
        g = gout.contiguous()
        gf1, gatt = torch.empty_like(f1), torch.empty_like(att)
        gf2 = torch.empty_like(f2) if f2 is not None else None
        with torch.cuda.device(f1.device):
            check(lib.ffb6d_att_pool_bwd(f1.data_ptr(), C1, f2.data_ptr() if f2 is not None else None, C2, att.data_ptr(),
                                         g.data_ptr(), B, N, K, gf1.data_ptr(), gf2.data_ptr() if gf2 is not None else None,
                                         gatt.data_ptr(), ops._stream(f1.device)))
        return gf1, gf2, gatt


def _gather_cm(feature, neigh_idx):
    """feature [B,C,N,1] -> neighbours channel-major [B,C,N,K]: ``gather_neighbour`` + ``permute(0,3,1,2)``
    (RandLANet.py:200-203) as one K = 1 gather (differentiable)."""
    B, N, K = neigh_idx.shape
    g = ops.nearest_interpolation(feature, neigh_idx.reshape(B, N * K, 1))
    return g.reshape(B, feature.shape[1], N, K)


class Att_pooling(nn.Module):
    """models/RandLA/RandLANet.py:237-250.  ``forward(feature_set)`` as the reference, or
    ``forward(f_neighbours, f_xyz)`` = the same on their concat without materialising it."""

    def __init__(self, d_in, d_out):
        super().__init__()
        self.fc = nn.Conv2d(d_in, d_in, (1, 1), bias=False)
        self.mlp = RandLAConv2d(d_in, d_out, kernel_size=(1, 1), bn=True)
        self._fc_pack = None

    def _att(self, f1, f2):
        w = self.fc.weight
        if torch.is_grad_enabled() and (w.requires_grad or f1.requires_grad or (f2 is not None and f2.requires_grad)):
            return _ConvBnActTrain.apply(f1, f2, w, None, None, None, None, None, 0.0, 0.0, _ACT_NONE, 0.0, False)
        ver = (w._version, w.data_ptr())
        if self._fc_pack is None or self._fc_pack[0] != ver:
            self._fc_pack = (ver, ops.fusion_mlp_pack(w.detach()))
        one, zero = _ones_zeros(w.shape[0], f1.device)
        return ops.fusion_mlp(f1, f2, self._fc_pack[1], one, zero, relu=False)

    def forward(self, feature_set, f2=None):
        att = self._att(feature_set, f2)
        if torch.is_grad_enabled() and att.requires_grad:
            f_agg = _AttPool.apply(feature_set, f2, att)
        else:
            f_agg = ops.att_pool(feature_set, f2, att)
        return self.mlp(f_agg)


class Building_block(nn.Module):
    """models/RandLA/RandLANet.py:187-214 (local spatial encoding + two attentive poolings)."""

    def __init__(self, d_out):
        super().__init__()
        self.mlp1 = RandLAConv2d(10, d_out // 2, kernel_size=(1, 1), bn=True)
        self.att_pooling_1 = Att_pooling(d_out, d_out // 2)
        self.mlp2 = RandLAConv2d(d_out // 2, d_out // 2, kernel_size=(1, 1), bn=True)
        self.att_pooling_2 = Att_pooling(d_out, d_out)

    def forward(self, xyz, feature, neigh_idx):
        f_xyz = ops.relative_pos_encoding(xyz, neigh_idx, channel_major=True)     # [B,10,N,K]
        f_xyz = self.mlp1(f_xyz)
        f_pc_agg = self.att_pooling_1(_gather_cm(feature, neigh_idx), f_xyz)
        f_xyz = self.mlp2(f_xyz)
        return self.att_pooling_2(_gather_cm(f_pc_agg, neigh_idx), f_xyz)

    relative_pos_encoding = staticmethod(ops.relative_pos_encoding)
    gather_neighbour = staticmethod(ops.gather_neighbour)


class Dilated_res_block(nn.Module):
    """models/RandLA/RandLANet.py:170-184."""

    def __init__(self, d_in, d_out):
        super().__init__()
        self.mlp1 = RandLAConv2d(d_in, d_out // 2, kernel_size=(1, 1), bn=True)
        self.lfa = Building_block(d_out)
        self.mlp2 = RandLAConv2d(d_out, d_out * 2, kernel_size=(1, 1), bn=True, activation=None)
        self.shortcut = RandLAConv2d(d_in, d_out * 2, kernel_size=(1, 1), bn=True, activation=None)

    def forward(self, feature, xyz, neigh_idx):
        if not self.training and not torch.is_grad_enabled():
            from . import randla
            return randla.dilated_res_block(self.state_dict(), "", feature, xyz, neigh_idx)   # fused residual GEMM
        f_pc = self.mlp1(feature)
        f_pc = self.lfa(xyz, f_pc, neigh_idx)
        f_pc = self.mlp2(f_pc)
        shortcut = self.shortcut(feature)
        return F_.leaky_relu(f_pc + shortcut, negative_slope=0.2)
