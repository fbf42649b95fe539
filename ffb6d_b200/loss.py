"""FFB6D's training loss on the GPU: the names of the reference's ``models/loss.py`` (``FocalLoss``,
``of_l1_loss``, ``OFLoss``) and :func:`ffb6d_loss`, the loss block of ``model_fn`` (train_ycb.py:237-253,
train_lm.py), over the fused kernels of ``csrc/loss.cu``.

Every loss takes an optional ``valid [B]`` mask (``build_ffb6d_item``'s ``item["valid"]``).  A masked frame adds
nothing and gets zero gradients, so every value equals the reference's on the sub-batch ``x[valid]``, without
the host synchronisation and the changing shapes of boolean indexing: the loss, its backward and ``info`` can be
captured in a CUDA graph.  If every frame is masked, the losses and the accuracy are 0 and the gradients are 0
(the reference, given an empty batch, would divide by zero).

Each forward and each backward is one C call; all are deterministic, whether or not
``torch.use_deterministic_algorithms`` is on.
"""
import torch

from . import ops


class _FocalFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, valid, gamma, alpha, size_average, layout):
        loss, acc, count, lse = ops.focal_loss_fwd(logits, labels, valid, gamma, alpha, size_average, layout)
        ctx.save_for_backward(logits, labels, valid, alpha, lse, count)
        ctx.args = (gamma, size_average, layout)
        ctx.mark_non_differentiable(acc)
        return loss, acc

    @staticmethod
    def backward(ctx, grad_loss, _grad_acc):
        logits, labels, valid, alpha, lse, count = ctx.saved_tensors
        gamma, size_average, layout = ctx.args
        grad = ops.focal_loss_bwd(logits, labels, valid, gamma, alpha, size_average, lse, count, grad_loss, layout)
        return grad, None, None, None, None, None, None


class _OfL1Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, targ, labels, valid):
        out, count = ops.of_l1_loss_fwd(pred, targ, labels, valid)
        ctx.save_for_backward(pred, targ, labels, valid, count)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        pred, targ, labels, valid, count = ctx.saved_tensors
        return ops.of_l1_loss_bwd(pred, targ, labels, valid, count, grad_out.contiguous()), None, None, None


def _valid(valid, B, device):
    return None if valid is None else ops._loss_valid(valid, B, device)


class FocalLoss(torch.nn.Module):
    """``FocalLoss(gamma, alpha, size_average)`` of models/loss.py:12-43.  ``pt`` is a constant of the backward, as
    the reference's ``Variable(logpt.data.exp())``.

    :param alpha: None, a float / int (the weights ``[alpha, 1 - alpha]`` of classes 0 and 1) or a list of per-class
      weights; anything else raises.  It must have an entry for every class of the input.
    """

    def __init__(self, gamma=0, alpha=None, size_average=True):
        super().__init__()
        if isinstance(alpha, bool) or not (alpha is None or isinstance(alpha, (float, int, list))):
            raise TypeError("alpha must be None, a float or a list, got %r" % (type(alpha),))
        self.gamma = float(gamma)
        if isinstance(alpha, (float, int)):
            alpha = [alpha, 1 - alpha]
        self.alpha = None if alpha is None else [float(a) for a in alpha]
        self.size_average = size_average
        self._alpha_dev = {}

    def _alpha(self, device, C):
        if self.alpha is None:
            return None
        if len(self.alpha) < C:
            raise ValueError("alpha has %d entries, the input %d classes" % (len(self.alpha), C))
        if device not in self._alpha_dev:          # copied once per device, so later calls can be captured
            self._alpha_dev[device] = torch.tensor(self.alpha, dtype=torch.float32, device=device)
        return self._alpha_dev[device]

    def forward_acc(self, input, target, valid=None):
        """The loss and ``acc_rgbd`` (arg-max == label, lowest class on ties, over the counted points) of one call.

        :param input: ``[B,C,N...]`` logits (any trailing shape, flattened as the reference's ``view``) or ``[M,C]``
        :param target: the labels, ``B*N`` (or ``M``) int32 / int64 values in any shape (``labels.view(-1)``)
        :param valid: ``[B]`` frame mask, for a ``[B,C,N...]`` input
        """
        if input.dim() > 2:
            x, layout = input.reshape(input.shape[0], input.shape[1], -1), 0
        elif input.dim() == 2:
            if valid is not None:
                raise ValueError("valid needs a [B,C,N] input; an [M,C] input is one frame")
            x, layout = input.reshape(1, input.shape[0], input.shape[1]), 1
        else:
            raise ValueError("input must be [B,C,N...] or [M,C], got %s" % (tuple(input.shape),))
        B, C = x.shape[0], x.shape[2 if layout else 1]
        return _FocalFn.apply(x, target, _valid(valid, B, x.device), self.gamma, self._alpha(x.device, C),
                              bool(self.size_average), layout)

    def forward(self, input, target, valid=None):
        return self.forward_acc(input, target, valid)[0]


def of_l1_loss(pred_ofsts, kp_targ_ofst, labels, sigma=1.0, normalize=True, reduce=False, valid=None):
    """``of_l1_loss`` of models/loss.py:46-74: per-frame, per-keypoint mean of the L1 offset error over the points
    with ``labels > 0``, ``[bs, n_kpts]``, or its mean with ``reduce``.  ``sigma`` is unused, as in the reference.

    :param pred_ofsts: ``[bs, n_kpts, n_pts, 3]``; :param kp_targ_ofst: ``[bs, n_pts, n_kpts, 3]``
    :param labels: ``bs * n_pts`` int32 / int64 values (``[bs, n_pts]`` or ``[bs, n_pts, 1]``)
    :param valid: ``[bs]`` frame mask; a masked frame's row is 0, and ``reduce`` averages over the valid frames
    ``normalize=False`` (the unreduced ``[bs, n_kpts, n_pts, 3]`` map, which no trainer uses) has no kernel and raises.
    """
    if not normalize:
        raise NotImplementedError("of_l1_loss(normalize=False) is not implemented: OFLoss always normalises")
    v = _valid(valid, pred_ofsts.shape[0], pred_ofsts.device)
    out = _OfL1Fn.apply(pred_ofsts, kp_targ_ofst, labels, v)
    if reduce:
        if v is None:
            return out.mean()
        return out.sum() / (v.sum() * out.shape[1]).clamp_min(1).to(out.dtype)
    return out


class OFLoss(torch.nn.Module):
    """``OFLoss`` of models/loss.py:77-90: ``of_l1_loss`` with ``normalize=True, reduce=False`` whatever the
    arguments say, as the reference's forward does; returns ``[bs, n_kpts]``."""

    def forward(self, pred_ofsts, kp_targ_ofst, labels, normalize=True, reduce=False, valid=None):
        return of_l1_loss(pred_ofsts, kp_targ_ofst, labels, sigma=1.0, normalize=True, reduce=False, valid=valid)


_focal = FocalLoss(gamma=2)
_of = OFLoss()


def ffb6d_loss(end_points, item, valid=None, weights=(2.0, 1.0, 1.0)):
    """The loss block of ``model_fn`` (train_ycb.py:237-253, train_lm.py):
    ``w0 * FocalLoss(gamma=2)(segs, labels) + w1 * OFLoss(kp).sum() + w2 * OFLoss(ctr).sum()`` and ``acc_rgbd``.

    :param end_points: the network's outputs ``pred_rgbd_segs [B,C,N]``, ``pred_kp_ofs [B,n_kps,N,3]``,
      ``pred_ctr_ofs [B,1,N,3]``
    :param item: ``labels [B,N]``, ``kp_targ_ofst [B,N,n_kps,3]``, ``ctr_targ_ofst [B,N,3]`` (``build_ffb6d_item``'s)
    :param valid: ``[B]`` frame mask, e.g. ``item["valid"]`` as it is; None: every frame
    :return: ``(loss, info)``; ``info`` holds ``loss_rgbd_seg``, ``loss_kp_of``, ``loss_ctr_of``, ``loss_all`` and
      ``acc_rgbd`` as detached device scalars (call ``.item()`` to read one; nothing here synchronises the host)
    """
    labels = item["labels"]
    segs = end_points["pred_rgbd_segs"]
    v = _valid(valid, segs.shape[0], segs.device)
    loss_rgbd_seg, acc_rgbd = _focal.forward_acc(segs, labels, v)
    loss_kp_of = _of(end_points["pred_kp_ofs"], item["kp_targ_ofst"], labels, valid=v).sum()
    loss_ctr_of = _of(end_points["pred_ctr_ofs"], item["ctr_targ_ofst"], labels, valid=v).sum()
    loss = loss_rgbd_seg * weights[0] + loss_kp_of * weights[1] + loss_ctr_of * weights[2]
    info = {"loss_rgbd_seg": loss_rgbd_seg.detach(), "loss_kp_of": loss_kp_of.detach(),
            "loss_ctr_of": loss_ctr_of.detach(), "loss_all": loss.detach(), "acc_rgbd": acc_rgbd}
    return loss, info
