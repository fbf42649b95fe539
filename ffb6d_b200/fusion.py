"""The bidirectional fusion stage of FFB6D on this package's kernels (inference, frozen BatchNorm; the training
form of the restructured pixel branch is :meth:`ffb6d_b200.modules.Conv2d.forward_interp`).

One stage of ``FFB6D.forward`` (models/ffb6d.py:231-263 encoder, :267-298 decoder) after the CNN /
RandLA layers of the stage have produced ``rgb_emb0 [B, C_r, h, w]`` and the point features::

    p_emb0  = random_sample(f_enc, cld_sub_idx)                        (encoder only, :240-241)
    p2r     = p2r_pre(p_emb0)                                          1x1 conv + BN + ReLU on N' points
    p2r     = nearest_interpolation(p2r, p2r_idx).view(B, -1, h, w)    K = 1 gather to every pixel
    rgb_emb = p2r_fuse(cat(rgb_emb0, p2r))                             1x1 conv over 2 C_r channels
    r2p     = random_sample(rgb_emb0.reshape(B, C_r, h*w, 1), r2p_idx) gather 16 + max from the image
    p_emb   = r2p_fuse(cat(p_emb0, r2p_pre(r2p)))

The pixel branch is restructured algebraically (SURVEY.md §8f-3): the conv is linear and the
interpolation is a selection, so with ``W = [W1 | W2]`` split at ``C_r``

    W . cat(rgb_emb0, p2r[idx]) = W1 . rgb_emb0 + (W2 . p2r)[idx].

``Z = W2 . p2r`` is a small product on the N' points; the big layer then runs over K = C_r only and adds
``Z[idx[pixel]]`` in its epilogue (:func:`ffb6d_b200.ops.fusion_mlp` with ``add=``).  The interpolated
map -- the largest gather of every stage -- is never materialised and the layer's FLOPs halve.
fp32 summation order differs from the reference's single K loop; results agree to ~1e-6 relative
(tests/test_gpu_fusion_stage.py).
"""
import torch

from . import ops


class FusedConv:
    """A fusion ``pt_utils.Conv2d`` (conv1x1 bias=False -> BatchNorm2d -> ReLU, models/pytorch_utils.py:75-129)
    prepared for inference: packed weights + folded BatchNorm."""

    def __init__(self, weight, scale, shift):
        w = weight.detach().reshape(weight.shape[0], -1).float()
        self.Co, self.Ci = int(w.shape[0]), int(w.shape[1])
        self.weight = w
        self.packed = ops.fusion_mlp_pack(w)
        self.scale, self.shift = scale.detach().float().contiguous(), shift.detach().float().contiguous()

    @classmethod
    def from_module(cls, conv2d):
        """From a reference ``pt_utils.Conv2d`` (children ``conv`` and ``normlayer.bn``) in eval mode."""
        scale, shift = ops.fold_batchnorm(conv2d.normlayer.bn)
        return cls(conv2d.conv.weight, scale, shift)

    def __call__(self, x1, x2=None):
        return ops.fusion_mlp(x1, x2, self.packed, self.scale, self.shift)


class SplitFuse:
    """``p2r_fuse`` split at the concat boundary: ``W1 = W[:, :C_r]`` (image half, keeps the BatchNorm and
    the activation) and ``W2 = W[:, C_r:]`` (point half, applied on the N' points, no affine, channels-last out).
    ``relu`` / ``negative_slope``: the activation, as :func:`ffb6d_b200.ops.fusion_mlp` takes it."""

    def __init__(self, fused, c_rgb, relu=True, negative_slope=None):
        self._setup(fused.weight, fused.scale, fused.shift, c_rgb, relu, negative_slope)

    @classmethod
    def from_weight(cls, weight, scale, shift, c_rgb, relu=True, negative_slope=None):
        """From a layer's ``conv.weight`` and its folded BatchNorm (``scale``, ``shift``)."""
        self = cls.__new__(cls)
        self._setup(weight.detach().reshape(weight.shape[0], -1).float(), scale, shift, c_rgb, relu, negative_slope)
        return self

    def _setup(self, w, scale, shift, c_rgb, relu, negative_slope):
        self.c_rgb = int(c_rgb)
        self.w1 = ops.fusion_mlp_pack(w[:, :c_rgb].contiguous())
        self.w2 = ops.fusion_mlp_pack(w[:, c_rgb:].contiguous())
        self.scale, self.shift = scale, shift
        self.ones = torch.ones_like(scale)
        self.zeros = torch.zeros_like(scale)
        self.relu, self.negative_slope = relu, negative_slope


def p2r_fuse(rgb_emb0, p2r, p2r_idx, split):
    """``p2r_fuse(cat(rgb_emb0, nearest_interpolation(p2r, p2r_idx).view(B,-1,h,w)))`` without the
    interpolated map (models/ffb6d.py:246-253, 282-289).

    :param rgb_emb0: ``[B, C_r, h, w]``; :param p2r: ``[B, C_r, N', 1]`` = ``p2r_pre(p_emb0)``
    :param p2r_idx: ``[B, h*w, 1]`` nearest cloud point of every pixel; :param split: :class:`SplitFuse`
    :return: ``[B, C_r, h, w]``"""
    z = ops.fusion_mlp(p2r, None, split.w2, split.ones, split.zeros, relu=False, out_channels_last=True)   # [B, N', C_r]
    return ops.fusion_mlp(rgb_emb0, None, split.w1, split.scale, split.shift, relu=split.relu,
                          negative_slope=split.negative_slope, add=z, add_idx=p2r_idx)


class FusionStage:
    """The four fusion layers of one stage (``*_fuse_r2p_pre``, ``*_fuse_r2p_fuse``, ``*_fuse_p2r_pre``,
    ``*_fuse_p2r_fuse``, models/ffb6d.py:55-80 / 104-129), each a :class:`FusedConv`."""

    def __init__(self, r2p_pre, r2p_fuse, p2r_pre, p2r_fuse_layer):
        self.r2p_pre, self.r2p_fuse, self.p2r_pre, self.p2r_fuse_layer = r2p_pre, r2p_fuse, p2r_pre, p2r_fuse_layer
        self.split = SplitFuse(p2r_fuse_layer, p2r_fuse_layer.Ci // 2)

    def __call__(self, rgb_emb0, p_emb0, p2r_idx, r2p_idx, restructured=True):
        """-> ``(rgb_emb [B,C_r,h,w], p_emb [B,C_p,N',1])`` of models/ffb6d.py:245-263 (= :281-298)."""
        B, C, h, w = rgb_emb0.shape
        p2r = self.p2r_pre(p_emb0)
        if restructured:
            rgb_emb = p2r_fuse(rgb_emb0, p2r, p2r_idx, self.split)
        else:   # the reference's order of operations, on the same kernels (A/B and parity checks)
            up = ops.nearest_interpolation(p2r, p2r_idx).view(B, -1, h, w)
            rgb_emb = self.p2r_fuse_layer(rgb_emb0, up)
        r2p = ops.random_sample(rgb_emb0.reshape(B, C, h * w, 1), r2p_idx)
        p_emb = self.r2p_fuse(p_emb0, self.r2p_pre(r2p))
        return rgb_emb, p_emb
