"""RandLA-Net local feature aggregation on the hot path's kernels (inference, frozen BatchNorm).

Functional mirrors of ``Att_pooling``, ``Building_block`` and ``Dilated_res_block``
(models/RandLA/RandLANet.py:170-250) that take the modules' ``state_dict()`` -- parameter names
are the reference's (``mlp1.conv.weight``, ``mlp1.bn.bn.running_mean``, ``lfa.att_pooling_1.fc.weight``
...), so published checkpoints work unchanged.  Every step is one of this package's CUDA kernels:

* 1x1 convs (+ BN(eps 1e-6) + LeakyReLU(0.2), RandLA's ``pt_utils.Conv2d``) -> ``fusion_mlp`` (wgmma),
  with the ``torch.cat`` in front of every attentive pooling fused as its two K ranges
* neighbour gathers (``gather_neighbour`` + ``permute(0,3,1,2).contiguous()``) -> the K = 1 gather
  kernel writing channel-major ``[B,C,N,K]`` directly
* ``relative_pos_encoding`` -> its kernel, channel-major
* softmax over K * features, summed over K -> ``att_pool``
* the residual ``leaky_relu(mlp2(f) + shortcut(x))`` -> ONE GEMM over the concatenated K ranges with
  BN-scaled weights and summed shifts.
"""
import torch

from . import ops


def _conv_bn(sd, prefix):
    """(weight [Co,Ci], scale, shift) of a RandLA ``pt_utils.Conv2d`` with bn=True, BN folded."""
    w = sd[prefix + ".conv.weight"]
    w = w.reshape(w.shape[0], -1)
    var, mean = sd[prefix + ".bn.bn.running_var"].float(), sd[prefix + ".bn.bn.running_mean"].float()
    scale = sd[prefix + ".bn.bn.weight"].float() / torch.sqrt(var + 1e-6)     # pytorch_utils.py:108: eps=1e-6
    shift = sd[prefix + ".bn.bn.bias"].float() - mean * scale
    return w, scale, shift


def _gather_cm(feature, neigh_idx):
    """feature [B,C,N,1] -> neighbours channel-major [B,C,N,K] (gather_neighbour + permute, :200-203)."""
    B, N, K = neigh_idx.shape
    g = ops.nearest_interpolation(feature, neigh_idx.reshape(B, N * K, 1))
    return g.reshape(B, feature.shape[1], N, K)


def att_pooling(sd, prefix, f1, f2):
    """``Att_pooling.forward`` on ``cat(f1, f2)`` (RandLANet.py:243-250): [B,C,N,K] x2 -> [B,d_out,N,1]."""
    fc = sd[prefix + ".fc.weight"]
    d = fc.shape[0]
    ones = torch.ones(d, device=f1.device)
    att = ops.fusion_mlp(f1, f2, fc, ones, torch.zeros_like(ones), relu=False)      # fc: conv, no bias
    agg = ops.att_pool(f1, f2, att)
    w, scale, shift = _conv_bn(sd, prefix + ".mlp")
    return ops.fusion_mlp(agg, None, w, scale, shift, negative_slope=0.2)


def building_block(sd, prefix, xyz, feature, neigh_idx, fused=True):
    """``Building_block.forward`` (RandLANet.py:196-214): xyz [B,N,3], feature [B,d/2,N,1],
    neigh_idx [B,N,K] -> [B,d,N,1].  With K = 16 and d/2 in {16, 32, 64} each attentive pooling is ONE fused
    kernel (``ops.lfa_att_pool_fused``: no [B,C,N,K] tensor touches HBM); other shapes, or ``fused=False``, run
    the per-op kernels below."""
    if fused and ops.lfa_fusable(feature.shape[1], neigh_idx.shape[2]):
        m1, m2 = _conv_bn(sd, prefix + ".mlp1"), _conv_bn(sd, prefix + ".mlp2")
        f_agg = ops.lfa_att_pool_fused(xyz, neigh_idx, feature, m1, None, sd[prefix + ".att_pooling_1.fc.weight"],
                                       _conv_bn(sd, prefix + ".att_pooling_1.mlp"))
        return ops.lfa_att_pool_fused(xyz, neigh_idx, f_agg, m1, m2, sd[prefix + ".att_pooling_2.fc.weight"],
                                      _conv_bn(sd, prefix + ".att_pooling_2.mlp"))
    f_xyz = ops.relative_pos_encoding(xyz, neigh_idx, channel_major=True)           # [B,10,N,K]
    w, scale, shift = _conv_bn(sd, prefix + ".mlp1")
    f_xyz = ops.fusion_mlp(f_xyz, None, w, scale, shift, negative_slope=0.2)
    f_agg = att_pooling(sd, prefix + ".att_pooling_1", _gather_cm(feature, neigh_idx), f_xyz)
    w, scale, shift = _conv_bn(sd, prefix + ".mlp2")
    f_xyz = ops.fusion_mlp(f_xyz, None, w, scale, shift, negative_slope=0.2)
    return att_pooling(sd, prefix + ".att_pooling_2", _gather_cm(f_agg, neigh_idx), f_xyz)


def dilated_res_block(sd, prefix, feature, xyz, neigh_idx, fused=True):
    """``Dilated_res_block.forward`` (RandLANet.py:179-184): feature [B,d_in,N,1] -> [B,2*d_out,N,1]."""
    p = prefix + "." if prefix else ""
    w, scale, shift = _conv_bn(sd, p + "mlp1")
    f_pc = ops.fusion_mlp(feature, None, w, scale, shift, negative_slope=0.2)
    f_pc = building_block(sd, p + "lfa", xyz, f_pc, neigh_idx, fused)
    # leaky_relu(mlp2(f_pc) + shortcut(feature)): one GEMM over [f_pc; feature] with BN-scaled weights
    w2, s2, b2 = _conv_bn(sd, p + "mlp2")
    ws, ss, bs = _conv_bn(sd, p + "shortcut")
    wcat = torch.cat((w2 * s2[:, None], ws * ss[:, None]), dim=1).contiguous()
    ones = torch.ones(wcat.shape[0], device=feature.device)
    return ops.fusion_mlp(f_pc, feature, wcat, ones, b2 + bs, negative_slope=0.2)
