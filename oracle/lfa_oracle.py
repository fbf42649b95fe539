"""Plain-torch restatement of RandLA's local feature aggregation and of the 1x1 fusion layer, in float64 by default
(any dtype, CPU or GPU), from BatchNorm-folded ``(weight [Co, Ci], scale [Co], shift [Co])`` tuples: the arguments
``ffb6d_b200.ops.lfa_att_pool_fused`` and ``ops.fusion_mlp`` take.

One attentive pooling of ``Building_block`` (models/RandLA/RandLANet.py:196-250):
``relative_pos_encoding -> mlp1 [-> mlp2] -> cat(gathered features, f_xyz) -> fc -> softmax_K -> weighted sum -> mlp``.
``relative_pos_encoding``, ``gather_cm`` and ``att_pool`` are also the pieces of tests/test_gpu_model.py's whole-network
restatement, which keeps its BatchNorm unfolded (training statistics)."""
import torch

ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2      # the ``act`` codes of ffb6d_fusion_mlp_fwd_ex


def fold(sd, prefix, eps=1e-6):
    """``(w [Co, Ci], scale, shift)`` of a ``pt_utils.Conv2d`` with bn=True in float64 (RandLA's BatchNorm eps is
    1e-6, models/RandLA/pytorch_utils.py:108)."""
    w = sd[prefix + ".conv.weight"].double()
    bn = prefix + ".bn.bn."
    scale = sd[bn + "weight"].double() / torch.sqrt(sd[bn + "running_var"].double() + eps)
    return w.reshape(w.shape[0], -1), scale, sd[bn + "bias"].double() - sd[bn + "running_mean"].double() * scale


def activation(y, act, slope=0.0):
    if act == ACT_RELU:
        return torch.relu(y)
    if act == ACT_LEAKY:
        return torch.nn.functional.leaky_relu(y, slope)
    return y


def fusion_layer(x1, x2, weight, scale, shift, act=ACT_RELU, slope=0.0, add=None, add_idx=None, dtype=torch.float64):
    """``act(scale * (W cat(x1, x2) [+ add[b, add_idx[b, p], :]]) + shift)`` over ``[B, C, ...]`` inputs: the 1x1
    conv + folded BatchNorm + activation of ``ops.fusion_mlp``, with its epilogue addend (``add [B, NA, Co]``,
    ``add_idx [B, P]``).  Returns ``[B, Co, ...]``."""
    x = (torch.cat((x1, x2), 1) if x2 is not None else x1).to(dtype)
    w = weight.reshape(weight.shape[0], -1).to(dtype)
    y = torch.einsum("oc,bc...->bo...", w, x)
    if add is not None:
        B, Co = y.shape[:2]
        g = torch.gather(add.to(dtype), 1, add_idx.reshape(B, -1, 1).long().expand(-1, -1, Co))    # [B, P, Co]
        y = y + g.permute(0, 2, 1).reshape(y.shape)
    bshape = (1, -1) + (1,) * (y.dim() - 2)
    return activation(y * scale.to(dtype).view(bshape) + shift.to(dtype).view(bshape), act, slope)


def relative_pos_encoding(xyz, idx):
    """``[B, 10, N, K]`` channel-major: (distance, centre - neighbour, centre, neighbour) of ``xyz [B, N, 3]`` and its
    neighbours ``idx [B, N, K]`` (RandLANet.py:216-223), in ``xyz``'s dtype."""
    B, N, K = idx.shape
    nb = torch.gather(xyz, 1, idx.reshape(B, -1, 1).expand(-1, -1, 3).long()).reshape(B, N, K, 3)
    tile = xyz.unsqueeze(2).expand(-1, -1, K, -1)
    rel = tile - nb
    dis = torch.sqrt(torch.sum(rel ** 2, dim=-1, keepdim=True))
    return torch.cat([dis, rel, tile, nb], dim=-1).permute(0, 3, 1, 2)


def gather_cm(f, idx):
    """``f [B, C, N]`` or ``[B, C, N, 1]`` -> the neighbours' features ``[B, C, N, K]`` (gather_neighbour + permute)."""
    f = f.reshape(f.shape[0], f.shape[1], -1)
    B, d = f.shape[:2]
    N, K = idx.shape[1:]
    return torch.gather(f, 2, idx.reshape(B, 1, -1).expand(-1, d, -1).long()).reshape(B, d, N, K)


def att_pool(fs, att):
    """``sum_K fs * softmax_K(att)`` -> ``[B, C, N, 1]`` (RandLANet.py:245-248)."""
    return torch.sum(fs * torch.softmax(att, dim=3), dim=3, keepdim=True)


def encode(xyz, idx, feature, mlp1, mlp2, negative_slope=0.2, dtype=torch.float64):
    """``cat(gathered features, mlp2(mlp1(relative_pos_encoding)))`` ``[B, d, N, K]``: what the pooling's ``fc`` sees."""
    f_xyz = fusion_layer(relative_pos_encoding(xyz.to(dtype), idx), None, *mlp1, ACT_LEAKY, negative_slope, dtype=dtype)
    if mlp2 is not None:
        f_xyz = fusion_layer(f_xyz, None, *mlp2, ACT_LEAKY, negative_slope, dtype=dtype)
    return torch.cat((gather_cm(feature.to(dtype), idx), f_xyz), 1)


def lfa_att_pool(xyz, idx, feature, mlp1, mlp2, fc_weight, mlp_out, negative_slope=0.2, dtype=torch.float64):
    """One attentive pooling with the arguments of ``ops.lfa_att_pool_fused``: ``xyz [B, N, 3]``, ``idx [B, N, K]``,
    ``feature [B, d/2, N(, 1)]``, ``mlp2`` may be None.  Returns ``[B, d_out, N, 1]``."""
    f_cat = encode(xyz, idx, feature, mlp1, mlp2, negative_slope, dtype)
    fc = fc_weight.reshape(fc_weight.shape[0], -1).to(dtype)
    agg = att_pool(f_cat, torch.einsum("oc,bcnk->bonk", fc, f_cat))
    return fusion_layer(agg, None, *mlp_out, ACT_LEAKY, negative_slope, dtype=dtype)


def building_block(sd, prefix, xyz, feature, idx, dtype=torch.float64):
    """``Building_block.forward`` (RandLANet.py:196-214) from its state dict: ``feature [B, d/2, N, 1]`` -> ``[B, d, N, 1]``."""
    m1, m2 = fold(sd, prefix + ".mlp1"), fold(sd, prefix + ".mlp2")
    f = lfa_att_pool(xyz, idx, feature, m1, None, sd[prefix + ".att_pooling_1.fc.weight"],
                     fold(sd, prefix + ".att_pooling_1.mlp"), dtype=dtype)
    return lfa_att_pool(xyz, idx, f, m1, m2, sd[prefix + ".att_pooling_2.fc.weight"],
                        fold(sd, prefix + ".att_pooling_2.mlp"), dtype=dtype)


def dilated_res_block(sd, feature, xyz, idx, dtype=torch.float64):
    """``Dilated_res_block.forward`` (RandLANet.py:179-184): ``leaky(mlp2(lfa(mlp1(f))) + shortcut(f), 0.2)``."""
    f_pc = fusion_layer(feature, None, *fold(sd, "mlp1"), ACT_LEAKY, 0.2, dtype=dtype)
    f_pc = building_block(sd, "lfa", xyz, f_pc, idx, dtype)
    y = fusion_layer(f_pc, None, *fold(sd, "mlp2"), ACT_NONE, dtype=dtype) + \
        fusion_layer(feature, None, *fold(sd, "shortcut"), ACT_NONE, dtype=dtype)
    return activation(y, ACT_LEAKY, 0.2)
