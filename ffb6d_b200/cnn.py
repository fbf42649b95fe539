"""FFB6D's image branch in plain torch: the ResNet34 trunk (models/cnn/extractors.py) and the PSPNet head
(models/cnn/pspnet.py), grouped into the stages the reference's ``FFB6D`` registers (models/ffb6d.py:27-45, 80-88)
so that a published checkpoint loads by name.

What the reference's code does, and these modules therefore do too:

* No dilation: ``ResNet._make_layer`` never passes its ``dilation`` on, so with ``output_stride=32`` every 3x3 conv is
  undilated and layer3 / layer4 run at stride 1 on the 1/8 map.  Layers 2-4 open with a 1x1 ``downsample``.
* ``PSPModule`` upsamples its priors with ``align_corners=False`` (``F.upsample(mode='bilinear')``);
  ``PSPUpsample`` with ``align_corners=True``.
* ``final`` (1x1 conv + LogSoftmax over the channels) and ``drop_2`` are single modules used at two stages each.
* ResNet's ``avgpool`` / ``fc`` and PSPNet's ``final_seg`` / ``classifier`` are not part of FFB6D and do not exist here.
* Construction never downloads anything: there is no pretrained path.  The trunk is initialised as the reference's
  ResNet (conv ``normal_(0, sqrt(2 / n))`` with n = k*k*out_channels, BatchNorm 1 / 0), the head with torch's defaults.

The modules' ``forward`` is the reference's, on any device and dtype.  :meth:`PSPModule.forward_fused` and
:meth:`Final.forward_fused` are the same on this package's kernels (:func:`ffb6d_b200.ops.psp_bottleneck`,
:func:`ffb6d_b200.ops.conv1x1_log_softmax`); :class:`ffb6d_b200.model.FFB6D` takes them in eval mode.  They are
differentiable: under autograd their backward is the adjoint kernels of DESIGN.md §4.18, which add in a fixed order and
so follow ``torch.use_deterministic_algorithms(True)``, where torch's adaptive-average-pool and bilinear backwards
raise.  :meth:`PSPUpsample.forward_fused` is the module with its x2 upsampling's backward on
:func:`ffb6d_b200.ops.upsample_bilinear2d_bwd`.  ``FFB6D(fused_image_head=True)`` trains through all three.
:meth:`PSPUpsample.forward_restructured` runs the whole stage (upsampling, 3x3 conv, BatchNorm, PReLU) on the kernels at
the input's resolution, forward and backward (DESIGN.md §4.23); ``FFB6D(fused_upsample=True)`` takes it.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

PSP_SIZES = (1, 2, 3, 6)


class BasicBlock(nn.Module):
    """ResNet's basic residual block: two 3x3 convs with BatchNorm, identity or 1x1 ``downsample`` shortcut."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        shortcut = x if self.downsample is None else self.downsample(x)
        return self.relu(out + shortcut)


class ResNet34(nn.Module):
    """The trunk of ``resnet34()`` as FFB6D uses it: stem, then layers of 3, 4, 6 and 3 basic blocks; layer2
    halves the map, layer3 and layer4 keep it (output stride 8)."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.inplanes = 64
        self.layer1 = self._make_layer(64, 3, 1)
        self.layer2 = self._make_layer(128, 4, 2)
        self.layer3 = self._make_layer(256, 6, 1)
        self.layer4 = self._make_layer(512, 3, 1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

    def _make_layer(self, planes, blocks, stride):
        downsample = None
        if stride != 1 or self.inplanes != planes:
            downsample = nn.Sequential(nn.Conv2d(self.inplanes, planes, 1, stride=stride, bias=False),
                                       nn.BatchNorm2d(planes))
        layers = [BasicBlock(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes
        layers += [BasicBlock(planes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)


def _version(params):
    return tuple((p._version, p.data_ptr()) for p in params)


def _cached_pack(module, params, pack):
    """``pack()`` of the weights ``params``, reused while their versions and storage are unchanged, and made afresh
    while a CUDA graph is being captured (:func:`ffb6d_b200.modules.weight_cache`)."""
    from .modules import weight_cache
    return weight_cache(module, "_packed", _version(params), pack)


class PSPModule(nn.Module):
    """Pyramid pooling: per size s an ``AdaptiveAvgPool2d(s)`` + bias-free 1x1 conv, each upsampled back
    (``align_corners=False``), concatenated with the input, 1x1 ``bottleneck`` (with bias), ReLU."""

    def __init__(self, features, out_features=1024, sizes=PSP_SIZES):
        super().__init__()
        self.stages = nn.ModuleList([nn.Sequential(nn.AdaptiveAvgPool2d(output_size=(s, s)),
                                                   nn.Conv2d(features, features, 1, bias=False)) for s in sizes])
        self.bottleneck = nn.Conv2d(features * (len(sizes) + 1), out_features, 1)
        self.relu = nn.ReLU()
        self._packed = None      # (parameter versions, ops.PSPWeights) of forward_fused

    def forward(self, feats):
        h, w = feats.shape[2], feats.shape[3]
        priors = [F.interpolate(stage(feats), size=(h, w), mode="bilinear", align_corners=False)
                  for stage in self.stages] + [feats]
        return self.relu(self.bottleneck(torch.cat(priors, 1)))

    def forward_fused(self, feats):
        """The same on the package's kernels: one pooling pass, the stage convs folded into the bottleneck's blocks,
        and a bottleneck GEMM over the input's channels only whose epilogue adds the upsampled priors (DESIGN.md
        §4.17).  Differentiable (:class:`_PSPFused`, DESIGN.md §4.18); the output is the same either way."""
        from . import ops
        if tuple(tuple(st[0].output_size) for st in self.stages) != tuple((s, s) for s in PSP_SIZES):
            raise ValueError("forward_fused: the kernels pool at the sizes %s only" % (PSP_SIZES,))
        packed = _cached_pack(self, list(self.parameters()), lambda: ops.psp_pack(
            [st[1].weight for st in self.stages], self.bottleneck.weight, self.bottleneck.bias))
        params = [st[1].weight for st in self.stages] + [self.bottleneck.weight, self.bottleneck.bias]
        if _needs_grad(feats, params):
            return _PSPFused.apply(feats, packed, *params)
        return ops.psp_bottleneck(feats, ops.psp_pool(feats), packed)


def _needs_grad(x, params):
    return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))


class _PSPFused(torch.autograd.Function):
    """PSPModule on the kernels, with its backward (DESIGN.md §4.18).  With ``M_s = W_s C_s``, ``p_s = pool_s(x)``,
    ``T_s = M_s p_s`` and ``out = relu(W_f x + b + sum_s up_s(T_s))``:

    * ``grad_z`` and every ``dT_s`` in one launch (:func:`ops.psp_bottleneck_bwd`);
    * ``dW_f = sum_b grad_z x^T`` (:func:`modules._wgrad`, ordered under deterministic mode), ``db = sum grad_z``;
    * ``dM_s = sum_b dT_s p_s^T``, ``dW_s = dM_s C_s^T``, ``dC_s = W_s^T dM_s``, ``dp_s = M_s^T dT_s`` (small; fp64);
    * ``dx = W_f^T grad_z`` (the forward GEMM on the transposed block), then ``+= pool^T(dp)``
      (:func:`ops.psp_pool_bwd`)."""

    @staticmethod
    def forward(ctx, x, packed, c1, c2, c3, c6, weight, bias):
        from . import ops
        x = x.contiguous()
        pooled = ops.psp_pool(x)
        out = ops.psp_bottleneck(x, pooled, packed)
        ctx.save_for_backward(x, out, weight, c1, c2, c3, c6, *pooled)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        from . import modules, ops
        x, out, weight = ctx.saved_tensors[:3]
        cs, pooled = ctx.saved_tensors[3:7], ctx.saved_tensors[7:]
        B, C, H, W = x.shape
        Co = out.shape[1]
        gz, table, gsum = ops.psp_bottleneck_bwd(grad.contiguous(), out)
        w = weight.detach().reshape(Co, -1)
        gw, gcs, gp = [], [], []
        row = 0
        for i, (s, cw, p) in enumerate(zip(PSP_SIZES, cs, pooled)):
            n = s * s
            dT = table[row:row + B * n].view(B, n, Co).double()
            row += B * n
            ws, cm = w[:, i * C:(i + 1) * C].double(), cw.detach().reshape(C, C).double()
            dM = torch.einsum("bno,bcn->oc", dT, p.reshape(B, C, n).double())
            gw.append((dM @ cm.t()).float())
            gcs.append((ws.t() @ dM).float().reshape(cw.shape))
            gp.append(torch.einsum("oc,bno->bcn", ws @ cm, dT).float().reshape(B, C, s, s))
        gw.append(modules._wgrad(gz, x, None, B, Co, H * W))
        gweight = torch.cat(gw, 1).reshape(weight.shape)
        gbias = gsum.double().sum(0).float()
        gx = None
        if ctx.needs_input_grad[0]:
            gx = modules._gemm(gz, None, w[:, len(PSP_SIZES) * C:].t().contiguous()).reshape(x.shape)
            ops.psp_pool_bwd(gp, gx)
        return (gx, None, *gcs, gweight, gbias)


class PSPUpsample(nn.Module):
    """x2 bilinear upsampling (``align_corners=True``), 3x3 conv, BatchNorm, PReLU."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.conv = nn.Sequential(nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True),
                                  nn.Conv2d(in_channels, out_channels, 3, padding=1),
                                  nn.BatchNorm2d(out_channels), nn.PReLU())
        self._upconv_packed = None      # (weight version, ops.UpConvWeights) of forward_restructured

    def forward(self, x):
        return self.conv(x)

    def forward_fused(self, x):
        """The same modules, with the x2 upsampling's backward on :func:`ffb6d_b200.ops.upsample_bilinear2d_bwd`
        (torch's forward; a backward that adds in a fixed order).  The conv, BatchNorm and PReLU stay torch's."""
        from . import ops
        up, conv, bn, act = self.conv
        if up.mode != "bilinear" or not up.align_corners or up.size is not None:
            raise ValueError("forward_fused: bilinear upsampling with align_corners=True by a scale factor only")
        return act(bn(conv(ops.upsample_bilinear2d(x, up.scale_factor))))

    def forward_restructured(self, x):
        """The same on this package's kernels at the input's resolution, without the upsampled map (DESIGN.md §4.23):
        ``conv3x3(up(x)) + b = b + sum_t S_t(up(W_t x))``, the stacked GEMM ``[9 Co, Ci] . x`` and a tap epilogue
        (:func:`ffb6d_b200.ops.upsample_conv3x3`), the weight stacked and packed once per weight version.

        * training mode: :class:`_UpConvTrain`, batch-statistics BatchNorm (running statistics updated as
          ``nn.BatchNorm2d`` does; synchronised over the ranks after ``convert_sync_batchnorm``), PReLU, and a
          backward that adds in a fixed order;
        * eval under autograd: the conv with that backward (:class:`_UpConv`), then the module's BatchNorm and PReLU;
        * eval without autograd: one epilogue applies the folded BatchNorm and PReLU.

        Raises ``ValueError`` unless the module is x2 bilinear upsampling with ``align_corners=True``, a 3x3 conv with
        padding 1 and stride 1, and a PReLU with one weight."""
        from . import modules, ops
        up, conv, bn, act = self.conv
        if (up.mode != "bilinear" or not up.align_corners or up.size is not None or
                tuple(up.scale_factor if isinstance(up.scale_factor, tuple) else (up.scale_factor,) * 2) != (2.0, 2.0)):
            raise ValueError("forward_restructured: x2 bilinear upsampling with align_corners=True only")
        if (tuple(conv.kernel_size) != (3, 3) or tuple(conv.padding) != (1, 1) or tuple(conv.stride) != (1, 1) or
                tuple(conv.dilation) != (1, 1) or conv.groups != 1 or conv.padding_mode != "zeros"):
            raise ValueError("forward_restructured: a 3x3 conv with padding 1 and stride 1 only")
        if not isinstance(act, nn.PReLU) or act.weight.numel() != 1:
            raise ValueError("forward_restructured: nn.PReLU() with one weight only")
        ops._tensor(x, "x", shape=4)
        packed = modules.weight_cache(self, "_upconv_packed", _version([conv.weight]),
                                      lambda: ops.upconv_pack(conv.weight))
        if self.training:
            B, _, Hi, Wi = x.shape
            sync = modules.bn_sync(bn, True)
            momentum = modules.bn_train_momentum(bn, (B, conv.out_channels, 2 * Hi, 2 * Wi), sync)
            return _UpConvTrain.apply(x, packed, conv.weight, conv.bias, bn.weight, bn.bias, act.weight,
                                      bn.running_mean, bn.running_var, bn.eps, momentum, sync)
        if _needs_grad(x, list(self.parameters())):
            return act(bn(_UpConv.apply(x, packed, conv.weight, conv.bias)))
        scale, shift = ops.fold_batchnorm(bn)
        return ops.upsample_conv3x3(x, packed, conv.bias, scale, shift, act.weight)


def _upconv_bwd(ctx, dz, x, weight, packed):
    """``(dx, dW, db)`` of ``z = conv3x3(up(x)) + b`` from ``dz``, per chunk of output channels: the tap adjoint
    ``G = up^T(S_t^T dz)`` (:func:`ops.upconv_taps_bwd`), ``dW = sum_b G x^T`` (:func:`modules._wgrad`, ordered under
    deterministic mode) unstacked to ``[Co, Ci, 3, 3]``, ``dx += W_stack^T G`` (the forward GEMM with K = 9 Cc), and
    ``db`` the sum of ``dz`` (per-plane sums, then the frames in fp64)."""
    from . import modules, ops
    B, Ci, Hi, Wi = x.shape
    w = weight.detach().float()
    gx = gw = gb = None
    gws = []
    for co0, cc in packed.chunks:
        g = ops.upconv_taps_bwd(dz, co0, cc)                         # [B, 9 cc, Hi, Wi]
        if ctx.needs_input_grad[2]:
            gws.append(modules._wgrad(g, x, None, B, 9 * cc, Hi * Wi).view(3, 3, cc, Ci).permute(2, 3, 0, 1))
        if ctx.needs_input_grad[0]:
            part = modules._gemm(g, None, ops.upconv_stack(w, co0, cc).t().contiguous())
            gx = part if gx is None else gx.add_(part)
        del g
    if gws:
        gw = torch.cat(gws, 0).contiguous()
    if ctx.needs_input_grad[3]:
        gb = dz.sum(dim=(2, 3)).double().sum(0).float()
    return gx, gw, gb


class _UpConv(torch.autograd.Function):
    """``conv3x3(up(x)) + b`` of PSPUpsample on the kernels (:func:`ops.upsample_conv3x3`), with its backward
    (:func:`_upconv_bwd`).  Saves ``x`` only."""

    @staticmethod
    def forward(ctx, x, packed, weight, bias):
        from . import ops
        x = x.contiguous()
        ctx.packed = packed
        ctx.save_for_backward(x, weight)
        return ops.upsample_conv3x3(x, packed, bias)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        x, weight = ctx.saved_tensors
        gx, gw, gb = _upconv_bwd(ctx, grad.contiguous(), x, weight, ctx.packed)
        return gx, None, gw, gb


class _UpConvTrain(torch.autograd.Function):
    """PSPUpsample in training mode: ``z = conv3x3(up(x)) + b`` (:func:`ops.upsample_conv3x3`), BatchNorm with batch
    statistics (:func:`modules._bn_act_fwd`, SyncBatchNorm included), PReLU (:func:`ops.prelu_`, in place on the
    BatchNorm's output).  Saves ``x``, ``z`` and the BatchNorm's stats; the backward recomputes the PReLU's input
    (:func:`ops.bn_prelu_bwd`), then :func:`modules._bn_act_bwd` and :func:`_upconv_bwd`."""

    @staticmethod
    def forward(ctx, x, packed, weight, bias, gamma, beta, alpha, running_mean, running_var, eps, momentum, sync):
        from . import modules, ops
        x = x.contiguous()
        z = ops.upsample_conv3x3(x, packed, bias)
        B, Co, Ho, Wo = z.shape
        y, stats, count = modules._bn_act_fwd(z, B, Co, Ho * Wo, gamma, beta, running_mean, running_var, eps, momentum,
                                              modules._ACT_NONE, 0.0, True, sync)
        ops.prelu_(y, alpha)
        ctx.packed, ctx.sync = packed, sync
        ctx.save_for_backward(x, z, stats, count, weight, alpha)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        from . import modules, ops
        x, z, stats, count, weight, alpha = ctx.saved_tensors
        B, Co, Ho, Wo = z.shape
        gu, galpha = ops.bn_prelu_bwd(z, grad.contiguous(), stats, alpha)
        dz, ggamma, gbeta = modules._bn_act_bwd(z, gu, stats, B, Co, Ho * Wo, modules._ACT_NONE, 0.0, True, ctx.sync,
                                                count)
        del gu
        gx, gw, gb = _upconv_bwd(ctx, dz, x, weight, ctx.packed)
        return gx, None, gw, gb, ggamma, gbeta, galpha.reshape(alpha.shape), None, None, None, None, None


class Final(nn.Sequential):
    """PSPNet's ``final``: ``Conv2d(64, 64, 1)`` and a LogSoftmax over the channels (state-dict keys ``0.weight``,
    ``0.bias``)."""

    def __init__(self, channels=64):
        super().__init__(nn.Conv2d(channels, channels, 1), nn.LogSoftmax(dim=1))
        self._packed = None      # (parameter versions, ops.PackedWeight) of forward_fused

    def forward_fused(self, x):
        """The same in one kernel (``ffb6d_conv1x1_log_softmax_fwd``).  Differentiable (:class:`_FinalFused`); the
        output is the same either way."""
        from . import ops
        conv = self[0]
        packed = _cached_pack(self, (conv.weight, conv.bias), lambda: ops.fusion_mlp_pack(conv.weight.detach()))
        if _needs_grad(x, (conv.weight, conv.bias)):
            return _FinalFused.apply(x, packed, conv.weight, conv.bias)
        return ops.conv1x1_log_softmax(x, packed, conv.bias)


class _FinalFused(torch.autograd.Function):
    """``final`` on the kernel, with its backward: ``dz`` = the log-softmax backward (:func:`ops.log_softmax_bwd`),
    then ``dW = sum_b dz x^T`` (:func:`modules._wgrad`), ``db = sum dz`` and ``dx = W^T dz`` (the forward GEMM on
    the transposed weight).  ``final`` is used twice per step; autograd adds the two uses' gradients."""

    @staticmethod
    def forward(ctx, x, packed, weight, bias):
        from . import ops
        x = x.contiguous()
        out = ops.conv1x1_log_softmax(x, packed, bias)
        ctx.save_for_backward(x, out, weight)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        from . import modules, ops
        x, out, weight = ctx.saved_tensors
        B, Co = out.shape[0], out.shape[1]
        dz = ops.log_softmax_bwd(grad.contiguous(), out)
        gw = modules._wgrad(dz, x, None, B, Co, out.numel() // (B * Co)).reshape(weight.shape)
        # per-plane sums first: torch.sum(..., dtype=float64) would make a float64 copy of dz (1.3 GB at B = 8, 480x640)
        gb = dz.sum(dim=(2, 3)).double().sum(0).float()
        gx = None
        if ctx.needs_input_grad[0]:
            gx = modules._gemm(dz, None, weight.detach().reshape(Co, -1).t().contiguous()).reshape(x.shape)
        return gx, None, gw, gb


class PSPNet34(nn.Module):
    """The parts of ``PSPNet(psp_size=512, deep_features_size=256, backend='resnet34')`` that FFB6D uses."""

    def __init__(self):
        super().__init__()
        self.feats = ResNet34()
        self.psp = PSPModule(512, 1024, PSP_SIZES)
        self.drop_1 = nn.Dropout2d(p=0.3)
        self.up_1 = PSPUpsample(1024, 256)
        self.up_2 = PSPUpsample(256, 64)
        self.up_3 = PSPUpsample(64, 64)
        self.drop_2 = nn.Dropout2d(p=0.15)
        self.final = Final(64)


def image_branch():
    """``(cnn_pre_stages, cnn_ds_stages, cnn_up_stages)`` grouped as models/ffb6d.py:30-45, 83-88 groups them:

    * pre: conv1, bn1, relu, maxpool (1/4 resolution);
    * ds: layer1 (1/4), layer2 (1/8), ``Sequential(layer3, layer4)`` (1/8), ``Sequential(psp, drop_1)`` (1/8, 1024 ch);
    * up: ``Sequential(up_1, drop_2)`` (1/4), ``Sequential(up_2, drop_2)`` (1/2), ``Sequential(final)`` (1/2),
      ``Sequential(up_3, final)`` (full resolution); ``final`` and ``drop_2`` are the same modules at both stages."""
    cnn = PSPNet34()
    f = cnn.feats
    pre = nn.Sequential(f.conv1, f.bn1, f.relu, f.maxpool)
    ds = nn.ModuleList([f.layer1, f.layer2, nn.Sequential(f.layer3, f.layer4), nn.Sequential(cnn.psp, cnn.drop_1)])
    up = nn.ModuleList([nn.Sequential(cnn.up_1, cnn.drop_2), nn.Sequential(cnn.up_2, cnn.drop_2),
                        nn.Sequential(cnn.final), nn.Sequential(cnn.up_3, cnn.final)])
    return pre, ds, up
