"""``FFB6DFusionNet``: everything of ``FFB6D.forward`` (models/ffb6d.py:203-337) except the ResNet/PSPNet
image backbone, on this package's kernels and with the reference's module names.

The reference interleaves two branches: a CNN producing ``rgb_emb0`` at every stage (cuDNN, out of this
repository's scope, SURVEY.md §2.1) and RandLA-Net on the points, tied together after every stage by the
bidirectional fusion layers.  This module owns the RandLA branch (``rndla_pre_stages``, ``rndla_ds_stages``,
``rndla_up_stages``), all 28 fusion layers (``{ds,up}_fuse_{r2p,p2r}_{pre,fuse}_layers``) and the three
prediction heads (``rgbd_seg_layer``, ``kp_ofst_layer``, ``ctr_ofst_layer``) under the reference's attribute
names, so the matching part of a published FFB6D checkpoint loads with ``load_state_dict(..., strict=False)``.
The image branch enters through ``rgb_feats``: the eight tensors the CNN stages would produce
(``cnn_ds_stages[i](...)`` x4, ``cnn_up_stages[i](...)`` x3, and the final full-resolution map); with
``rgb_stage_fn`` a caller can instead run its own CNN stage on the fused map, exactly where the reference does.

Used by ``tools/train_bench.py`` for BASELINE configs 3-4 (forward + backward under DDP, synthetic data).

``FFB6D`` is the whole network: ``FFB6DFusionNet`` plus the ResNet34-PSPNet image branch of :mod:`ffb6d_b200.cnn`
driven through ``rgb_stage_fn``, with every name of the reference's state dict (``load_reference_checkpoint`` loads
its trainer's checkpoints with ``strict=True``).
"""
import os

import torch
import torch.nn as nn

from . import cnn, ops
from . import tables as T
from .modules import Conv1d, Conv2d, Dilated_res_block, RandLAConv1d, RandLAConv2d


def _head(in_c, out_c):
    """``pt_utils.Seq(in_c).conv1d(128, bn).conv1d(128, bn).conv1d(128, bn).conv1d(out_c, activation=None)``
    (models/ffb6d.py:133-155); children are named "0".."3" like ``Seq`` names them."""
    seq = nn.Sequential()
    c = in_c
    for i in range(3):
        seq.add_module(str(i), Conv1d(c, 128, bn=True, activation=nn.ReLU()))
        c = 128
    seq.add_module("3", Conv1d(c, out_c, activation=None))
    return seq


class FFB6DFusionNet(nn.Module):
    def __init__(self, n_classes=2, n_pts=12288, n_kps=8, in_c=9, d_out=(32, 64, 128, 256), restructured=False,
                 fused_lfa=False):
        """``restructured``: run the pixel branch of every fusion as ``W1 . rgb + (W2 . p2r)[idx]``
        (:meth:`ffb6d_b200.modules.Conv2d.forward_interp`) instead of the reference's order of operations; the
        interpolated maps are never built.  A plain attribute: it can be switched on a built or loaded model, and
        the state dict is the same either way.

        ``fused_lfa``: when the encoder's ``Dilated_res_block`` s run under autograd or in training mode, the gather,
        ``fc`` and softmax pooling of each attentive pooling whose shape the fused kernels cover (K = 16, d/2 in
        {16, 32, 64}: encoder levels 0-2) run on them (:meth:`ffb6d_b200.modules.Building_block.forward`, DESIGN.md
        §4.19).  A plain attribute like ``restructured``; off by default."""
        super().__init__()
        self.n_cls, self.n_pts, self.n_kps = n_classes, n_pts, n_kps
        self.restructured = bool(restructured)
        self.fused_lfa = bool(fused_lfa)
        # RandLA branch (models/RandLA/RandLANet.py:12-38)
        self.rndla_pre_stages = RandLAConv1d(in_c, 8, kernel_size=1, bn=True)
        self.rndla_ds_stages = nn.ModuleList()
        d_in = 8
        for d in d_out:
            self.rndla_ds_stages.append(Dilated_res_block(d_in, d))
            d_in = 2 * d
        self.rndla_up_stages = nn.ModuleList()
        d_o = d_in
        for j in range(len(d_out)):
            if j < 3:
                d_i = d_o + 2 * d_out[-j - 2]
                d_o = 2 * d_out[-j - 2]
            else:
                d_i = 4 * d_out[-4]
                d_o = 2 * d_out[-4]
            self.rndla_up_stages.append(RandLAConv2d(d_i, d_o, kernel_size=(1, 1), bn=True))
        # fusion layers (models/ffb6d.py:49-80, 89-129)
        self.ds_rgb_oc, self.ds_rndla_oc = list(T.DS_RGB_OC), [2 * d for d in d_out]
        self.up_rgb_oc = list(T.UP_RGB_OC)
        self.up_rndla_oc = [self.ds_rndla_oc[-j - 2] if j < 3 else self.ds_rndla_oc[0] for j in range(len(d_out))]
        for tag, rgb_oc, rnd_oc, n in (("ds", self.ds_rgb_oc, self.ds_rndla_oc, 4), ("up", self.up_rgb_oc, self.up_rndla_oc, 3)):
            r2p_pre, r2p_fuse, p2r_pre, p2r_fuse = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
            for i in range(n):
                r2p_pre.append(Conv2d(rgb_oc[i], rnd_oc[i], kernel_size=(1, 1), bn=True))
                r2p_fuse.append(Conv2d(rnd_oc[i] * 2, rnd_oc[i], kernel_size=(1, 1), bn=True))
                p2r_pre.append(Conv2d(rnd_oc[i], rgb_oc[i], kernel_size=(1, 1), bn=True))
                p2r_fuse.append(Conv2d(rgb_oc[i] * 2, rgb_oc[i], kernel_size=(1, 1), bn=True))
            setattr(self, tag + "_fuse_r2p_pre_layers", r2p_pre)
            setattr(self, tag + "_fuse_r2p_fuse_layers", r2p_fuse)
            setattr(self, tag + "_fuse_p2r_pre_layers", p2r_pre)
            setattr(self, tag + "_fuse_p2r_fuse_layers", p2r_fuse)
        c = self.up_rndla_oc[-1] + self.up_rgb_oc[-1]
        self.rgbd_seg_layer = _head(c, n_classes)
        self.ctr_ofst_layer = _head(c, 3)
        self.kp_ofst_layer = _head(c, n_kps * 3)

    def _fuse(self, tag, i, rgb_emb0, p_emb0, p2r_idx, r2p_idx):
        """One bidirectional fusion (models/ffb6d.py:245-263 / 281-298): the reference's order of operations, or
        with ``restructured`` the pixel branch without the interpolated map."""
        bs, c, hr, wr = rgb_emb0.shape
        p2r = getattr(self, tag + "_fuse_p2r_pre_layers")[i](p_emb0)
        if self.restructured:
            rgb_emb = getattr(self, tag + "_fuse_p2r_fuse_layers")[i].forward_interp(rgb_emb0, p2r, p2r_idx)
        else:
            p2r = ops.nearest_interpolation(p2r, p2r_idx).view(bs, -1, hr, wr)
            rgb_emb = getattr(self, tag + "_fuse_p2r_fuse_layers")[i](rgb_emb0, p2r)      # concat fused in the layer
        r2p = ops.random_sample(rgb_emb0.reshape(bs, c, hr * wr, 1), r2p_idx)
        r2p = getattr(self, tag + "_fuse_r2p_pre_layers")[i](r2p)
        p_emb = getattr(self, tag + "_fuse_r2p_fuse_layers")[i](p_emb0, r2p)
        return rgb_emb, p_emb

    def forward(self, inputs, rgb_feats=None, rgb_stage_fn=None):
        """``inputs``: the reference's dict (``cld_rgb_nrm [B,9,N]``, ``cld_xyz{i}``, the index tensors of
        :func:`ffb6d_b200.schedule.build_ffb6d_indices`, ``choose [B,1,N]``).  ``rgb_feats``: the 8 CNN stage
        outputs, or ``rgb_stage_fn(stage_index, fused_rgb_emb_or_None) -> rgb_emb0`` to compute them on the fly.
        Returns the reference's ``end_points`` keys ``pred_rgbd_segs``, ``pred_kp_ofs``, ``pred_ctr_ofs`` plus
        ``fused_rgb`` (the fused image maps of the seven stages, inputs of the caller's next CNN stage)."""
        def rgb_stage(j, prev):
            return rgb_stage_fn(j, prev) if rgb_stage_fn is not None else rgb_feats[j]

        p_emb = self.rndla_pre_stages(inputs["cld_rgb_nrm"]).unsqueeze(3)            # [B,8,N,1]
        rgb_emb = None
        ds_emb, fused_rgb = [], []
        for i in range(4):
            rgb_emb0 = rgb_stage(i, rgb_emb)
            f_enc = self.rndla_ds_stages[i](p_emb, inputs["cld_xyz%d" % i], inputs["cld_nei_idx%d" % i],
                                            fused_lfa=self.fused_lfa)
            p_emb0 = ops.random_sample(f_enc, inputs["cld_sub_idx%d" % i])
            if i == 0:
                ds_emb.append(f_enc)
            rgb_emb, p_emb = self._fuse("ds", i, rgb_emb0, p_emb0, inputs["p2r_ds_nei_idx%d" % i],
                                        inputs["r2p_ds_nei_idx%d" % i])
            ds_emb.append(p_emb)
            fused_rgb.append(rgb_emb)
        n_up = len(self.rndla_up_stages)
        for i in range(n_up - 1):
            rgb_emb0 = rgb_stage(4 + i, rgb_emb)
            f_interp = ops.nearest_interpolation(p_emb, inputs["cld_interp_idx%d" % (n_up - i - 1)])
            p_emb0 = self.rndla_up_stages[i](ds_emb[-i - 2], f_interp)                   # cat fused in the layer
            rgb_emb, p_emb = self._fuse("up", i, rgb_emb0, p_emb0, inputs["p2r_up_nei_idx%d" % i],
                                        inputs["r2p_up_nei_idx%d" % i])
            fused_rgb.append(rgb_emb)
        rgb_emb = rgb_stage(7, rgb_emb)
        f_interp = ops.nearest_interpolation(p_emb, inputs["cld_interp_idx0"])
        p_emb = self.rndla_up_stages[n_up - 1](ds_emb[0], f_interp).squeeze(-1)        # [B,64,N]
        bs, di = rgb_emb.shape[0], rgb_emb.shape[1]
        rgb_emb_c = ops.choose_gather(rgb_emb, inputs["choose"])                      # [B,64,N]
        # heads: the first layer takes the concat as two inputs (no materialised cat)
        outs = []
        for head in (self.rgbd_seg_layer, self.kp_ofst_layer, self.ctr_ofst_layer):
            x = head[0](rgb_emb_c, p_emb)
            for layer in list(head)[1:]:
                x = layer(x)
            outs.append(x)
        rgbd_segs, pred_kp_ofs, pred_ctr_ofs = outs
        pred_kp_ofs = pred_kp_ofs.view(bs, self.n_kps, 3, -1).permute(0, 1, 3, 2).contiguous()
        pred_ctr_ofs = pred_ctr_ofs.view(bs, 1, 3, -1).permute(0, 1, 3, 2).contiguous()
        # `fused_rgb`: the seven fused image maps the reference hands to its next CNN stage (models/ffb6d.py:251, 287)
        return {"pred_rgbd_segs": rgbd_segs, "pred_kp_ofs": pred_kp_ofs, "pred_ctr_ofs": pred_ctr_ofs,
                "fused_rgb": fused_rgb}

    @staticmethod
    def rgb_feature_shapes(batch, h=480, w=640):
        """Shapes of the 8 ``rgb_feats`` (models/ffb6d.py:31-43, 84-87)."""
        shapes = [(batch, T.DS_RGB_OC[i], h // T.RGB_DS_SR[i], w // T.RGB_DS_SR[i]) for i in range(4)]
        shapes += [(batch, T.UP_RGB_OC[i], h // T.RGB_UP_SR[i], w // T.RGB_UP_SR[i]) for i in range(3)]
        shapes.append((batch, T.UP_RGB_OC[2], h, w))
        return shapes


class FFB6D(FFB6DFusionNet):
    """The whole network of models/ffb6d.py: :class:`FFB6DFusionNet` plus the ResNet34-PSPNet image branch
    (:mod:`ffb6d_b200.cnn`) under the reference's names ``cnn_pre_stages``, ``cnn_ds_stages`` and ``cnn_up_stages``, so
    a reference checkpoint loads with ``strict=True`` (:func:`load_reference_checkpoint`).

    ``forward(inputs)`` takes the reference's dict with ``inputs['rgb'] [B,3,H,W]`` float and returns its
    ``end_points`` (plus ``fused_rgb``, as :class:`FFB6DFusionNet`).  The image branch runs where the reference runs
    it: stage 0 is ``cnn_ds_stages[0](cnn_pre_stages(rgb))``, stages 1-3 take the previous fused map through
    ``cnn_ds_stages[j]``, stages 4-7 through ``cnn_up_stages[j - 4]``.

    * Training mode, or whenever autograd needs the image branch: its torch modules (cuDNN, batch statistics, active
      dropout), as the reference.
    * Eval mode without autograd: the PSP head (:meth:`ffb6d_b200.cnn.PSPModule.forward_fused`) and both uses of
      ``final`` (:meth:`ffb6d_b200.cnn.Final.forward_fused`) run on this package's kernels; the trunk and (unless
      ``fused_upsample``) the ``PSPUpsample`` stages stay on cuDNN.
    * ``fused_image_head=True`` (a plain attribute like ``restructured``; it may be switched on a built or loaded
      model and does not change the state dict): whenever autograd needs the image branch, the PSP head, the x2
      upsampling of ``up_1`` / ``up_2`` / ``up_3`` and both uses of ``final`` run their ``forward_fused`` paths,
      whose backwards are this package's kernels (DESIGN.md §4.18).  Their backwards add in a fixed order, so the
      whole network trains under ``torch.use_deterministic_algorithms(True)``, where torch's adaptive-average-pool
      and bilinear-upsampling backwards raise.  The trunk, the 3x3 convs, BatchNorms and PReLUs of ``PSPUpsample``
      and the dropouts stay torch modules (the CUDA RNG is drawn as on the torch path).  Off by default.
    * ``fused_upsample=True`` (a plain attribute like ``fused_image_head``, independent of it): ``up_1``, ``up_2`` and
      ``up_3`` run :meth:`ffb6d_b200.cnn.PSPUpsample.forward_restructured` -- upsampling, 3x3 conv, BatchNorm and
      PReLU on this package's kernels at the input's resolution (DESIGN.md §4.23) -- in training and in eval, with
      or without autograd.  ``drop_2`` stays torch's.  Off by default.
    * ``fused_lfa``: as :class:`FFB6DFusionNet`."""

    def __init__(self, n_classes, n_pts=12288, n_kps=8, restructured=False, fused_image_head=False, fused_lfa=False,
                 fused_upsample=False):
        super().__init__(n_classes=n_classes, n_pts=n_pts, n_kps=n_kps, restructured=restructured,
                         fused_lfa=fused_lfa)
        self.cnn_pre_stages, self.cnn_ds_stages, self.cnn_up_stages = cnn.image_branch()
        self.fused_image_head = bool(fused_image_head)
        self.fused_upsample = bool(fused_upsample)

    def _image_needs_grad(self, rgb):
        return torch.is_grad_enabled() and (rgb.requires_grad or any(
            p.requires_grad for m in (self.cnn_pre_stages, self.cnn_ds_stages, self.cnn_up_stages) for p in m.parameters()))

    def forward(self, inputs, end_points=None):
        rgb = inputs["rgb"]
        needs_grad = self._image_needs_grad(rgb)
        fused = not self.training and not needs_grad
        train_fused = self.fused_image_head and needs_grad
        final = self.cnn_up_stages[2][0]
        up = self.cnn_up_stages
        fused_up = self.fused_upsample

        def upsample(m, prev):
            if fused_up:
                return m.forward_restructured(prev)
            return m.forward_fused(prev) if train_fused else m(prev)

        def stage(j, prev):
            if j == 0:
                return self.cnn_ds_stages[0](self.cnn_pre_stages(rgb))
            if train_fused and j == 3:
                psp, drop_1 = self.cnn_ds_stages[3]
                return drop_1(psp.forward_fused(prev))
            if (train_fused or fused_up) and j in (4, 5):
                ups, drop_2 = up[j - 4]
                return drop_2(upsample(ups, prev))
            if (train_fused or fused) and j == 6:
                return final.forward_fused(prev)
            if (train_fused or fused) and j == 7:
                return final.forward_fused(upsample(up[3][0], prev))             # up_3, then final
            if fused_up and j == 7:
                return final(upsample(up[3][0], prev))
            if fused and j == 3:
                return self.cnn_ds_stages[3][0].forward_fused(prev)              # psp (+ drop_1, identity in eval)
            return (self.cnn_ds_stages[j] if j < 4 else self.cnn_up_stages[j - 4])(prev)

        out = super().forward(inputs, rgb_stage_fn=stage)
        if end_points is not None:
            end_points.update(out)
            return end_points
        return out


def load_reference_checkpoint(model, path_or_dict):
    """Load what the reference's training script saves (train_ycb.py:130-178) into ``model`` with ``strict=True``:
    a path to a ``torch.save``'d checkpoint or the object itself, either ``{'model_state': state_dict, ...}`` or a bare
    state dict, with or without the ``module.`` prefix of a (Distributed)DataParallel model.  Returns the result of
    ``load_state_dict``."""
    ck = path_or_dict
    if isinstance(ck, (str, os.PathLike)):
        ck = torch.load(ck, map_location="cpu", weights_only=False)
    if isinstance(ck, dict) and "model_state" in ck:
        ck = ck["model_state"]
    if ck is None:
        raise ValueError("the checkpoint holds no model_state")
    keys = list(ck.keys())
    if keys and all(k.startswith("module.") for k in keys):
        ck = {k[len("module."):]: v for k, v in ck.items()}
    return model.load_state_dict(ck, strict=True)
