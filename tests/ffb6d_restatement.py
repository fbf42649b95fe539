"""Plain-torch restatements of ``FFB6D.forward`` (models/ffb6d.py:203-337) that the GPU tests compare the package's
network with: :class:`TorchRef` (the RandLA branch, the 28 fusion layers and the heads, image maps given) and
:class:`FullRef` (with the image branch).  Both are themselves held to the reference's own ``FFB6D`` by
tests/test_ffb6d_golden.py, stage by stage (``trace``), on the CPU."""
import copy
import re

import numpy as np
import torch
import torch.nn.functional as Fn

from oracle import lfa_oracle


class TorchRef:
    """The reference's forward with torch ops only (float64), parameters taken from a state dict by the
    reference's names.  ``train``: BatchNorm uses batch statistics, and ``after`` receives every BatchNorm's updated
    running statistics by state-dict key.  With ``trace`` set to a list, every stage appends ``(name, output)``
    under the name of the reference's module that computes it."""

    def __init__(self, sd, train, n_kps, dtype=torch.float64):
        self.p = {k: v.detach().to(dtype).requires_grad_(v.dtype.is_floating_point and "running" not in k)
                  for k, v in sd.items() if v.dtype.is_floating_point}
        self.train, self.n_kps, self.dtype = train, n_kps, dtype
        self.after, self.trace = {}, None

    def note(self, name, out):
        if self.trace is not None:
            self.trace.append((name, out))
        return out

    def conv(self, pre, x, bn_name, eps, act, slope=0.2, momentum=0.1):
        w = self.p[pre + ".conv.weight"]
        y = torch.einsum("oc,bc...->bo...", w.reshape(w.shape[0], -1), x)
        if pre + ".conv.bias" in self.p:
            y = y + self.p[pre + ".conv.bias"].view(1, -1, *([1] * (y.dim() - 2)))
        b = pre + "." + bn_name + ".bn."
        if b + "weight" in self.p:
            mean, var = self.p[b + "running_mean"].clone(), self.p[b + "running_var"].clone()
            y = Fn.batch_norm(y, mean, var, self.p[b + "weight"], self.p[b + "bias"], self.train, momentum, eps)
            if self.train:
                self.after[b + "running_mean"], self.after[b + "running_var"] = mean, var
        if act == "relu":
            y = torch.relu(y)
        elif act == "leaky":
            y = Fn.leaky_relu(y, slope)
        return y

    def fconv(self, pre, x):                        # fusion flavour
        return self.conv(pre, x, "normlayer", 1e-5, "relu")

    def rconv(self, pre, x, act="leaky"):           # RandLA flavour (RandLA/pytorch_utils.py:108)
        return self.conv(pre, x, "bn", 1e-6, act, momentum=0.99)

    @staticmethod
    def random_sample(feature, idx):                # models/ffb6d.py:159-177
        f = feature.squeeze(3) if feature.dim() == 4 else feature
        B, d, K = f.shape[0], f.shape[1], idx.shape[-1]
        g = torch.gather(f, 2, idx.reshape(B, 1, -1).expand(-1, d, -1).long())
        return g.reshape(B, d, -1, K).max(dim=3, keepdim=True)[0]

    @staticmethod
    def nearest(feature, idx):                      # :179-194
        f = feature.squeeze(3)
        B, d = f.shape[0], f.shape[1]
        return torch.gather(f, 2, idx.reshape(B, 1, -1).expand(-1, d, -1).long()).unsqueeze(3)

    def att_pool(self, pre, fs):                    # RandLANet.py:243-250
        w = self.p[pre + ".fc.weight"]
        agg = lfa_oracle.att_pool(fs, torch.einsum("oc,bcnk->bonk", w.reshape(w.shape[0], -1), fs))
        return self.rconv(pre + ".mlp", agg)

    def block(self, pre, feature, xyz, idx):        # RandLANet.py:170-234
        f_pc = self.rconv(pre + ".mlp1", feature)
        f_xyz = self.rconv(pre + ".lfa.mlp1", lfa_oracle.relative_pos_encoding(xyz, idx))
        agg = self.att_pool(pre + ".lfa.att_pooling_1", torch.cat([lfa_oracle.gather_cm(f_pc, idx), f_xyz], 1))
        f_xyz = self.rconv(pre + ".lfa.mlp2", f_xyz)
        agg = self.att_pool(pre + ".lfa.att_pooling_2", torch.cat([lfa_oracle.gather_cm(agg, idx), f_xyz], 1))
        return self.note(pre, Fn.leaky_relu(
            self.rconv(pre + ".mlp2", agg, None) + self.rconv(pre + ".shortcut", feature, None), 0.2))

    def fuse(self, tag, i, rgb0, p0, p2r_idx, r2p_idx):      # models/ffb6d.py:245-263
        bs, c, hr, wr = rgb0.shape
        names = ["%s_fuse_%s_layers.%d" % (tag, k, i) for k in ("p2r_pre", "p2r_fuse", "r2p_pre", "r2p_fuse")]
        p2r = self.nearest(self.note(names[0], self.fconv(names[0], p0)), p2r_idx).view(bs, -1, hr, wr)
        rgb = self.note(names[1], self.fconv(names[1], torch.cat((rgb0, p2r), 1)))
        r2p = self.random_sample(rgb0.reshape(bs, c, hr * wr, 1), r2p_idx)
        r2p = self.note(names[2], self.fconv(names[2], r2p))
        return rgb, self.note(names[3], self.fconv(names[3], torch.cat((p0, r2p), 1)))

    def rgb_stage(self, j, prev, rgb_feats):
        """The image map of stage ``j`` (0-3 ``cnn_ds_stages``, 4-7 ``cnn_up_stages``); here it is given."""
        return rgb_feats[j]

    def forward(self, inp, rgb_feats):
        p_emb = self.note("rndla_pre_stages", self.rconv("rndla_pre_stages", inp["cld_rgb_nrm"].to(self.dtype))).unsqueeze(3)
        rgb = None
        ds_emb, fused = [], []
        for i in range(4):
            rgb0 = self.rgb_stage(i, rgb, rgb_feats)
            f_enc = self.block("rndla_ds_stages.%d" % i, p_emb, inp["cld_xyz%d" % i].to(self.dtype), inp["cld_nei_idx%d" % i])
            p0 = self.random_sample(f_enc, inp["cld_sub_idx%d" % i])
            if i == 0:
                ds_emb.append(f_enc)
            rgb, p_emb = self.fuse("ds", i, rgb0, p0, inp["p2r_ds_nei_idx%d" % i], inp["r2p_ds_nei_idx%d" % i])
            ds_emb.append(p_emb)
            fused.append(rgb)
        for i in range(3):
            rgb0 = self.rgb_stage(4 + i, rgb, rgb_feats)
            f_interp = self.nearest(p_emb, inp["cld_interp_idx%d" % (3 - i)])
            p0 = self.note("rndla_up_stages.%d" % i,
                           self.rconv("rndla_up_stages.%d" % i, torch.cat([ds_emb[-i - 2], f_interp], 1)))
            rgb, p_emb = self.fuse("up", i, rgb0, p0, inp["p2r_up_nei_idx%d" % i], inp["r2p_up_nei_idx%d" % i])
            fused.append(rgb)
        rgb = self.rgb_stage(7, rgb, rgb_feats)
        f_interp = self.nearest(p_emb, inp["cld_interp_idx0"])
        p_emb = self.note("rndla_up_stages.3",
                          self.rconv("rndla_up_stages.3", torch.cat([ds_emb[0], f_interp], 1))).squeeze(-1)
        bs, di = rgb.shape[0], rgb.shape[1]
        rgb_c = torch.gather(rgb.view(bs, di, -1), 2, inp["choose"].expand(-1, di, -1).long())
        x0 = torch.cat([rgb_c, p_emb], 1)
        outs = []
        for head in ("rgbd_seg_layer", "kp_ofst_layer", "ctr_ofst_layer"):
            x = x0
            for j in range(3):
                x = self.conv("%s.%d" % (head, j), x, "normlayer", 1e-5, "relu")
            outs.append(self.conv("%s.3" % head, x, "normlayer", 1e-5, None))
        segs, kp, ctr = outs
        kp = kp.view(bs, self.n_kps, 3, -1).permute(0, 1, 3, 2).contiguous()
        ctr = ctr.view(bs, 1, 3, -1).permute(0, 1, 3, 2).contiguous()
        return {"pred_rgbd_segs": segs, "pred_kp_ofs": kp, "pred_ctr_ofs": ctr, "fused_rgb": fused}


class FullRef(TorchRef):
    """TorchRef with the image branch: float64 copies of the model's own ``cnn_*`` torch modules (``cnn``), run where
    models/ffb6d.py runs them (the reference's order of operations) on ``forward``'s second argument, the image.
    ``train``: the image branch is in training mode too, except its dropouts, which stay off.  ``dtype``: float64, or
    float32 for the yardstick of what float32 arithmetic in the reference's order reaches."""

    def __init__(self, model, sd, n_kps, train=False, dtype=torch.float64):
        super().__init__({k: v for k, v in sd.items() if not k.startswith("cnn_")}, train, n_kps, dtype=dtype)
        self.cnn = copy.deepcopy(model).to(dtype).train(train)
        self.cnn.load_state_dict({k: v.to(dtype) if v.dtype.is_floating_point else v for k, v in sd.items()})
        for m in self.cnn.modules():
            if isinstance(m, (torch.nn.Dropout, torch.nn.Dropout2d)):
                m.eval()

    def rgb_stage(self, j, prev, rgb):
        if j == 0:
            prev = self.note("cnn_pre_stages", self.cnn.cnn_pre_stages(rgb.to(self.dtype)))
        name = "cnn_ds_stages.%d" % j if j < 4 else "cnn_up_stages.%d" % (j - 4)
        return self.note(name, (self.cnn.cnn_ds_stages[j] if j < 4 else self.cnn.cnn_up_stages[j - 4])(prev))


def close(got, want, what, tol):
    got, want = got.detach().double().cpu().numpy(), want.detach().double().cpu().numpy()
    scale = max(np.abs(want).max(), 1e-6)
    err = np.abs(got - want).max()
    assert err <= tol * scale, "%s: max abs err %.3e at scale %.3e (%.2e relative)" % (what, err, scale, err / scale)


def unit(name):
    """The layer a parameter belongs to: its conv + BatchNorm unit in the point branch, the fusion layers and the
    heads; its residual block, PSP module, ``PSPUpsample`` or stem in the image branch.  Gradient errors are measured
    against the largest gradient norm of the layer: a BatchNorm bias gradient is a sum of terms that nearly cancel
    behind another BatchNorm, its own norm is no yardstick for round-off."""
    m = re.match(r"cnn_pre_stages|cnn_(?:ds|up)_stages(?:\.\d+)+", name)
    if m:
        return m.group(0)
    return name.rsplit(".conv.", 1)[0].rsplit(".normlayer.", 1)[0].rsplit(".bn.bn.", 1)[0].rsplit(".fc.", 1)[0]


def first_divergence(got, stored, seed, n, bound):
    """Walk the fixture's tensors ``stored`` (:func:`oracle.net_oracle.unpack`; the order in which the reference
    computes them) and compare those present in ``got {name: tensor}`` at the fixture's sampled positions.
    The error is the root mean square of the differences there as a fraction of the tensor's scale (its largest
    sampled value; the largest difference of a few hundred samples is too noisy a yardstick); ``bound(e32)`` is the
    largest allowed error, given the reference's own float32 error ``e32`` in the same measure.  Returns ``(first, rows)``: a message naming the first stage beyond
    its bound (None if there is none) and ``(error, e32, name)`` of every stage compared, in order."""
    from oracle.net_oracle import sample
    first, rows = None, []
    for name, e in stored.items():
        if name not in got:
            continue
        if tuple(got[name].shape) != e["shape"]:
            return "%s: shape %s, the reference's is %s" % (name, tuple(got[name].shape), e["shape"]), rows
        scale = max(np.abs(e["f64"]).max(), 1e-30)
        rms = np.sqrt(e["f64"].size)
        err = np.linalg.norm(sample(got[name], seed + e["k"], n) - e["f64"]) / rms / scale
        e32 = e["e32norm"] / rms / scale
        rows.append((float(err), float(e32), name))
        if first is None and not err <= bound(e32):
            first = "%s is the first stage that differs from the reference: %.3e of its scale %.3g (the reference's " \
                    "own float32: %.3e)" % (name, err, scale, e32)
    return first, rows
