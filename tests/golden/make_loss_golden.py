#!/usr/bin/env python
"""Generate tests/golden/loss_cases.npz by running the reference's own models/loss.py on the CPU.

Source of truth: ``FocalLoss``, ``of_l1_loss`` and ``OFLoss`` of the reference's models/loss.py, executed from its
source text (the file imports only torch and numpy), and the loss block of ``model_fn`` (train_ycb.py:237-253,
train_lm.py) written around them.  Nothing of the reference is copied: only seeded inputs and the reference's
outputs are stored.

Cases, each under a ``kind:name:`` prefix:
* ``focal`` -- logits, labels, gamma, alpha (``alpha_kind`` 0 none, 1 float, 2 list), size_average, the upstream
  gradient ``g``; outputs ``loss`` and the autograd ``grad`` of the logits.  YCB (C = 22) and LineMOD (C = 2)
  shapes, gamma 0 / 0.5 / 2, ``size_average=False``, float and list alpha, an ``[M,C]`` input, a 4-D input,
  logits of +-80 and all-equal rows.
* ``of`` -- pred ``[B,K,N,3]``, targ ``[B,N,K,3]`` (or ``[B,N,3]`` for K = 1), labels, upstream ``g [B,K]``; outputs
  ``out [B,K]`` and ``grad``.  n_kps 8 and 16, a frame without positive labels, exact-zero differences, N not a
  multiple of 128, ``[B,N,1]`` labels.
* ``model`` -- whole loss blocks: the full batch's end_points and item arrays with a ``valid`` mask; the reference
  runs on the sub-batch ``x[valid]`` and its five info values and the gradients of the end_points (zero on masked
  frames) are stored.

Run:  python tests/golden/make_loss_golden.py      (needs /root/reference; rewrites loss_cases.npz)
"""
import io
import os
import sys
import warnings
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader as R                                  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "loss_cases.npz")


def reference_loss_module():
    path = os.path.join(R.REF_ROOT, "ffb6d", "models", "loss.py")
    ns = {"__name__": "reference_loss"}
    with open(path) as f:
        exec(compile(f.read(), path, "exec"), ns)
    return ns


def t32(a, grad=False):
    return torch.tensor(np.asarray(a, np.float32), requires_grad=grad)


def focal_case(ns, data, name, logits, labels, gamma, alpha=None, size_average=True, g=1.0):
    x = t32(logits, True)
    loss = ns["FocalLoss"](gamma=gamma, alpha=alpha, size_average=size_average)(x, torch.as_tensor(labels).long()
                                                                                  .view(-1))
    loss.backward(torch.tensor(g, dtype=torch.float32))
    p = "focal:%s:" % name
    data[p + "logits"] = np.asarray(logits, np.float32)
    data[p + "labels"] = np.asarray(labels, np.int64)
    data[p + "gamma"] = np.float64(gamma)
    data[p + "alpha_kind"] = np.int64(0 if alpha is None else (1 if np.isscalar(alpha) else 2))
    data[p + "alpha"] = np.asarray([0.0] if alpha is None else ([alpha] if np.isscalar(alpha) else alpha), np.float64)
    data[p + "size_average"] = np.int64(size_average)
    data[p + "g"] = np.float32(g)
    data[p + "loss"] = np.float32(loss.detach().numpy())
    data[p + "grad"] = x.grad.numpy()


def of_case(ns, data, name, pred, targ, labels, g):
    p_t = t32(pred, True)
    out = ns["OFLoss"]()(p_t, t32(targ), torch.as_tensor(labels).long())
    out.backward(t32(g))
    p = "of:%s:" % name
    data[p + "pred"] = np.asarray(pred, np.float32)
    data[p + "targ"] = np.asarray(targ, np.float32)
    data[p + "labels"] = np.asarray(labels, np.int32)
    data[p + "g"] = np.asarray(g, np.float32)
    data[p + "out"] = out.detach().numpy()
    data[p + "grad"] = p_t.grad.numpy()


def model_case(ns, data, name, rs, B, C, K, N, valid):
    valid = np.asarray(valid, bool)
    segs = (rs.randn(B, C, N) * 2).astype(np.float32)
    kp = rs.randn(B, K, N, 3).astype(np.float32)
    ctr = rs.randn(B, 1, N, 3).astype(np.float32)
    labels = rs.randint(0, C, (B, N)).astype(np.int32)
    labels[rs.rand(B, N) < 0.5] = 0
    kp_t = rs.randn(B, N, K, 3).astype(np.float32)
    ctr_t = rs.randn(B, N, 3).astype(np.float32)
    v = torch.from_numpy(valid)
    ep = {k: t32(a[valid], True) for k, a in (("pred_rgbd_segs", segs), ("pred_kp_ofs", kp), ("pred_ctr_ofs", ctr))}
    lab = torch.from_numpy(labels)[v].long()
    # model_fn's loss block (train_ycb.py:237-253) on the sub-batch of valid frames
    loss_rgbd_seg = ns["FocalLoss"](gamma=2)(ep["pred_rgbd_segs"], lab.view(-1)).sum()
    loss_kp_of = ns["OFLoss"]()(ep["pred_kp_ofs"], torch.from_numpy(kp_t)[v], lab).sum()
    loss_ctr_of = ns["OFLoss"]()(ep["pred_ctr_ofs"], torch.from_numpy(ctr_t)[v], lab).sum()
    loss = sum([ls * w for ls, w in [(loss_rgbd_seg, 2.0), (loss_kp_of, 1.0), (loss_ctr_of, 1.0)]])
    _, cls_rgbd = torch.max(ep["pred_rgbd_segs"], 1)
    acc = (cls_rgbd == lab).float().sum() / lab.numel()
    loss.backward()
    p = "model:%s:" % name
    for k, a in (("pred_rgbd_segs", segs), ("pred_kp_ofs", kp), ("pred_ctr_ofs", ctr), ("labels", labels),
                 ("kp_targ_ofst", kp_t), ("ctr_targ_ofst", ctr_t), ("valid", valid)):
        data[p + k] = a
    for k, t in (("loss_rgbd_seg", loss_rgbd_seg), ("loss_kp_of", loss_kp_of), ("loss_ctr_of", loss_ctr_of),
                 ("loss_all", loss), ("acc_rgbd", acc)):
        data[p + k] = np.float32(t.detach().numpy())
    for k in ep:
        full = np.zeros(data[p + k].shape, np.float32)
        full[valid] = ep[k].grad.numpy()
        data[p + "grad_" + k] = full


def cases():
    ns = reference_loss_module()
    data = {}
    rs = np.random.RandomState(20261016)
    # focal loss
    focal_case(ns, data, "ycb", rs.randn(2, 22, 300) * 3, rs.randint(0, 22, (2, 300)), 2)
    focal_case(ns, data, "lm", rs.randn(3, 2, 257) * 3, rs.randint(0, 2, (3, 257)), 2, g=0.7)
    focal_case(ns, data, "gamma0_sum", rs.randn(2, 5, 70), rs.randint(0, 5, (2, 70)), 0, size_average=False)
    focal_case(ns, data, "gamma05", rs.randn(2, 22, 90) * 2, rs.randint(0, 22, (2, 90)), 0.5)
    focal_case(ns, data, "alpha_float", rs.randn(2, 2, 130) * 2, rs.randint(0, 2, (2, 130)), 2, alpha=0.25)
    focal_case(ns, data, "alpha_list", rs.randn(2, 22, 60) * 2, rs.randint(0, 22, (2, 60)), 2,
               alpha=[float(a) for a in rs.rand(22)], size_average=False, g=1.3)
    focal_case(ns, data, "rows", rs.randn(190, 22) * 2, rs.randint(0, 22, 190), 2)
    focal_case(ns, data, "image", rs.randn(2, 22, 6, 7) * 2, rs.randint(0, 22, (2, 6, 7)), 2)
    ext = rs.choice([-80.0, 80.0], (1, 22, 100))
    ext[0, :, :20] = 0.0                                      # all-equal rows: the arg-max is class 0
    ext[0, :, 20:40] = 80.0
    ext[0, :5, 40:60] = 80.0                                  # ties between the first classes
    focal_case(ns, data, "extreme", ext, rs.randint(0, 22, (1, 100)), 2)
    # offset L1
    lab = rs.randint(0, 22, (2, 250))
    lab[rs.rand(2, 250) < 0.4] = 0
    of_case(ns, data, "ycb_k8", rs.randn(2, 8, 250, 3), rs.randn(2, 250, 8, 3), lab, rs.randn(2, 8))
    of_case(ns, data, "lm_k16", rs.randn(3, 16, 131, 3), rs.randn(3, 131, 16, 3), rs.randint(0, 2, (3, 131)),
            rs.randn(3, 16))
    lab = rs.randint(0, 22, (2, 130))
    lab[1] = 0                                                # a frame without positive labels
    of_case(ns, data, "no_positive", rs.randn(2, 8, 130, 3), rs.randn(2, 130, 8, 3), lab, np.ones((2, 8)))
    targ = rs.randn(2, 70, 8, 3).astype(np.float32)
    pred = rs.randn(2, 8, 70, 3).astype(np.float32)
    same = rs.rand(2, 8, 70, 3) < 0.5
    pred[same] = targ.transpose(0, 2, 1, 3)[same]             # exact-zero differences
    pred[0, 0, :4] = -0.0
    targ[0, :4, 0] = 0.0
    of_case(ns, data, "zero_diff", pred, targ, rs.randint(0, 3, (2, 70)), rs.randn(2, 8))
    of_case(ns, data, "ctr", rs.randn(2, 1, 200, 3), rs.randn(2, 200, 3), rs.randint(0, 22, (2, 200)), np.ones((2, 1)))
    of_case(ns, data, "labels_3d", rs.randn(1, 8, 129, 3), rs.randn(1, 129, 8, 3), rs.randint(0, 2, (1, 129, 1)),
            rs.randn(1, 8))
    # model_fn loss blocks
    model_case(ns, data, "lm_masked", rs, 4, 2, 8, 140, [1, 0, 1, 1])
    model_case(ns, data, "ycb", rs, 3, 22, 8, 131, [1, 1, 1])
    model_case(ns, data, "ycb_masked", rs, 3, 22, 8, 131, [0, 1, 0])
    return data


def main():
    if not R.reference_sources_present():
        raise SystemExit("needs the reference's sources (FFB6D_REFERENCE)")
    warnings.simplefilter("ignore")                           # log_softmax without dim, _Loss(size_average)
    torch.manual_seed(0)
    data = cases()
    # fixed member order and timestamps, so the file is reproducible byte for byte
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(data):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(data[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k.replace(":", "/") + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
