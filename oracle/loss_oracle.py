"""oracle/loss_oracle.py -- TEST INFRASTRUCTURE ONLY.  FFB6D's training loss (models/loss.py:12-90, combined as in
train_ycb.py:237-253) restated twice:

* in float64 numpy, for the tests: ``focal_loss``, ``of_l1_loss`` and ``ffb6d_loss`` with the package's ``valid``
  semantics (every value equals the reference's on the sub-batch of valid frames; masked frames get zero gradients;
  no counted point gives 0), plus ``of_l1_grad_f32``, the reference's float32 autograd product for the offsets;
* in float32 torch ops as the reference writes them (``*_torch``), for the benchmark's comparator and the GPU
  tests; ``ffb6d_loss_torch`` takes the sub-batch by boolean indexing, as a trainer using the reference would.
"""
import numpy as np


# --------------------------------------------------------------------------- float64 numpy
def _rows(logits, labels, valid):
    """``[M,C]`` float64 rows (b-major, then n), their labels and the frame mask of a ``[B,C,N...]`` / ``[M,C]``
    input."""
    x = np.asarray(logits, np.float64)
    lab = np.asarray(labels).reshape(-1).astype(np.int64)
    if x.ndim == 2:
        return x, lab, None
    B, C = x.shape[:2]
    x = x.reshape(B, C, -1)
    v = np.ones(B, bool) if valid is None else np.asarray(valid, bool).reshape(B)
    lab = lab.reshape(B, -1)
    return x[v].transpose(0, 2, 1).reshape(-1, C), lab[v].reshape(-1), v


def focal_loss(logits, labels, gamma=0.0, alpha=None, size_average=True, valid=None, grad_loss=1.0):
    """``(loss, acc, grad)``: FocalLoss with ``pt`` detached, the arg-max accuracy (lowest class on ties) over the
    counted points, and the gradient of the logits for the upstream ``grad_loss``, in the input's shape.  A label
    outside ``[0, C)`` makes its term and its row of the gradient NaN."""
    x = np.asarray(logits, np.float64)
    rows, lab, v = _rows(logits, labels, valid)
    M, C = rows.shape
    if M == 0:
        return 0.0, 0.0, np.zeros(x.shape)
    inside = (lab >= 0) & (lab < C)
    t = np.where(inside, lab, 0)
    m = rows.max(1)
    lse = m + np.log(np.exp(rows - m[:, None]).sum(1))
    logpt = np.where(inside, rows[np.arange(M), t] - lse, np.nan)
    w = (1.0 - np.exp(logpt)) ** gamma
    at = np.ones(M)
    if alpha is not None:
        a = np.asarray([alpha, 1 - alpha] if np.isscalar(alpha) else alpha, np.float64)
        at = np.where(inside, a[np.minimum(t, len(a) - 1)], np.nan)
    term = -w * logpt * at
    loss = term.mean() if size_average else term.sum()
    acc = float((rows.argmax(1) == lab).sum()) / M
    gt = -w * at * (grad_loss / M if size_average else grad_loss)
    g = -np.exp(rows - lse[:, None]) * gt[:, None]
    g[np.arange(M), t] += np.where(inside, gt, np.nan)
    if v is None:
        return float(loss), acc, g
    B, Cx = x.shape[:2]
    full = np.zeros((B, Cx, x.reshape(B, Cx, -1).shape[2]))
    full[v] = g.reshape(int(v.sum()), -1, C).transpose(0, 2, 1)
    return float(loss), acc, full.reshape(x.shape)


def _of_parts(pred, targ, labels):
    bs, K, N, c = pred.shape
    w = (np.asarray(labels).reshape(bs, N) > 0)
    t = np.asarray(targ).reshape(bs, N, K, c).transpose(0, 2, 1, 3)
    return w, t


def of_l1_loss(pred, targ, labels, valid=None):
    """``[B,n_kps]``: ``sum_n sum_c w_n |pred - targ| / (cnt_b + 1e-3)`` in float64 (0 on masked frames)."""
    p = np.asarray(pred, np.float64)
    w, t = _of_parts(p, targ, labels)
    d = np.abs(p - t.astype(np.float64)) * w[:, None, :, None]
    den = w.sum(1).astype(np.float64) + np.float64(np.float32(1e-3))
    out = d.sum((2, 3)) / den[:, None]
    if valid is not None:
        out[~np.asarray(valid, bool)] = 0.0
    return out


def of_l1_grad_f32(pred, targ, labels, grad_out, valid=None):
    """The reference's autograd gradient of ``of_l1_loss`` in float32: ``(g / (cnt + 1e-3)) * w * sign(d)``."""
    p = np.asarray(pred, np.float32)
    w, t = _of_parts(p, targ, labels)
    d = p - t.astype(np.float32)
    den = w.sum(1).astype(np.float32) + np.float32(1e-3)
    gd = np.asarray(grad_out, np.float32) / den[:, None]
    sgn = (d > 0).astype(np.float32) - (d < 0).astype(np.float32)          # sign(0) = sign(-0) = +0, as torch's
    g = (gd[:, :, None, None] * w[:, None, :, None].astype(np.float32)) * sgn
    if valid is not None:
        g[~np.asarray(valid, bool)] = 0.0
    return g.astype(np.float32)


def ffb6d_loss(end_points, item, valid=None, weights=(2.0, 1.0, 1.0)):
    """float64 ``{loss_rgbd_seg, loss_kp_of, loss_ctr_of, loss_all, acc_rgbd}`` of model_fn's loss block."""
    lab = np.asarray(item["labels"])
    seg, acc, _ = focal_loss(end_points["pred_rgbd_segs"], lab, gamma=2, valid=valid)
    kp = of_l1_loss(end_points["pred_kp_ofs"], item["kp_targ_ofst"], lab, valid).sum()
    ctr = of_l1_loss(end_points["pred_ctr_ofs"], item["ctr_targ_ofst"], lab, valid).sum()
    return {"loss_rgbd_seg": seg, "loss_kp_of": kp, "loss_ctr_of": ctr,
            "loss_all": seg * weights[0] + kp * weights[1] + ctr * weights[2], "acc_rgbd": acc}


# --------------------------------------------------------------------------- float32 torch, as the reference
def focal_loss_torch(input, target, gamma=0.0, alpha=None, size_average=True):
    import torch
    import torch.nn.functional as F
    if input.dim() > 2:
        C = input.size(1)
        input = input.reshape(input.size(0), C, -1).transpose(1, 2).contiguous().view(-1, C)
    target = target.reshape(-1, 1).long()
    logpt = F.log_softmax(input, dim=1).gather(1, target).view(-1)
    pt = logpt.detach().exp()
    if alpha is not None:
        a = torch.tensor([alpha, 1 - alpha] if np.isscalar(alpha) else alpha, dtype=input.dtype, device=input.device)
        logpt = logpt * a.gather(0, target.view(-1))
    loss = -1 * (1 - pt) ** gamma * logpt
    return loss.mean() if size_average else loss.sum()


def of_l1_loss_torch(pred, targ, labels):
    bs, K, N, c = pred.size()
    w = (labels > 1e-8).float().view(bs, 1, N, 1).repeat(1, K, 1, 1).contiguous()
    t = targ.view(bs, N, K, c).permute(0, 2, 1, 3).contiguous()
    s = (w * (pred - t).abs()).view(bs, K, -1).sum(2)
    return s / (w.view(bs, K, -1).sum(2) + 1e-3)


def ffb6d_loss_torch(end_points, item, valid=None, weights=(2.0, 1.0, 1.0)):
    """``(loss, info)`` of model_fn's loss block in the reference's float32 torch ops, on the sub-batch
    ``x[valid]`` (boolean indexing, a host synchronisation) when ``valid`` is given."""
    labels = item["labels"]
    segs, kp, ctr = end_points["pred_rgbd_segs"], end_points["pred_kp_ofs"], end_points["pred_ctr_ofs"]
    kp_t, ctr_t = item["kp_targ_ofst"], item["ctr_targ_ofst"]
    if valid is not None:
        v = valid.bool()
        labels, segs, kp, ctr, kp_t, ctr_t = (a[v] for a in (labels, segs, kp, ctr, kp_t, ctr_t))
    labels = labels.long()
    loss_rgbd_seg = focal_loss_torch(segs, labels.view(-1), gamma=2).sum()
    loss_kp_of = of_l1_loss_torch(kp, kp_t, labels).sum()
    loss_ctr_of = of_l1_loss_torch(ctr, ctr_t, labels).sum()
    loss = sum([ls * w for ls, w in ((loss_rgbd_seg, weights[0]), (loss_kp_of, weights[1]),
                                     (loss_ctr_of, weights[2]))])
    _, cls_rgbd = segs.max(1)
    acc = (cls_rgbd == labels).float().sum() / labels.numel()
    return loss, {"loss_rgbd_seg": loss_rgbd_seg.detach(), "loss_kp_of": loss_kp_of.detach(),
                  "loss_ctr_of": loss_ctr_of.detach(), "loss_all": loss.detach(), "acc_rgbd": acc}
