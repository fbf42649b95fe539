"""oracle/eval_record_oracle.py -- TEST INFRASTRUCTURE ONLY. NOT A PRODUCT PATH.

A numpy restatement of the test run's device record (``ffb6d_eval_record``) and of its summary (``ffb6d_eval_auc``),
as include/ffb6d_b200.h states them:

* ``record`` -- the rows of one batch: slot ``(b, j)`` at row ``b * n_obj + j``, -1 for a skipped slot (an invalid
  frame; YCB from the frame's first zero class id on; LineMOD every slot but 0), the keypoint error in float32;
* ``summary`` -- per class and over every object (class 0), the reference's ``cal_auc`` (utils/basic_utils.py:
  642-649) on ADD, ADD-S and ADD(-S), the LineMOD ``< 0.1 diameter`` percentages and the keypoint-error sum and
  count, written from the statement rather than from :mod:`ffb6d_b200.pose`.
"""
import numpy as np

ROW_WORDS = 20


def record(cls_ids, present, pred_RT, add, adds, kps=None, gt_kps=None, valid=None, obj_id=0, frame_base=0):
    """``[B * n_obj, ROW_WORDS]`` int32 rows of one batch.  Shapes as ``ffb6d_b200.ops.eval_record`` takes them
    (numpy): ``cls_ids [B, n_obj]``, ``present [B, n_cls]``, ``pred_RT`` ``[B, n_obj, 3, 4]`` (YCB) / ``[B, 3, 4]``
    (LineMOD), ``add``, ``adds`` flat, ``kps [B, n_cls, n_kps + 1, 3]``, ``gt_kps [B, n_obj, n_kps, 3]``."""
    cls_ids = np.asarray(cls_ids)
    B, n_obj = cls_ids.shape
    present = np.asarray(present).astype(bool)
    n_cls = present.shape[1]
    rows = np.zeros((B * n_obj, ROW_WORDS), np.int32)
    vals = rows.view(np.float32)
    for b in range(B):
        zero_seen = False
        for j in range(n_obj):
            r = b * n_obj + j
            rows[r, 1] = frame_base + b
            c = int(cls_ids[b, j])
            zero_seen = zero_seen or c == 0
            skip = (valid is not None and not valid[b]) or (j > 0 if obj_id else zero_seen)
            if skip:
                rows[r, 0] = -1
                continue
            if obj_id:
                c, s, pc = obj_id, b, 1
            else:
                s, pc = r, c
            pres = 0 <= pc < n_cls and bool(present[b, pc])
            err = np.float32(0)
            if not obj_id:
                g = np.asarray(gt_kps[b, j], np.float32)
                p = np.asarray(kps[b, pc, :g.shape[0]], np.float32) if pres else np.zeros_like(g)
                d = g - p
                norms = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
                acc = norms[0]
                for x in norms[1:]:
                    acc = np.float32(acc + x)
                err = np.float32(acc / np.float32(len(norms)))
            rows[r, 0], rows[r, 2] = c, int(pres)
            vals[r, 3], vals[r, 4], vals[r, 5] = np.float32(add[s]), np.float32(adds[s]), err
            vals[r, 6:18] = np.asarray(pred_RT, np.float32).reshape(-1, 12)[s]
    return rows


def cal_auc(dist, max_dis=0.1):
    """The area under the accuracy-threshold curve in percent: misses are the distances above ``max_dis``; the
    accuracy at the i-th smallest distance is float32 ``(i + 1) / n``; the curve is closed at ``max_dis``."""
    d = np.asarray(dist, np.float64)
    n = len(d)
    if n == 0:
        return 0.0
    if np.isnan(d).any():
        return float("nan")
    hit = np.sort(d[d <= max_dis])
    if len(hit) == 0:
        return 0.0
    acc = (np.arange(1, len(hit) + 1, dtype=np.float32) / np.float32(n)).astype(np.float64)
    prev = np.concatenate(([0.0], hit[:-1]))
    area = float(np.sum((hit - prev) * acc)) + (max_dis - hit[-1]) * acc[-1]
    return area * 10 * 100


def class_lists(rows, count, n_cls, sym=()):
    """``(add, adds, add_s, kp_err)``: per class, the distances of the first ``count`` rows whose class lies in
    ``[1, n_cls)``, class 0 every such row."""
    rows = np.asarray(rows)[:count]
    vals = rows.view(np.float32)
    out = [[[] for _ in range(n_cls)] for _ in range(4)]
    for r in range(len(rows)):
        c = int(rows[r, 0])
        if not 1 <= c < n_cls:
            continue
        a, s, e = (float(vals[r, k]) for k in (3, 4, 5))
        for lst, v in zip(out, (a, s, s if c in sym else a, e)):
            lst[c].append(v)
            lst[0].append(v)
    return out


def summary(rows, count, n_cls, sym=(), lm_thr=0.0):
    """``(auc [3, n_cls], pct [2, n_cls], kp [2])`` float64 of the first ``count`` rows."""
    add, adds, add_s, kp = class_lists(rows, count, n_cls, sym)
    auc = np.array([[cal_auc(lst[c]) for c in range(n_cls)] for lst in (add, adds, add_s)])
    with np.errstate(invalid="ignore", divide="ignore"):
        pct = np.array([[np.sum(np.array(lst[c]) < lm_thr) / len(lst[c]) * 100 if lst[c] else float("nan")
                         for c in range(n_cls)] for lst in (add, adds)])
    return auc, pct, np.array([float(np.sum(kp[0], dtype=np.float64)), float(len(kp[0]))])
