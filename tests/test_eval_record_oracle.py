"""CPU: the numpy restatement of the test run's record and summary (oracle/eval_record_oracle.py) equals
``pose.cal_auc`` and ``TorchEval.cal_auc`` / ``cal_lm_add`` over lists built from its rows by the product's own row
reader, on hand-made tables: empty classes, all distances missed, a distance of exactly 0.1, ties, inf and NaN,
symmetric classes, skipped slots and an invalid frame."""
import numpy as np
import pytest

from ffb6d_b200 import _lib, pose
from oracle import eval_record_oracle as O

N_CLS = 6
SYM = (2, 5)


def _table_free_eval(n_cls=N_CLS, sym=SYM):
    """A TorchEval whose lists the test fills: no mesh table, no GPU."""
    te = pose.TorchEval.__new__(pose.TorchEval)
    te.n_cls, te.sym_cls_ids = n_cls, list(sym)
    te.cls_add_dis, te.cls_adds_dis, te.pred_kp_errs, te.cls_add_s_dis = ([[] for _ in range(n_cls)]
                                                                         for _ in range(4))
    te.pred_id2pose_lst = []
    return te


def _same(got, want, tol=1e-9):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    np.testing.assert_allclose(got[ok], want[ok], rtol=0, atol=tol)


def _batch(rs, B, n_obj, cls_rows, dists, n_kps=4):
    """A YCB batch whose slots hold ``cls_rows`` and whose ADD / ADD-S are ``dists [B*n_obj, 2]``."""
    cls_ids = np.asarray(cls_rows, np.int32).reshape(B, n_obj)
    present = rs.rand(B, N_CLS) < 0.7
    kps = rs.uniform(-0.1, 0.1, (B, N_CLS, n_kps + 1, 3)).astype(np.float32)
    gt_kps = rs.uniform(-0.1, 0.1, (B, n_obj, n_kps, 3)).astype(np.float32)
    pred = rs.normal(size=(B, n_obj, 3, 4)).astype(np.float32)
    d = np.asarray(dists, np.float32).reshape(B * n_obj, 2)
    return dict(cls_ids=cls_ids, present=present, pred_RT=pred, add=d[:, 0], adds=d[:, 1], kps=kps, gt_kps=gt_kps)


def _tables():
    rs = np.random.RandomState(5)
    nan, inf = float("nan"), float("inf")
    return [
        # skipped slots after a zero id, an empty class (4), ties, a miss, exactly-representable small values
        (_batch(rs, 2, 4, [1, 2, 0, 3, 2, 2, 1, 0],
                [[0.01, 0.005], [0.02, 0.02], [0.5, 0.5], [0.03, 0.01],
                 [0.02, 0.02], [0.02, 0.001], [0.2, 0.07], [0.0, 0.0]]), None),
        # every distance above 0.1, and inf
        (_batch(rs, 1, 3, [1, 3, 5], [[0.3, 0.11], [inf, inf], [0.1000001, 0.9]]), None),
        # NaN in class 3's ADD only, and an invalid frame whose slots are all skipped
        (_batch(rs, 2, 3, [3, 1, 5, 2, 2, 2], [[nan, 0.04], [0.06, 0.05], [0.08, 0.02],
                                               [0.01, 0.01], [0.02, 0.02], [0.03, 0.03]]), np.array([True, False])),
        # float32 0.1 lies above the double 0.1: a miss
        (_batch(rs, 1, 2, [5, 1], [[np.float32(0.1), 0.1], [0.099999, 0.05]]), None),
    ]


def _rows():
    rows, base = [], 0
    for bt, valid in _tables():
        rows.append(O.record(valid=valid, frame_base=base, **bt))
        base += bt["cls_ids"].shape[0]
    return np.concatenate(rows)


def test_cal_auc_restatement():
    for d in ([], [0.2, 0.3], [0.1], [0.05, 0.05, 0.1, 0.02], [0.01, float("inf"), 0.03], [0.02, float("nan")],
              [float(np.float32(0.1))], list(np.random.RandomState(1).uniform(0, 0.15, 500))):
        want = pose.cal_auc(list(d))
        got = O.cal_auc(d)
        _same(got, want)
    assert O.cal_auc([0.1]) == pose.cal_auc([0.1]) == pytest.approx(100.0)     # exactly 0.1 is a hit
    assert O.cal_auc([float(np.float32(0.1))]) == 0.0                           # float32 0.1 lies above it
    assert O.cal_auc([0.05, 0.2]) == pytest.approx(50.0)


def test_record_layout():
    rs = np.random.RandomState(2)
    bt = _batch(rs, 2, 4, [1, 0, 3, 2, 4, 2, 1, 0], rs.uniform(0, 0.2, (8, 2)))
    rows = O.record(frame_base=7, **bt)
    assert rows.dtype == np.int32 and rows.shape == (8, _lib.EVAL_ROW_WORDS)
    assert list(rows[:, 0]) == [1, -1, -1, -1, 4, 2, 1, -1]
    assert list(rows[:, 1]) == [7] * 4 + [8] * 4
    vals = rows.view(np.float32)
    for r in (0, 4, 5, 6):
        b, j = divmod(r, 4)
        c = rows[r, 0]
        assert rows[r, 2] == int(bt["present"][b, c])
        assert vals[r, 3] == bt["add"][r] and vals[r, 4] == bt["adds"][r]
        np.testing.assert_array_equal(vals[r, 6:18], bt["pred_RT"][b, j].reshape(-1))
        p = bt["kps"][b, c, :-1] if bt["present"][b, c] else 0.0
        want = np.linalg.norm(bt["gt_kps"][b, j] - p, axis=1).mean()
        assert abs(vals[r, 5] - want) <= 2e-7 * max(1.0, abs(want))
    assert not rows[[1, 2, 3, 7], 2:].any()
    # an invalid frame: every slot skipped; LineMOD: slot 0 only, with the object's id and the vote's row 1
    assert (O.record(valid=np.array([False, True]), **bt)[:4, 0] == -1).all()
    lm = O.record(bt["cls_ids"], bt["present"][:, :2], bt["pred_RT"][:, 0], bt["add"][:2], bt["adds"][:2], obj_id=9)
    assert list(lm[:, 0]) == [9, -1, -1, -1, 9, -1, -1, -1]
    assert list(lm[[0, 4], 2]) == [int(bt["present"][0, 1]), int(bt["present"][1, 1])]
    assert lm.view(np.float32)[4, 3] == bt["add"][1] and lm.view(np.float32)[0, 5] == 0.0


def test_summary_equals_torch_eval_ycb():
    rows = _rows()
    te = _table_free_eval()
    pose._append_rows(rows, te.cls_add_dis, te.cls_adds_dis, te.pred_kp_errs)
    want = te.cal_auc()
    auc, _, kp = O.summary(rows, len(rows), N_CLS, SYM)
    for m, name in enumerate(("add_auc_lst", "adds_auc_lst", "add_s_auc_lst")):
        _same(auc[m], want[name])
    assert want["add_auc_lst"][4] == 0 and auc[0, 4] == 0                # the empty class
    assert np.isnan(want["add_auc_lst"][3]) and not np.isnan(want["adds_auc_lst"][3])
    assert np.isnan(want["add_auc_lst"][0])                               # class 0 holds the NaN too
    assert np.isnan(want["add_s_auc_lst"][0]) and not np.isnan(want["add_s_auc_lst"][1])
    _same(kp[0] / kp[1], want["mean_kp_err"], 1e-12)
    # the row count bounds what is read
    auc2, _, kp2 = O.summary(rows, 8, N_CLS, SYM)
    te2 = _table_free_eval()
    pose._append_rows(rows[:8], te2.cls_add_dis, te2.cls_adds_dis, te2.pred_kp_errs)
    _same(auc2[1], te2.cal_auc()["adds_auc_lst"])
    assert kp2[1] == sum(len(x) for x in te2.pred_kp_errs)


def test_summary_equals_torch_eval_linemod():
    rs = np.random.RandomState(4)
    obj = 5
    d = np.concatenate([rs.uniform(0, 0.03, (40, 2)), [[0.0172, 0.0172], [0.0171, 0.0173], [float("inf")] * 2]])
    d = d.astype(np.float32)
    B = len(d)
    rows = O.record(np.zeros((B, 2), np.int32), rs.rand(B, 2) < 0.8, rs.normal(size=(B, 3, 4)), d[:, 0], d[:, 1],
                    obj_id=obj)
    for sym in ((), (obj,)):
        te = _table_free_eval(sym=sym)
        pose._append_rows(rows, te.cls_add_dis, te.cls_adds_dis)
        want = te.cal_lm_add(obj, 172.0)
        auc, pct, _ = O.summary(rows, len(rows), N_CLS, sym, 172.0 / 1000.0 * 0.1)
        _same([auc[0, obj]], want["add_auc_lst"])
        _same([auc[1, obj]], want["adds_auc_lst"])
        _same([auc[2, obj]], want["add_s_auc_lst"])
        assert pct[0, obj] == want["add"] and pct[1, obj] == want["adds"]
    assert np.isnan(pct[0, 1])                                            # an empty class: numpy's mean of nothing
