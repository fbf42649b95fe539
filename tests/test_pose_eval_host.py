"""CPU: the ADD / ADD-S entry point refuses bad arguments before any launch; its limits are the header's; ``cal_auc``,
``VOCap`` and ``TorchEval``'s summaries equal the reference's (tests/golden/pose_eval_cases.npz, made by
tests/golden/make_pose_eval_golden.py; the distance lists are rebuilt by tests/pose_eval_cases.py); the rebuilt
inputs are the ones the reference was run on."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from ffb6d_b200 import _lib, pose
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, last_error
import pose_eval_cases as PC

GT_TILE, PRED_TILE = 512, 512
MAX_OBJECTS, MAX_POINTS, MAX_MESHES = 65535, 1 << 20, 2 ** 31 - 2


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "pose_eval_cases.npz"))
    return {k: z[k] for k in z.files}


def header_limits():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()
    return {k: int(v) for k, v in re.findall(r"#define FFB6D_POSE_EVAL_(\w+) (\d+)", text)}


def test_header_limits():
    assert header_limits() == dict(GT_TILE=GT_TILE, PRED_TILE=PRED_TILE, MAX_OBJECTS=MAX_OBJECTS,
                                   MAX_POINTS=MAX_POINTS, MAX_MESHES=MAX_MESHES)
    assert (_lib.POSE_EVAL_GT_TILE, _lib.POSE_EVAL_PRED_TILE, _lib.POSE_EVAL_MAX_OBJECTS, _lib.POSE_EVAL_MAX_POINTS,
            _lib.POSE_EVAL_MAX_MESHES) == (GT_TILE, PRED_TILE, MAX_OBJECTS, MAX_POINTS, MAX_MESHES)


def test_workspace_bytes():
    ws = lib.ffb6d_pose_add_adds_workspace_bytes
    assert ws(40, 2621) == 40 * 6 * 16
    assert ws(1, 1) == 16 and ws(0, 100) == 0
    assert ws(MAX_OBJECTS, MAX_POINTS) == MAX_OBJECTS * (MAX_POINTS // GT_TILE) * 16


def test_entry_point_checks():
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    need = lib.ffb6d_pose_add_adds_workspace_bytes(2, 100)

    def call(pts=p, off=p, nm=3, mp=100, om=p, pr=p, gt=p, M=2, add=p, adds=p, ws=p, wsb=need):
        return lib.ffb6d_pose_add_adds(pts, off, nm, mp, om, pr, gt, M, add, adds, ws, wsb, None)

    for kw, rc, text in ((dict(M=-1), ERR_INVALID, "M"), (dict(M=MAX_OBJECTS + 1), ERR_INVALID, "M"),
                         (dict(mp=0), ERR_INVALID, "max_points"), (dict(mp=MAX_POINTS + 1), ERR_INVALID, "max_points"),
                         (dict(mp=-5), ERR_INVALID, "max_points"), (dict(nm=-1), ERR_INVALID, "n_meshes"),
                         (dict(nm=MAX_MESHES + 1), ERR_INVALID, "n_meshes"), (dict(nm=0), ERR_INVALID, "n_meshes is 0"),
                         (dict(pts=None), ERR_INVALID, "null"), (dict(off=None), ERR_INVALID, "null"),
                         (dict(om=None), ERR_INVALID, "null"), (dict(pr=None), ERR_INVALID, "null"),
                         (dict(gt=None), ERR_INVALID, "null"), (dict(add=None), ERR_INVALID, "null"),
                         (dict(adds=None), ERR_INVALID, "null"), (dict(pts=p + 2), ERR_INVALID, "aligned"),
                         (dict(om=p + 1), ERR_INVALID, "aligned"), (dict(adds=p + 2), ERR_INVALID, "aligned"),
                         (dict(ws=p + 8), ERR_INVALID, "workspace must be 16-byte aligned"),
                         (dict(ws=None), ERR_WORKSPACE, "workspace"), (dict(wsb=need - 1), ERR_WORKSPACE, "workspace")):
        assert call(**kw) == rc, kw
        assert text in last_error(), (kw, last_error())
    # M = 0 is a successful no-op, whatever the pointers
    assert call(M=0, pts=None, off=None, om=None, pr=None, gt=None, add=None, adds=None, ws=None, wsb=0, nm=0) == 0


def test_op_refuses_bad_arguments():
    import torch
    from ffb6d_b200 import ops
    pts = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.pose_add_adds(pts, torch.zeros(2, dtype=torch.int32), torch.zeros(1, dtype=torch.int32),
                          torch.zeros(1, 3, 4), torch.zeros(1, 3, 4), 4)
    with pytest.raises(TypeError):
        ops.pose_add_adds([[0.0, 0.0, 0.0]], None, None, None, None, 4)
    with pytest.raises(ValueError):
        pose.MeshTable({})
    with pytest.raises(ValueError):
        pose.MeshTable({1: np.zeros((4, 2))}, device="cpu")
    with pytest.raises(ValueError):
        pose.MeshTable({-1: np.zeros((4, 3))}, device="cpu")


AUC_LISTS = tuple(PC.auc_lists())


@pytest.mark.parametrize("name", AUC_LISTS)
def test_cal_auc_and_vocap_equal_reference(golden, name):
    dis = np.array(PC.auc_lists()[name], np.float64)
    want = golden["auc:%s:auc" % name]
    for arg in (list(dis), dis):
        got = pose.cal_auc(arg)
        if np.isnan(want):
            assert np.isnan(got)
        else:
            assert abs(got - want) <= 1e-12, (got, want)
    D = dis.copy()
    D[D > 0.1] = np.inf
    acc = np.cumsum(np.ones(len(dis)), dtype=np.float32) / max(len(dis), 1)
    got, want = pose.VOCap(np.sort(D), acc), golden["auc:%s:vocap" % name]
    assert (np.isnan(got) and np.isnan(want)) or abs(got - want) <= 1e-12, (got, want)


def test_cal_auc_quirks():
    assert pose.cal_auc([]) == 0
    assert pose.cal_auc([0.2, 0.3]) == 0                  # every distance a miss
    assert pose.cal_auc([0.1]) > 0                        # exactly max_dis stays
    assert np.isnan(pose.cal_auc([0.05, float("nan")]))


def unflatten(golden, key, n_cls=22):
    out = [[] for _ in range(n_cls)]
    for c, v in zip(golden[key + ":cls"], golden[key + ":val"]):
        out[int(c)].append(float(v))
    return out


def _table_free_eval(n_cls=22, sym=()):
    """A TorchEval whose lists the test fills itself: no mesh table, no GPU."""
    te = pose.TorchEval.__new__(pose.TorchEval)
    te.n_cls, te.sym_cls_ids = n_cls, list(sym)
    te.cls_add_s_dis = [[] for _ in range(n_cls)]
    te.pred_id2pose_lst = []
    return te


def test_torch_eval_cal_auc_equals_reference(golden):
    te = _table_free_eval(sym=(13, 16, 19, 20, 21))
    te.cls_add_dis = unflatten(golden, "te:add_dis_lst")
    te.cls_adds_dis = unflatten(golden, "te:adds_dis_lst")
    te.pred_kp_errs = unflatten(golden, "te:pred_kp_errs")
    first = te.cal_auc()
    for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        np.testing.assert_allclose(first[name], golden["te:" + name], rtol=0, atol=1e-12)
    assert first["add_dis_lst"] == unflatten(golden, "te:add_dis_lst")
    assert np.isclose(first["add_s_auc_mean"], np.mean(golden["te:add_s_auc_lst"][1:]), rtol=0, atol=1e-12)
    kp = unflatten(golden, "te:pred_kp_errs")
    assert np.isclose(first["mean_kp_err"], sum(map(sum, kp)) / sum(map(len, kp)), rtol=0, atol=1e-12)
    second = te.cal_auc()                                 # the reference would count class 0's ADD(-S) twice
    for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        assert second[name] == first[name]


def test_torch_eval_cal_lm_add_equals_reference(golden):
    te = _table_free_eval(sym=(10, 11))
    te.cls_add_dis = unflatten(golden, "telm:add_dis_lst")
    te.cls_adds_dis = unflatten(golden, "telm:adds_dis_lst")
    for _ in range(2):
        got = te.cal_lm_add(10, 172.0)
        for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
            np.testing.assert_allclose(got[name], golden["telm:" + name], rtol=0, atol=1e-12)
        assert got["add"] == golden["telm:add"] and got["adds"] == golden["telm:adds"]


def test_torch_eval_bookkeeping():
    """Symmetric classes score ADD-S in ADD(-S), the others ADD; class 0 gathers every class in class order; the
    LineMOD ``< 0.1 diameter`` share counts strictly smaller distances."""
    te = _table_free_eval(n_cls=4, sym=(2,))
    te.cls_add_dis = [[0.01, 0.5, 0.02], [0.01, 0.5], [0.02], []]
    te.cls_adds_dis = [[0.005, 0.05, 0.001], [0.005, 0.05], [0.001], []]
    te.pred_kp_errs = [[], [0.1, 0.3], [0.2], []]
    r = te.cal_auc()
    assert te.cls_add_s_dis == [[0.01, 0.5, 0.001], [0.01, 0.5], [0.001], []]
    assert r["add_s_auc_lst"][2] == pose.cal_auc([0.001]) and r["add_s_auc_lst"][3] == 0
    assert np.isclose(r["mean_kp_err"], 0.2)
    te.cls_add_dis[1] = [0.0172, 0.0171, 0.02]
    assert te.cal_lm_add(1, 172.0)["add"] == pytest.approx(100.0 / 3)


def test_rebuilt_frames_match_golden(golden):
    """The voting frames tests/pose_eval_cases.py rebuilds are those the golden run was made from."""
    frs, _, _ = PC.frames()
    np.testing.assert_allclose(PC.frame_fingerprint(PC.ycb_batch(frs)), golden["te:fingerprint"], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(PC.frame_fingerprint(PC.lm_batch()[0]), golden["telm:fingerprint"], rtol=1e-9,
                               atol=1e-9)
