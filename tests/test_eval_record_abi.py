"""CPU: the record and summary entry points refuse bad arguments before any launch, their limits are the header's,
the workspace query is consistent, and ``GraphedTestStep`` rejects what it cannot capture before any CUDA work."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import ROOT
from ffb6d_b200 import _lib, evaluate
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, last_error
from ffb6d_b200.model import FFB6D, FFB6DFusionNet

MAX_ROWS = 1 << 24


def test_header_constants():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()
    assert int(re.search(r"#define FFB6D_EVAL_ROW_WORDS (\d+)", text).group(1)) == _lib.EVAL_ROW_WORDS == 20
    assert re.search(r"#define FFB6D_EVAL_MAX_ROWS \(1 << 24\)", text) and _lib.EVAL_MAX_ROWS == MAX_ROWS


def test_workspace_bytes():
    ws = lib.ffb6d_eval_auc_workspace_bytes
    assert ws(0, 22) == 0 and ws(10, 0) == 0 and ws(MAX_ROWS + 1, 22) == 0 and ws(10, _lib.VOTE_MAX_CLASSES + 1) == 0
    assert ws(-1, 22) == 0
    prev = 0
    for cap in (1, 10, 1000, 100000, MAX_ROWS):
        n = ws(cap, 22)
        assert n >= 2 * 6 * 8 * cap + 11 * 22 * 4 and n > prev     # two key arrays, the counters, CUB's scratch
        prev = n
    assert ws(1000, 1024) >= ws(1000, 22)


def _buf():
    buf = (C.c_double * 256)()
    return buf, C.addressof(buf)


def test_record_checks():
    buf, p = _buf()

    def call(ids=p, valid=None, pres=p, kps=p, poses=None, gk=p, pr=p, a=p, s=p, B=2, n_obj=3, n_cls=4, R=9, n_kps=8,
             obj=0, rows=p, cap=6, state=p, fp=None, ff=None, fcap=0):
        return lib.ffb6d_eval_record(ids, valid, pres, kps, poses, gk, pr, a, s, B, n_obj, n_cls, R, n_kps, obj, rows,
                                     cap, state, fp, ff, fcap, None)

    for kw, text in ((dict(cap=0), "capacity"), (dict(cap=-3), "capacity"), (dict(cap=MAX_ROWS + 1), "capacity"),
                     (dict(B=0), "B >= 1"), (dict(n_obj=0), "n_obj"), (dict(B=65536, n_obj=1), "B \\* n_obj"),
                     (dict(n_cls=0), "n_cls"), (dict(n_cls=_lib.VOTE_MAX_CLASSES + 1), "n_cls"),
                     (dict(R=8), "R"), (dict(n_kps=0), "n_kps"), (dict(n_kps=65, R=66), "n_kps"),
                     (dict(obj=-1), "obj_id"), (dict(obj=3, n_cls=1), "two-class"),
                     (dict(pres=None), "null"), (dict(rows=None), "null"), (dict(state=None), "null"),
                     (dict(a=None), "null"), (dict(kps=None), "YCB reads"), (dict(gk=None), "YCB reads"),
                     (dict(fp=p), "go together"), (dict(fp=p, ff=p, fcap=4), "poses"),
                     (dict(fp=p, ff=p, poses=p, fcap=0), "frame_capacity"), (dict(rows=p + 2), "misaligned"),
                     (dict(state=p + 4), "misaligned")):
        n0 = _lib.launch_count()
        assert call(**kw) == ERR_INVALID, kw
        assert re.search(text, last_error()), (kw, last_error())
        assert _lib.launch_count() == n0


def test_auc_checks():
    buf, p = _buf()
    wp = p + (-p % 256)                        # a 256-byte aligned address inside the buffer (never written)
    need = lib.ffb6d_eval_auc_workspace_bytes(10, 4)

    def call(rows=p, state=p, cap=10, n_cls=4, sym=None, thr=0.0, auc=p, pct=p, kp=p, ws=wp, wsb=need):
        return lib.ffb6d_eval_auc(rows, state, cap, n_cls, sym, thr, auc, pct, kp, ws, wsb, None)

    for kw, rc, text in ((dict(cap=0), ERR_INVALID, "capacity"), (dict(cap=MAX_ROWS + 1), ERR_INVALID, "capacity"),
                         (dict(n_cls=0), ERR_INVALID, "n_cls"), (dict(thr=float("nan")), ERR_INVALID, "lm_thr"),
                         (dict(rows=None), ERR_INVALID, "null"), (dict(kp=None), ERR_INVALID, "null"),
                         (dict(state=p + 4), ERR_INVALID, "misaligned"), (dict(ws=wp + 8), ERR_INVALID, "256-byte"),
                         (dict(ws=None, wsb=0), ERR_WORKSPACE, "workspace"), (dict(wsb=need - 1), ERR_WORKSPACE,
                                                                              "workspace")):
        n0 = _lib.launch_count()
        assert call(**kw) == rc, kw
        assert re.search(text, last_error()), (kw, last_error())
        assert _lib.launch_count() == n0


def _cpu_batch():
    z = torch.zeros
    b = {"dpt": z(2, 8, 8, dtype=torch.uint16), "rgb": z(2, 8, 8, 3, dtype=torch.uint8),
         "labels": z(2, 8, 8, dtype=torch.uint8), "nrm_map": z(2, 8, 8, 3)}
    b.update({k: z(2, 3, 3, 4) for k in ("RTs", "kp_3ds", "ctr_3ds", "cls_ids", "obj_cls", "obj_kps", "obj_ctr")})
    return b


def test_graphed_test_step_rejections(monkeypatch):
    model = FFB6D(n_classes=2, n_pts=256, n_kps=8).eval()
    kw = dict(dataset="ycb", cam_scale=1e4, K=None, mesh_pts={1: [[0, 0, 0]]}, mesh_kps={}, capacity=4)
    batch = _cpu_batch()
    G = evaluate.GraphedTestStep
    with pytest.raises(ValueError, match="DataParallel"):
        G(torch.nn.DataParallel(model), batch, **kw)
    with pytest.raises(ValueError, match="no image branch"):
        G(FFB6DFusionNet(n_classes=2, n_pts=256).eval(), batch, **kw)
    with pytest.raises(ValueError, match="dataset must be"):
        G(model, batch, **dict(kw, dataset="coco"))
    with pytest.raises(ValueError, match="obj_id"):
        G(model, batch, **dict(kw, dataset="linemod"))
    for cap in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match="capacity"):
            G(model, batch, **dict(kw, capacity=cap))
    with pytest.raises(ValueError, match="must be a dict"):
        G(model, [batch], **kw)
    with pytest.raises(ValueError, match="lacks"):
        G(model, {k: v for k, v in batch.items() if k != "kp_3ds"}, **kw)
    with pytest.raises(ValueError, match="unknown batch keys"):
        G(model, dict(batch, extra=batch["dpt"]), **kw)
    with pytest.raises(ValueError, match="CUDA tensor"):
        G(model, batch, **kw)
    model.train()
    with pytest.raises(ValueError, match="GraphedTestStep: the model is in training mode"):
        G(model, batch, **kw)
    model.eval()
    assert not lib.ffb6d_check_indices_enabled()
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="GraphedTestStep: FFB6D_CHECK_INDICES"):
        G(model, batch, **kw)
