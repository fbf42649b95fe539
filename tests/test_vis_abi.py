"""CPU: the drawing entry points (``ffb6d_project_p3d``, ``ffb6d_draw_p2ds``) refuse bad arguments before any launch,
their limits are the header's, and the draw workspace is B H W 8 bytes."""
import ctypes as C
import os
import re

from conftest import ROOT
from ffb6d_b200 import _lib
from ffb6d_b200._lib import lib, ERR_INVALID, ERR_WORKSPACE, last_error

LIMITS = dict(MAX_RADIUS=64, MAX_SIDE=16384, MAX_SETS=1 << 24, MAX_ROWS=1 << 24, MAX_TABLE_ROWS=2 ** 31 - 1,
              MAX_FRAMES=65535)


def test_header_limits():
    text = open(os.path.join(ROOT, "include", "ffb6d_b200.h")).read()
    got = {k: eval(v) for k, v in re.findall(r"#define FFB6D_VIS_(\w+) (.+)", text)}
    assert got == LIMITS
    assert {k: getattr(_lib, "VIS_" + k) for k in LIMITS} == LIMITS


def test_workspace_bytes():
    ws = lib.ffb6d_draw_p2ds_workspace_bytes
    assert ws(8, 480, 640) == 8 * 480 * 640 * 8
    assert ws(0, 480, 640) == 0 and ws(1, 1, 1) == 8
    for args in ((-1, 4, 4), (LIMITS["MAX_FRAMES"] + 1, 4, 4), (1, 0, 4), (1, 4, 0), (1, LIMITS["MAX_SIDE"] + 1, 4),
                 (1, 4, LIMITS["MAX_SIDE"] + 1)):
        assert ws(*args) == 0, args
    s = LIMITS["MAX_SIDE"]
    assert ws(LIMITS["MAX_FRAMES"], s, s) == LIMITS["MAX_FRAMES"] * s * s * 8      # no overflow at the limits


def test_project_checks():
    buf = (C.c_double * 64)()
    p = C.addressof(buf)

    def call(pts=p, f64=0, n_rows=10, start=p, count=p, en=None, S=2, max_rows=5, pose=None, K=p, cs=p, per_set=0,
             out=p):
        return lib.ffb6d_project_p3d(pts, f64, n_rows, start, count, en, S, max_rows, pose, K, cs, per_set, out, None)

    cases = [(dict(S=-1), "S"), (dict(S=LIMITS["MAX_SETS"] + 1), "S"), (dict(max_rows=0), "max_rows"),
             (dict(max_rows=LIMITS["MAX_ROWS"] + 1), "max_rows"), (dict(n_rows=-1), "n_rows"),
             (dict(n_rows=2 ** 31), "n_rows"), (dict(f64=2), "pts_f64"), (dict(per_set=-1), "per_set"),
             (dict(pts=p + 2), "aligned"), (dict(f64=1, pts=p + 4), "aligned"), (dict(K=p + 4), "aligned"),
             (dict(pose=p + 4), "aligned"), (dict(out=p + 4), "aligned"), (dict(start=p + 2), "aligned")]
    for name in ("pts", "start", "count", "K", "cs", "out"):
        cases.append((dict(**{name: None}), "null"))
    for kw, text in cases:
        assert call(**kw) == ERR_INVALID, kw
        assert text in last_error(), (kw, last_error())
    assert call(S=0, pts=None, start=None, count=None, K=None, cs=None, out=None) == 0     # S = 0: a no-op


def test_draw_checks():
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    need = lib.ffb6d_draw_p2ds_workspace_bytes(2, 4, 4)

    def call(img=p, B=2, H=4, W=4, p2ds=p, S=2, max_rows=5, frame=p, start=p, count=p, en=None, n_rows=10, rad=p,
             col=p, per_row=0, ws=p, wsb=need):
        return lib.ffb6d_draw_p2ds(img, B, H, W, p2ds, S, max_rows, frame, start, count, en, n_rows, rad, col,
                                   per_row, ws, wsb, None)

    cases = [(dict(B=-1), ERR_INVALID, "B"), (dict(B=LIMITS["MAX_FRAMES"] + 1), ERR_INVALID, "B"),
             (dict(H=0), ERR_INVALID, "H, W"), (dict(W=LIMITS["MAX_SIDE"] + 1), ERR_INVALID, "H, W"),
             (dict(S=-1), ERR_INVALID, "S"), (dict(S=LIMITS["MAX_SETS"] + 1), ERR_INVALID, "S"),
             (dict(max_rows=0), ERR_INVALID, "max_rows"), (dict(max_rows=LIMITS["MAX_ROWS"] + 1), ERR_INVALID,
                                                            "max_rows"),
             (dict(n_rows=-1), ERR_INVALID, "n_rows"), (dict(per_row=2), ERR_INVALID, "color_per_row"),
             (dict(p2ds=p + 4), ERR_INVALID, "aligned"), (dict(frame=p + 2), ERR_INVALID, "aligned"),
             (dict(rad=p + 1), ERR_INVALID, "aligned"), (dict(ws=p + 4), ERR_INVALID, "workspace"),
             (dict(ws=None), ERR_WORKSPACE, "workspace"), (dict(wsb=need - 1), ERR_WORKSPACE, "workspace")]
    for name in ("img", "p2ds", "frame", "start", "count", "rad", "col"):
        cases.append((dict(**{name: None}), ERR_INVALID, "null"))
    for kw, rc, text in cases:
        assert call(**kw) == rc, kw
        assert text in last_error(), (kw, last_error())
    none = dict(img=None, p2ds=None, frame=None, start=None, count=None, rad=None, col=None, ws=None, wsb=0)
    assert call(B=0, **none) == 0 and call(S=0, **none) == 0
