"""oracle/vis_oracle.py -- TEST INFRASTRUCTURE ONLY. NOT A PRODUCT PATH.

A numpy restatement of the pose and label drawing of ``ffb6d_b200.vis``, without cv2:

* ``fma`` -- a correctly rounded float64 fused multiply-add, vectorised: the error-free product and sum, then the
  rounding-to-odd step of Boldo and Melquiond ("Emulation of FMA and correctly rounded sums: proved algorithms using
  rounding to odd", IEEE Trans. Computers 57(4), 2008).  Exact for finite operands away from under- and overflow;
  elsewhere (a non-finite operand or result) it is the plain ``a * b + c``, which agrees there.
* ``project_p3d`` -- ``Basic_Utils.project_p3d`` (utils/basic_utils.py:268-277) as numpy computes it with the
  OpenBLAS Haswell dgemm kernel: the ``np.dot`` products as fma chains, optionally after the demo's posing.
* ``circle_offsets`` -- the pixels of ``cv2.circle(img, c, r, colour, -1)`` (LINE_8, shift 0) relative to the
  centre: OpenCV's integer midpoint walk, filled by horizontal spans.
* ``draw_sets`` / ``draw_p2ds`` -- the reference's drawing loop: clip each centre to ``[0,W] x [0,H]``, draw its
  circle clipped to the image, later draws over earlier ones.
* ``demo_draw`` / ``view_labels`` -- the drawing block of demo.py's ``cal_view_pred_pose`` (demo.py:116-145, which
  cannot be imported) and the trainers' ``view_labels`` (train_ycb.py:189-204), restated over these functions.
* ``reference_functions`` -- the reference's own ``project_p3d``, ``draw_p2ds``, ``get_label_color`` (methods of
  ``Basic_Utils``), ``view_labels`` and ``color_lst`` (train_ycb.py), taken out of the source files with ``ast`` and
  run with cv2.  Used by tests/golden/make_vis_golden.py and tools/vis_bench.py; the tests do not need the
  reference tree.
"""
import ast
import os

import numpy as np

from . import ref_loader as R

INT32_MIN = np.int32(-2 ** 31)


# ------------------------------------------------------------------------------------------------------- arithmetic
def _split(a):
    c = 134217729.0 * a                           # 2^27 + 1: Veltkamp's split into two 26-bit halves
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _two_sum(a, b):
    s = a + b
    bp = s - a
    return s, (a - (s - bp)) + (b - bp)


def _add_odd(a, b):
    """a + b rounded to odd: the neighbour with an odd significand when the sum is inexact."""
    s, e = _two_sum(a, b)
    even = (s.view(np.int64) & 1) == 0
    toward = np.nextafter(s, np.where(e > 0, np.inf, -np.inf))
    return np.where((e != 0) & even, toward, s)


def fma(a, b, c):
    """Correctly rounded ``a * b + c`` in float64, elementwise."""
    a, b, c = (np.asarray(v, np.float64) for v in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    with np.errstate(all="ignore"):
        plain = a * b + c
        uh, ul = _two_prod(a, b)
        th, tl = _two_sum(c, uh)
        exact = th + _add_odd(tl, ul)
        ok = np.isfinite(a) & np.isfinite(b) & np.isfinite(c) & np.isfinite(plain) & np.isfinite(exact)
        ok &= np.abs(uh) < 2.0 ** 990
    return np.where(ok, exact, plain)


def to_int32(q):
    """numpy's ``astype(np.int32)`` of float64 on x86 (cvttsd2si): NaN and values outside [-2^31, 2^31) give
    INT32_MIN."""
    with np.errstate(invalid="ignore"):
        ok = (q >= -2.0 ** 31) & (q < 2.0 ** 31)
        return np.where(ok, np.where(ok, q, 0).astype(np.int64), INT32_MIN).astype(np.int32)


def dot3(p, M):
    """``np.dot(p, M.T)`` for ``p [N,3]``, ``M [3,3]`` float64: out_j = fma(p2, M[j,2], fma(p1, M[j,1], p0 M[j,0]))."""
    p = np.asarray(p, np.float64)
    M = np.asarray(M, np.float64)
    with np.errstate(all="ignore"):
        return np.stack([fma(p[:, 2], M[j, 2], fma(p[:, 1], M[j, 1], p[:, 0] * M[j, 0])) for j in range(3)], axis=1)


def project_p3d(p3d, cam_scale, K, pose=None):
    """``[N,3]`` float32 or float64 -> int32 ``[N,2]``.  With ``pose [3,4]`` the points are first posed in float64
    (``np.dot(p, R.T) + t``); the scale is applied in the points' dtype as numpy casts ``p3d * cam_scale``."""
    p = np.asarray(p3d)
    K = np.asarray(K, np.float64)
    with np.errstate(all="ignore"):
        if pose is not None:
            pose = np.asarray(pose, np.float64)
            p = dot3(p, pose[:, :3]) + pose[:, 3]
        p = p * cam_scale
        q = dot3(p, K)
        z = q[:, 2]
        z = np.where(z < 1e-8, 1.0, z)
        return np.stack([to_int32(np.rint(q[:, 0] / z)), to_int32(np.rint(q[:, 1] / z))], axis=1)


# ------------------------------------------------------------------------------------------------------------ drawing
_offsets = {}


def circle_offsets(r):
    """``(dy [n], dx [n])`` int64: the pixels of OpenCV's filled circle of radius ``r`` around its centre."""
    if r not in _offsets:
        half = {}                                 # row offset -> half width, over every span of the walk
        err, dx, dy, plus, minus = 0, r, 0, 1, 2 * r - 1
        while dx >= dy:
            for row, hw in ((dy, dx), (-dy, dx), (dx, dy), (-dx, dy)):
                half[row] = max(half.get(row, -1), hw)
            dy += 1
            err += plus
            plus += 2
            mask = -1 if err > 0 else 0
            err -= minus & mask
            dx += mask
            minus -= mask & 2
        pix = [(row, x) for row, hw in sorted(half.items()) for x in range(-hw, hw + 1)]
        _offsets[r] = tuple(np.array(v, np.int64) for v in zip(*pix))
    return _offsets[r]


def draw_sets(imgs, sets):
    """Draw in place, in order, into ``imgs [B,H,W,3]`` uint8: ``sets`` is a list of ``(frame, p2ds [n,2], radius,
    colours [n,3] or [3])``.  Each centre is clipped to ``[0,W] x [0,H]`` and its circle to the image; where circles
    overlap the later draw wins.  Returns ``imgs``."""
    B, H, W, _ = imgs.shape
    keys = np.zeros(B * H * W, np.int64)
    paint = [np.zeros((0, 3), np.uint8)]
    base = 0
    for b, p2ds, r, col in sets:
        p2ds = np.asarray(p2ds, np.int64).reshape(-1, 2)
        n = len(p2ds)
        col = np.broadcast_to(np.asarray(col, np.uint8).reshape(-1, 3), (n, 3))
        paint.append(col)
        if n == 0:
            continue
        cx = np.clip(p2ds[:, 0], 0, W)
        cy = np.clip(p2ds[:, 1], 0, H)
        dy, dx = circle_offsets(int(r))
        x = cx[:, None] + dx[None]
        y = cy[:, None] + dy[None]
        k = np.broadcast_to(base + 1 + np.arange(n)[:, None], x.shape)
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        np.maximum.at(keys, (b * H + y[ok]) * W + x[ok], k[ok])
        base += n
    colours = np.concatenate(paint)
    flat = imgs.reshape(-1, 3)
    hit = keys > 0
    flat[hit] = colours[keys[hit] - 1]
    return imgs


def draw_p2ds(img, p2ds, r=1, color=((255, 0, 0),)):
    """The reference's ``draw_p2ds`` on one ``[H,W,3]`` image (a colour list whose length is not ``len(p2ds)`` means
    ``color[0]`` for every point); the caller's ``p2ds`` are not modified.  Returns ``img``, drawn in place."""
    if isinstance(color, tuple) and len(color) == 3 and not isinstance(color[0], (tuple, list, np.ndarray)):
        color = [color]
    n = len(p2ds)
    col = np.asarray(color, np.uint8).reshape(-1, 3)
    if len(col) != n:
        col = col[:1]
    draw_sets(img[None], [(0, p2ds, r, col)])
    return img


def label_color_mode2(cls_id, n_obj=22):
    """``get_label_color(cls_id, n_obj, mode=2)``: the demo's colours."""
    m = 255 * 255 * 255 // n_obj * cls_id
    return (m // 255 // 255, (m // 255) % 255, m % 255)


def color_lst(n_objects):
    """The trainers' ``color_lst`` (train_ycb.py:50-54)."""
    out = [(0, 0, 0)]
    for i in range(n_objects):
        m = (255 * 255 * 255) // (i + 1)
        out.append((m // (255 * 255), (m // 255) % 255, m % 255))
    return out


def demo_draw(rgb_chw, cls_ids, pred_cls_ids, pred_pose_lst, mesh_pts, K, dataset, obj_id=-1, fns=None):
    """The drawing block of ``cal_view_pred_pose`` (demo.py:116-145) for one frame: ``rgb_chw [3,H,W]`` (the
    network's input, cast to uint8), ``cls_ids [n_obj,1]`` its ground-truth slots, the voting's ``pred_cls_ids`` and
    ``pred_pose_lst`` (LineMOD: one pose, class 1), ``mesh_pts {id: [P,3]}``.  Returns the BGR image the demo writes.
    ``fns``: ``{'project_p3d', 'draw_p2ds', 'get_label_color'}`` to draw with (the reference's, from
    :func:`reference_functions`), or None for this module's."""
    project = fns["project_p3d"] if fns else (lambda p, s, k: project_p3d(p, s, k))
    draw = fns["draw_p2ds"] if fns else draw_p2ds
    colour = fns["get_label_color"] if fns else (lambda c, n_obj=22, mode=2: label_color_mode2(c, n_obj))
    if dataset != "ycb":
        pred_cls_ids = np.array([[1]])
    np_rgb = np.asarray(rgb_chw).astype("uint8").transpose(1, 2, 0).copy()
    if dataset == "ycb":
        np_rgb = np_rgb[:, :, ::-1].copy()
    for cls_id in np.asarray(cls_ids):
        idx = np.where(pred_cls_ids == cls_id)[0]
        if len(idx) == 0:
            continue
        pose = pred_pose_lst[idx[0]]
        if dataset == "ycb":
            obj_id = int(cls_id[0])
        pts = np.asarray(mesh_pts[obj_id]).copy()
        pts = np.dot(pts, pose[:, :3].T) + pose[:, 3] if fns else pts
        p2ds = project(pts, 1.0, K) if fns else project_p3d(pts, 1.0, K, pose)
        np_rgb = draw(np_rgb, p2ds, color=colour(obj_id, n_obj=22, mode=2))
    return np_rgb if dataset == "ycb" else np_rgb[:, :, ::-1]


def view_labels(h, w, cld_nc, labels, K, n_objects=22):
    """The trainers' ``view_labels`` of one frame: ``cld_nc [N,3]`` float32, ``labels [N]`` -> ``[h,w,3]`` uint8."""
    p2ds = project_p3d(np.asarray(cld_nc, np.float32), 1.0, K)
    lst = color_lst(n_objects)
    col = np.array([lst[int(lb)] if int(lb) else (0, 0, 0) for lb in labels], np.uint8).reshape(-1, 3)
    img = np.zeros((h, w, 3), np.uint8)
    return draw_sets(img[None], [(0, p2ds, 3, col)])[0]


# ------------------------------------------------------------------------------------------ the reference's own code
def reference_functions(n_objects=22):
    """The reference's ``project_p3d``, ``draw_p2ds`` and ``get_label_color`` (``Basic_Utils`` methods, bound to a
    stub ``self``), ``view_labels`` with its ``K`` default removed (train_ycb.py) and ``color_lst`` built by
    train_ycb.py's own loop with ``config.n_objects = n_objects``.  Needs the reference's sources and cv2."""
    if not R.reference_sources_present():
        raise RuntimeError("reference sources not found under %s" % R.REF_ROOT)
    import cv2
    ffb6d = os.path.join(R.REF_ROOT, "ffb6d")
    path = os.path.join(ffb6d, "utils", "basic_utils.py")
    with open(path) as fh:
        tree = ast.parse(fh.read())
    ns = {"np": np, "cv2": cv2, "intrinsic_matrix": {}}
    want = ("project_p3d", "draw_p2ds", "get_label_color")
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == "Basic_Utils":
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in want:
                    item.args.defaults = [ast.copy_location(ast.Constant(None), d) if isinstance(d, ast.Subscript)
                                          else d for d in item.args.defaults]   # K=intrinsic_matrix['ycb_K1']
                    exec(compile(ast.Module(body=[item], type_ignores=[]), path, "exec"), ns)
    bs = R._Stub()
    fns = {n: (lambda f: lambda *a, **k: f(bs, *a, **k))(ns[n]) for n in want}
    bs.__dict__.update(fns)
    path = os.path.join(ffb6d, "train_ycb.py")
    with open(path) as fh:
        tree = ast.parse(fh.read())
    tns = {"np": np, "bs_utils": bs, "config": R._Stub(n_objects=n_objects)}
    for i, node in enumerate(tree.body):
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "color_lst" for t in node.targets):
            exec(compile(ast.Module(body=tree.body[i:i + 2], type_ignores=[]), path, "exec"), tns)
        if isinstance(node, ast.FunctionDef) and node.name == "view_labels":
            node.args.defaults = []
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), tns)
    fns["color_lst"] = tns["color_lst"]
    fns["view_labels"] = tns["view_labels"]
    return fns
