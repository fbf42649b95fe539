"""oracle/pose_eval_oracle.py -- TEST INFRASTRUCTURE ONLY. NOT A PRODUCT PATH.

* ``add_adds_f64`` -- ADD and ADD-S (utils/basic_utils.py:651-669) in float64 over the float32 inputs: the exact
  answer the kernel's fp32 arithmetic is held to.
* ``eval_functions`` -- the reference's own scoring code (``Basic_Utils.cal_add_cuda``, ``cal_adds_cuda``,
  ``cal_auc``, module-level ``VOCap`` of utils/basic_utils.py; ``eval_metric``, ``eval_metric_lm`` and
  ``TorchEval`` of utils/pvn3d_eval_utils_kpls.py) taken out of its source files with ``ast`` and executed on the CPU
  with the module-level objects they read stubbed (the pattern of oracle/ref_loader.frame_pose_functions).  Used by
  tests/golden/make_pose_eval_golden.py only; the reference tree is not needed to run the tests.
"""
import ast
import concurrent.futures
import os

import numpy as np

from . import ref_loader as R


def add_adds_f64(mesh, pred_RT, gt_RT):
    """``mesh [N,3]``, ``pred_RT``, ``gt_RT [3,4]`` (read as float32, computed in float64) -> ``(add, adds)``.
    The nearest pred-posed point of each gt-posed point is found by brute force in blocks up to 4096 points, and
    by a float64 k-d tree above (an exact nearest-neighbour search, for the 10^4-10^6-point meshes)."""
    x = np.asarray(mesh, np.float32).astype(np.float64)
    P = np.asarray(pred_RT, np.float32).astype(np.float64)
    G = np.asarray(gt_RT, np.float32).astype(np.float64)
    p = x @ P[:, :3].T + P[:, 3]
    g = x @ G[:, :3].T + G[:, 3]
    add = np.linalg.norm(p - g, axis=1).mean()
    if not (np.isfinite(p).all() and np.isfinite(g).all()):
        return float("nan"), float("nan")
    if len(x) <= 4096:
        best = np.empty(len(x))
        for s in range(0, len(x), 512):
            d = g[s:s + 512, None, :] - p[None, :, :]
            best[s:s + 512] = np.sqrt((d * d).sum(2).min(1))
    else:
        from scipy.spatial import cKDTree
        best = cKDTree(p).query(g, k=1)[0]
    return float(add), float(best.mean())


def _functions(path, names, ns):
    with open(path) as fh:
        tree = ast.parse(fh.read())
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
        if isinstance(node, ast.ClassDef) and node.name == "Basic_Utils":
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in names:
                    exec(compile(ast.Module(body=[item], type_ignores=[]), path, "exec"), ns)
    missing = [n for n in names if n not in ns]
    if missing:
        raise RuntimeError("%s: %s not found" % (path, missing))


def eval_functions(mesh_pts, mesh_kps, cls_radius=(), ycb_sym_cls_ids=(), lm_sym_cls_ids=(), lm_diameters=None):
    """The reference's scoring functions with stubbed module state:

    * ``config``: ``n_classes = 22``, ``ycb_r_lst = cls_radius``, ``ycb_sym_cls_ids``; ``config_lm``:
      ``lm_sym_cls_ids``, ``lm_r_lst[obj]['diameter'] = lm_diameters[obj]``;
    * ``cls_lst[i] = i + 1``; ``bs_utils`` / ``bs_utils_lm``: ``get_pointxyz_cuda(cls)`` = ``mesh_pts[cls]`` as a
      float32 tensor, ``get_kps`` / ``get_ctr`` = the rows of ``mesh_kps[cls]`` (centre last), and the reference's
      own ``cal_add_cuda``, ``cal_adds_cuda`` and ``cal_auc``;
    * ``print`` and ``open`` inert; ``pkl.dump`` appends what it is given to the returned ``'dumped'`` list.

    Returns {'cal_add_cuda', 'cal_adds_cuda', 'cal_auc', 'VOCap', 'eval_metric', 'eval_metric_lm', 'TorchEval',
    'dumped'}.  The functions call ``.cuda()``: run them under ``ref_loader.cuda_is_identity``."""
    if not R.reference_sources_present():
        raise RuntimeError("reference sources not found under %s" % R.REF_ROOT)
    import torch
    utils = os.path.join(R.REF_ROOT, "ffb6d", "utils")
    bu = {"torch": torch, "np": np}
    _functions(os.path.join(utils, "basic_utils.py"), ("VOCap", "cal_add_cuda", "cal_adds_cuda", "cal_auc"), bu)
    dumped = []
    bs = R._Stub(get_kps=lambda cls, kp_type="farthest", ds_type="ycb": np.asarray(mesh_kps[int(cls)])[:-1].copy(),
                 get_ctr=lambda cls, ds_type="ycb": np.asarray(mesh_kps[int(cls)])[-1].copy(),
                 get_pointxyz_cuda=lambda cls, ds_type="ycb": torch.from_numpy(
                     np.asarray(mesh_pts[int(cls)], np.float32)).clone(),
                 cal_add_cuda=lambda *a: bu["cal_add_cuda"](None, *a),
                 cal_adds_cuda=lambda *a: bu["cal_adds_cuda"](None, *a),
                 cal_auc=lambda *a, **k: bu["cal_auc"](None, *a, **k))
    lm_r = {int(o): {"diameter": float(d)} for o, d in (lm_diameters or {}).items()}
    pose = R.pose_functions()
    ns = {"torch": torch, "np": np, "os": os, "concurrent": concurrent,
          "config": R._Stub(n_classes=22, ycb_r_lst=list(cls_radius), ycb_sym_cls_ids=list(ycb_sym_cls_ids),
                            log_eval_dir=""),
          "config_lm": R._Stub(n_classes=22, lm_sym_cls_ids=list(lm_sym_cls_ids), lm_r_lst=lm_r,
                               lm_id2obj_dict={o: "obj_%02d" % o for o in lm_r}, log_eval_dir=""),
          "bs_utils": bs, "bs_utils_lm": bs, "cls_lst": list(range(1, 22)),
          "MeanShiftTorch": pose["MeanShiftTorch"], "best_fit_transform": pose["best_fit_transform"],
          "pkl": R._Stub(dump=lambda obj, fh: dumped.append(obj)), "print": lambda *a, **k: None,
          "open": lambda *a, **k: None}
    names = ("cal_frame_poses", "cal_frame_poses_lm", "eval_metric", "eval_one_frame_pose", "eval_metric_lm",
             "eval_one_frame_pose_lm", "TorchEval")
    _functions(os.path.join(utils, "pvn3d_eval_utils_kpls.py"), names, ns)
    return {"cal_add_cuda": bs.cal_add_cuda, "cal_adds_cuda": bs.cal_adds_cuda, "cal_auc": bs.cal_auc,
            "VOCap": bu["VOCap"], "eval_metric": ns["eval_metric"], "eval_metric_lm": ns["eval_metric_lm"],
            "TorchEval": ns["TorchEval"], "dumped": dumped}
