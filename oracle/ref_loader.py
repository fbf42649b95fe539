"""oracle/ref_loader.py -- TEST INFRASTRUCTURE ONLY. NOT A PRODUCT PATH.

Access to the REFERENCE'S OWN code, used to pin the restatements in cpu_oracle.py and
as the CPU baseline of bench.py (``cpu_baseline.kind == "reference"``):

* ``oracle/_ref/libknn_ref.so``  -- the unmodified NN/knn_.cxx + nanoflann.hpp, built by
  ``make -C oracle ref`` from /root/reference (C++ linkage: called by mangled name).
* ``oracle/_ref/libgrid_ref.so`` -- the unmodified grid_subsampling.cpp + cloud.cpp behind
  the extern "C" doorway of oracle/grid_ref_shim.cpp.
* the reference's torch functions, taken out of its source files with ``ast`` at run time
  (only where /root/reference exists; nothing is copied into this repository).

The built .so files are git-ignored but travel to the GPU box with the snapshot;
/root/reference does not, so the AST-extracted functions exist only in this container
(their outputs on seeded inputs are committed under tests/golden/).
"""
import ast
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = os.environ.get("FFB6D_REFERENCE", "/root/reference")
KNN_SO = os.path.join(_HERE, "_ref", "libknn_ref.so")
GRID_SO = os.path.join(_HERE, "_ref", "libgrid_ref.so")


def reference_sources_present():
    return os.path.isdir(os.path.join(REF_ROOT, "ffb6d", "models", "RandLA"))


def build_ref():
    """(Re)build oracle/_ref from the reference sources; needs /root/reference."""
    if not reference_sources_present():
        raise RuntimeError("reference sources not found under %s" % REF_ROOT)
    subprocess.check_call(["make", "-s", "-C", _HERE, "ref", "REF=%s" % REF_ROOT])


def knn_available():
    return os.path.exists(KNN_SO)


def grid_available():
    return os.path.exists(GRID_SO)


_knn = None
_grid = None


def _knn_lib():
    global _knn
    if _knn is None:
        lib = C.CDLL(KNN_SO)
        sig = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t,
               C.c_void_p]
        # void cpp_knn_batch[_omp](const float*, size_t, size_t, size_t, const float*, size_t,
        #                          size_t, long*)                       (NN/knn_.h:10-16)
        for name in ("_Z17cpp_knn_batch_ompPKfmmmS0_mmPl", "_Z13cpp_knn_batchPKfmmmS0_mmPl"):
            fn = getattr(lib, name)
            fn.restype = None
            fn.argtypes = sig
        _knn = lib
    return _knn


def knn_batch(pts, queries, K, omp=False):
    """The reference's ``nearest_neighbors.knn_batch`` (NN/knn.pyx:71-109) with the Cython
    marshalling restated: contiguous float32 in, int64 [B,Q,K] out."""
    pts_c = np.ascontiguousarray(pts, dtype=np.float32)
    qry_c = np.ascontiguousarray(queries, dtype=np.float32)
    B, S, dim = pts_c.shape
    Q = qry_c.shape[1]
    indices = np.zeros((B, Q, K), dtype=np.int64)
    lib = _knn_lib()
    fn = lib._Z17cpp_knn_batch_ompPKfmmmS0_mmPl if omp else lib._Z13cpp_knn_batchPKfmmmS0_mmPl
    fn(pts_c.ctypes.data, B, S, dim, qry_c.ctypes.data, Q, K, indices.ctypes.data)
    return indices


def knn_search(support_pts, query_pts, k, omp=True):
    """``DataProcessing.knn_search`` (helper_tool.py:160-170) on the reference's compiled code."""
    return knn_batch(support_pts, query_pts, k, omp=omp).astype(np.int32)


def grid_subsampling(points, features=None, classes=None, sampleDl=0.1):
    """The reference's ``grid_subsampling.compute`` (GS/cpp_subsampling/wrapper.cpp:58-286);
    rows in the reference's own (hash-map) order."""
    global _grid
    if _grid is None:
        _grid = C.CDLL(GRID_SO)
        _grid.ref_grid_subsampling.restype = C.c_long
        _grid.ref_grid_subsampling.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                               C.c_void_p, C.c_size_t, C.c_float, C.c_void_p,
                                               C.c_void_p, C.c_void_p]
    pts = np.ascontiguousarray(points, dtype=np.float32)
    N = pts.shape[0]
    feats = None if features is None else np.ascontiguousarray(features, dtype=np.float32)
    cls = None if classes is None else np.ascontiguousarray(classes, dtype=np.int32)
    fdim = 0 if feats is None else feats.shape[1]
    ldim = 0 if cls is None else (1 if cls.ndim == 1 else cls.shape[1])
    sp = np.empty((N, 3), np.float32)
    sf = np.empty((N, max(fdim, 1)), np.float32)
    sc = np.empty((N, max(ldim, 1)), np.int32)
    M = _grid.ref_grid_subsampling(pts.ctypes.data, N,
                                   feats.ctypes.data if feats is not None else None, fdim,
                                   cls.ctypes.data if cls is not None else None, ldim,
                                   float(sampleDl), sp.ctypes.data, sf.ctypes.data, sc.ctypes.data)
    out = [sp[:M].copy()]
    if feats is not None:
        out.append(sf[:M, :fdim].copy())
    if cls is not None:
        out.append(sc[:M, :ldim].copy())
    return tuple(out)


# ----------------------------------------------------------------------------- torch functions
def _extract(path, class_name, func_names):
    """Pull methods out of a reference source file without importing it (importing
    models.ffb6d drags in the native extension modules, SURVEY.md §8c)."""
    import torch
    with open(path) as fh:
        tree = ast.parse(fh.read())
    found = {}
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == class_name:
            for item in node.body:
                if isinstance(item, ast.FunctionDef) and item.name in func_names:
                    item.decorator_list = []
                    mod = ast.Module(body=[item], type_ignores=[])
                    ns = {"torch": torch}
                    exec(compile(mod, path, "exec"), ns)
                    found[item.name] = ns[item.name]
    missing = set(func_names) - set(found)
    if missing:
        raise RuntimeError("%s: %s not found in class %s" % (path, sorted(missing), class_name))
    return found


_torch_fns = None


def torch_functions():
    """{'random_sample', 'nearest_interpolation' (models/ffb6d.py:159-194, FFB6D),
    'gather_neighbour', 'relative_pos_encoding' (models/RandLA/RandLANet.py:216-234)} as
    plain functions executed from the reference's own source text."""
    global _torch_fns
    if _torch_fns is None:
        if not reference_sources_present():
            raise RuntimeError("reference sources not found under %s" % REF_ROOT)
        f1 = _extract(os.path.join(REF_ROOT, "ffb6d", "models", "ffb6d.py"), "FFB6D",
                      ["random_sample", "nearest_interpolation"])
        f2 = _extract(os.path.join(REF_ROOT, "ffb6d", "models", "RandLA", "RandLANet.py"),
                      "Building_block", ["gather_neighbour", "relative_pos_encoding"])
        gn = f2["gather_neighbour"]
        rpe_raw = f2["relative_pos_encoding"]

        class _Self:  # relative_pos_encoding is an instance method calling self.gather_neighbour
            gather_neighbour = staticmethod(gn)

        f2["relative_pos_encoding"] = lambda xyz, idx: rpe_raw(_Self(), xyz, idx)
        _torch_fns = dict(f1, **f2)
    return _torch_fns


# ----------------------------------------------------------------------------- pose voting
_pose_fns = None


def pose_functions():
    """{'MeanShiftTorch' (utils/meanshift_pytorch.py:27-57, the class itself), 'best_fit_transform'
    (utils/pvn3d_eval_utils_kpls.py:28-59)} executed from the reference's own source text on the CPU.
    (Importing pvn3d_eval_utils_kpls runs ``Config`` and reads dataset files; the function is taken out of the
    file with ``ast`` instead.)"""
    global _pose_fns
    if _pose_fns is None:
        if not reference_sources_present():
            raise RuntimeError("reference sources not found under %s" % REF_ROOT)
        import math
        import torch
        fns = {}
        for path, names in ((os.path.join(REF_ROOT, "ffb6d", "utils", "meanshift_pytorch.py"),
                             ("gaussian_kernel", "distance_batch", "MeanShiftTorch")),
                            (os.path.join(REF_ROOT, "ffb6d", "utils", "pvn3d_eval_utils_kpls.py"), ("best_fit_transform",))):
            with open(path) as fh:
                tree = ast.parse(fh.read())
            ns = {"torch": torch, "np": np, "math": math}
            for node in tree.body:
                if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
                    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
            for n in names:
                fns[n] = ns[n]
        _pose_fns = fns
    return _pose_fns


class _Stub:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def frame_pose_functions(mesh_kps, cls_radius):
    """{'cal_frame_poses', 'cal_frame_poses_lm'} (utils/pvn3d_eval_utils_kpls.py:65-160, 220-284) executed from
    the reference's own source text on the CPU, with the module-level objects they read stubbed: ``config.ycb_r_lst``
    = ``cls_radius``; ``cls_lst[i]`` = ``i + 1`` and ``bs_utils.get_kps`` / ``get_ctr`` = the rows of
    ``mesh_kps[cls_id]`` ``[n_kps+1,3]`` (centre last); ``bs_utils_lm`` the same, keyed by ``obj_id``;
    ``MeanShiftTorch`` and ``best_fit_transform`` the reference's own (:func:`pose_functions`).  The functions
    call ``.cuda()``: run them under :func:`cuda_is_identity`."""
    if not reference_sources_present():
        raise RuntimeError("reference sources not found under %s" % REF_ROOT)
    import torch
    base = pose_functions()
    path = os.path.join(REF_ROOT, "ffb6d", "utils", "pvn3d_eval_utils_kpls.py")
    bs = _Stub(get_kps=lambda cls, kp_type="farthest", ds_type="ycb": mesh_kps[int(cls)][:-1].copy(),
               get_ctr=lambda cls, ds_type="ycb": mesh_kps[int(cls)][-1].copy())
    ns = {"torch": torch, "np": np, "config": _Stub(ycb_r_lst=list(cls_radius)), "bs_utils": bs, "bs_utils_lm": bs,
          "cls_lst": list(range(1, len(cls_radius) + 1)), "MeanShiftTorch": base["MeanShiftTorch"],
          "best_fit_transform": base["best_fit_transform"]}
    with open(path) as fh:
        tree = ast.parse(fh.read())
    names = ("cal_frame_poses", "cal_frame_poses_lm")
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return {n: ns[n] for n in names}


class cuda_is_identity:
    """Context manager: ``Tensor.cuda()`` returns the tensor itself (the reference's eval code on the CPU)."""

    def __enter__(self):
        import torch
        self._saved = torch.Tensor.cuda
        torch.Tensor.cuda = lambda self, *a, **k: self
        return self

    def __exit__(self, *exc):
        import torch
        torch.Tensor.cuda = self._saved
        return False
