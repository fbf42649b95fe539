"""oracle/fps_oracle.py -- TEST INFRASTRUCTURE ONLY. NOT A PRODUCT PATH.

The reference's farthest point sampling on the CPU: ``oracle/_ref/libfps_ref.so`` is the unmodified
utils/dataset_tools/fps/src/farthest_point_sampling.cpp, built by :func:`build` (the recipe
oracle/fps_ref.mk) with the flags of fps/setup.py.  Its two extern "C" functions are what the reference's cffi module
``_ext`` binds; :func:`fps` restates the marshalling of fps/fps_utils.py:8-23 (contiguous float32 in, int32 [sn] out) and returns the indices,
where ``fps_utils.farthest_point_sampling`` returns ``pts[idxs]``.

Without ``init_center`` the reference seeds ``srand(time(0))`` and starts from ``rand() % pn``: ``idxs[0]`` is that
random start, and every later index is a function of it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import ref_loader

_HERE = os.path.dirname(os.path.abspath(__file__))
FPS_SO = os.path.join(_HERE, "_ref", "libfps_ref.so")
_lib = None


def available():
    return os.path.exists(FPS_SO)


def build():
    """(Re)build oracle/_ref/libfps_ref.so from the reference's source with oracle/fps_ref.mk."""
    if not ref_loader.reference_sources_present():
        raise RuntimeError("reference sources not found under %s" % ref_loader.REF_ROOT)
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "fps_ref.mk", "REF=%s" % ref_loader.REF_ROOT])


def _load():
    global _lib
    if _lib is None:
        if not available() and ref_loader.reference_sources_present():
            build()
        lib = C.CDLL(FPS_SO)
        for name in ("farthest_point_sampling", "farthest_point_sampling_init_center"):
            fn = getattr(lib, name)          # void f(float *pts [pn,3], int *idxs [sn], int pn, int sn)
            fn.restype = None
            fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        _lib = lib
    return _lib


def fps(pts, sn, init_center=False):
    """Indices [sn] int32 the reference's farthest point sampling selects from ``pts [pn,3]``."""
    pts = np.ascontiguousarray(pts, np.float32)
    pn, d = pts.shape
    assert d == 3 and pn >= 1 and sn >= 1
    idxs = np.zeros([sn], np.int32)
    lib = _load()
    fn = lib.farthest_point_sampling_init_center if init_center else lib.farthest_point_sampling
    fn(pts.ctypes.data, idxs.ctypes.data, pn, sn)
    return idxs
