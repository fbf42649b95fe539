"""CPU: the farthest point sampling entry point and op refuse bad arguments without a GPU; the object-info
restatement equals the reference's MeshUtils; the reference's FPS builds from oracle/fps_ref.mk and reproduces the
golden indices."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import fps_cases as FC
from conftest import GOLDEN
from ffb6d_b200 import objinfo, ops
from ffb6d_b200._lib import lib, ERR_INVALID, FPS_MAX_CLOUDS, FPS_MAX_POINTS, FPS_MAX_SAMPLES, last_error
from oracle import fps_oracle, ref_loader


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "fps_cases.npz"))
    return {k: z[k] for k in z.files}


def test_entry_point_checks():
    buf = (C.c_float * 16)()
    p = C.addressof(buf)

    def call(pts=p, counts=None, G=1, P=4, S=2, start=p, ic=0, out=p):
        return lib.ffb6d_farthest_point_sampling(pts, counts, G, P, S, start, ic, out, None, 0, None)

    for kw, text in ((dict(S=0), "S"), (dict(S=-1), "S"), (dict(S=FPS_MAX_SAMPLES + 1), "S"),
                     (dict(P=0), "P"), (dict(P=FPS_MAX_POINTS + 1), "P"), (dict(G=0), "G"),
                     (dict(G=FPS_MAX_CLOUDS + 1), "G"), (dict(ic=2), "init_center"), (dict(pts=None), "null"),
                     (dict(out=None), "null"), (dict(start=None), "start"), (dict(pts=p + 2), "aligned"),
                     (dict(counts=p + 1), "aligned")):
        assert call(**kw) == ERR_INVALID, kw
        assert text in last_error(), (kw, last_error())
    assert lib.ffb6d_farthest_point_sampling_workspace_bytes(FPS_MAX_CLOUDS, FPS_MAX_POINTS, FPS_MAX_SAMPLES) == 0


def test_op_refuses_bad_arguments():
    pts = np.zeros((4, 3), np.float32)
    with pytest.raises(ValueError):
        ops.farthest_point_sampling(np.zeros((4, 2)), 2, init_center=True)            # not [P,3]
    with pytest.raises(ValueError):
        ops.farthest_point_sampling(np.zeros((2, 4, 3)), 2, init_center=True)         # numpy takes one cloud
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.farthest_point_sampling(torch.zeros(4, 3), 2, init_center=True)           # host tensor
    if torch.cuda.is_available():
        dev = torch.device("cuda")
        with pytest.raises(TypeError):
            ops.farthest_point_sampling(torch.zeros(4, 3, dtype=torch.float64, device=dev), 2, init_center=True)
        with pytest.raises(ValueError):
            ops.farthest_point_sampling(torch.zeros(4, 3, 2, device=dev), 2, init_center=True)
        with pytest.raises(ValueError):
            ops.farthest_point_sampling(torch.zeros(2, 4, 3, device=dev), 2, start=[0, 4])
    for sn in (0, -3, FPS_MAX_SAMPLES + 1):
        with pytest.raises(ValueError):
            ops.farthest_point_sampling(pts, sn, init_center=True)
    with pytest.raises(TypeError):
        ops.farthest_point_sampling(pts, 2.0, init_center=True)
    for start in (4, -1, [0, 1]):
        with pytest.raises(ValueError):
            ops.farthest_point_sampling(pts, 2, start=start)
    with pytest.raises(TypeError):
        ops.farthest_point_sampling(pts, 2, start=1.5)
    with pytest.raises(ValueError):
        ops.farthest_point_sampling(pts, 2, init_center=True, n_points=5)


@pytest.mark.parametrize("name", sorted(FC.objinfo_arrays()))
def test_objinfo_equals_reference_mesh_utils(golden, name, tmp_path):
    a = FC.objinfo_arrays()[name]
    c = objinfo.get_3D_bbox(a)
    want = golden["objinfo:%s:corners" % name]
    assert c.dtype == want.dtype and np.array_equal(c, want)
    r = objinfo.get_r(c)
    assert np.asarray(r).dtype == golden["objinfo:%s:radius" % name].dtype
    assert np.array_equal(r, golden["objinfo:%s:radius" % name])
    ctr = objinfo.get_centers_3d(c)
    assert ctr.dtype == golden["objinfo:%s:center" % name].dtype
    assert np.array_equal(ctr, golden["objinfo:%s:center" % name])
    info = dict(corners=c, radius=r, center=ctr, fps=a[:8])
    paths = objinfo.write_obj_info(info, str(tmp_path), name)
    for key in ("corners", "fps"):
        assert np.array_equal(np.loadtxt(paths[key], dtype=np.float32), np.asarray(info[key], np.float32))
    assert np.array_equal(np.loadtxt(paths["center"], dtype=np.float32), np.asarray(ctr, np.float32))


def test_oracle_builds_and_matches_golden(golden):
    if ref_loader.reference_sources_present():
        fps_oracle.build()
    elif not fps_oracle.available():
        pytest.skip("neither the reference's sources nor a built oracle/_ref/libfps_ref.so is present")
    for name in ("n33", "lattice_ties", "duplicates", "s_gt_p", "ycb_2621_kps"):
        make, S = FC.CASES[name]
        pts = make()
        assert np.array_equal(fps_oracle.fps(pts, S, init_center=True), golden[name + ":ic"])
        assert len(fps_oracle.fps(pts, S)) == S
