"""GPU: the tool's pyrender branch (``gen_obj_info.py --use_pyrender``) on the example cracker box (DESIGN.md §4.35),
with ORB and with SIFT: ``textured_kp3ds`` of a ``TexturedMeshTable`` equals the oracle composition -- the detector's
oracle on the device's renders, lifted with the centred poses -- bit for bit; ``gen_obj_info(points, 8,
mesh=table)`` is farthest point sampling of that cloud, and ``write_obj_info`` writes ``cracker_box_<ext>_fps.txt``."""
import numpy as np
import pytest

import ffb6d_b200 as F
from ffb6d_b200 import objinfo
from ffb6d_b200.render import TexturedMeshTable
from oracle import orb_oracle as O
from oracle import sift_oracle as S
import textured_cases as TC

pytestmark = pytest.mark.gpu

K = objinfo.TOOL_K


def _poses(points):
    """The pyrender branch's views: ``get_o2c_pose_cv(cam_pose, T(-mean))`` of the tool's sphere of cameras."""
    pts = np.asarray(points)
    T = np.eye(4)
    T[:3, 3] = -np.mean(pts.astype(np.float64), axis=0)
    r = objinfo.get_r(objinfo.get_3D_bbox(pts))
    cams = [objinfo.camera_pose(p) for p in objinfo.camera_positions(3, 3, r / 0.035 * 0.18)]
    return np.stack([objinfo.o2c_pose(c) @ T for c in cams])


@pytest.mark.parametrize("extractor", ["ORB", "SIFT"])
def test_box_pipeline_matches_oracle(extractor, tmp_path):
    points = TC.GOLDEN["points"]
    table = TexturedMeshTable([TC.box_mesh()])
    poses = _poses(points)
    assert np.array_equal(poses, objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(points)),
                                                      centre=np.mean(points.astype(np.float64), axis=0)))
    centre = np.mean(points.astype(np.float64), axis=0)
    r = objinfo.get_r(objinfo.get_3D_bbox(points))
    cloud, n_points, short = objinfo.textured_kp3ds(table, 0, radius=r, centre=centre, extractor=extractor)
    depth, rgb, _ = F.render_rgbd(table, np.zeros((9, 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                                  np.ones((9, 1), np.uint8), K, 480, 640)
    depth, rgb = depth.cpu().numpy(), rgb.cpu().numpy()
    detect = (lambda im: O.detect(im)["pt"]) if extractor == "ORB" else (lambda im: S.detect(im)["pt"])
    want = []
    for b in range(9):
        assert np.count_nonzero(depth[b] > 1e-8) >= O.MIN_RENDER_PIXELS
        want.append(O.lift(detect(rgb[b]), depth[b], K, poses[b])[0])
    want = np.concatenate(want).astype(np.float32)
    n = int(n_points[0])
    assert not short.any() and n == len(want) and n > 50, (n, len(want))
    got = cloud[0, :n].cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))

    info = objinfo.gen_obj_info(points, 8, start=0, mesh=table, textured_start=0, extractor=extractor)
    assert np.array_equal(info["textured_fps"], F.farthest_point_sampling(got, 8, start=0))
    assert len(info["short_views"]) == 0 and info["textured_fps"].shape == (8, 3)
    paths = objinfo.write_obj_info(info, str(tmp_path), "cracker_box")
    key = "%s_fps" % extractor
    assert paths[key].endswith("cracker_box_%s_fps.txt" % extractor)
    assert np.array_equal(np.loadtxt(paths[key], dtype=np.float32), info["textured_fps"])


def test_default_centre_is_the_tables_mean():
    table = TexturedMeshTable([TC.box_mesh()])
    xyz = table.xyz.cpu().numpy()
    a = objinfo.textured_kp3ds(table, 0)
    b = objinfo.textured_kp3ds(table, 0, centre=np.mean(xyz.astype(np.float64), axis=0))
    n = int(a[1][0])
    assert n == int(b[1][0]) and n > 0 and (a[0][0, :n] == b[0][0, :n]).all()
