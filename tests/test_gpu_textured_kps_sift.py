"""GPU: the textured keypoint pipeline with the tool's SIFT extractor (DESIGN.md §4.33) -- ``render_rgbd`` ->
``sift_detect`` -> ``sift_lift`` of the ape's sphere of views -- equals the oracle composition bit for bit and the
reference tool's SIFT-branch points (tests/golden/sift_cases.npz) to the bound DESIGN states;
``gen_obj_info(..., extractor="SIFT")`` and ``write_obj_info`` give ``<obj>_SIFT_fps.txt``; a view below 500 drawn
pixels is skipped and flagged; one CUDA-graph capture of render + detect + lift replays and equals the eager call."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import objinfo
from ffb6d_b200.render import RenderMeshTable
from oracle import orb_oracle as O
from oracle import sift_oracle as S
import orb_cases as OC
from test_sift_oracle import GOLDEN

pytestmark = pytest.mark.gpu

K = objinfo.TOOL_K


def renders(table, poses):
    return F.render_rgbd(table, np.zeros((len(poses), 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                         np.ones((len(poses), 1), np.uint8), K, 480, 640)


def oracle_cloud(depth, rgb, poses):
    pts = []
    for b in range(len(poses)):
        if np.count_nonzero(depth[b] > 1e-8) < O.MIN_RENDER_PIXELS:
            continue
        pts.append(O.lift(S.detect(rgb[b])["pt"], depth[b], K, poses[b])[0])
    return np.concatenate(pts).astype(np.float32) if pts else np.zeros((0, 3), np.float32)


def test_ape_pipeline_matches_oracle_and_reference():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    cloud, n_points, short = objinfo.textured_kp3ds(table, 0, extractor="SIFT")
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(xyz)))
    depth, img, _ = renders(table, poses)
    want = oracle_cloud(depth.cpu().numpy(), img.cpu().numpy(), poses)
    n = int(n_points[0])
    assert not short.any() and n == len(want) and n > 50
    got = cloud[0, :n].cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the reference tool's lifted points, as a multiset of float32 points
    ref = np.concatenate([GOLDEN["lift:ape%d" % v] for v in range(9)]).astype(np.float32)
    assert sorted(map(tuple, got.tolist())) == sorted(map(tuple, ref.tolist()))


def test_gen_obj_info_and_sift_file(tmp_path):
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    info = objinfo.gen_obj_info(xyz, 8, start=0, mesh=table, textured_start=0, extractor="SIFT")
    orb = objinfo.gen_obj_info(xyz, 8, start=0, mesh=table, textured_start=0)
    assert info["extractor"] == "SIFT" and "extractor" not in orb
    for k in ("corners", "radius", "center", "fps"):
        assert np.array_equal(info[k], orb[k])
    cloud, n_points, _ = objinfo.textured_kp3ds(table, 0, extractor="SIFT")
    want = F.farthest_point_sampling(cloud[0, :int(n_points[0])].cpu().numpy(), 8, start=0)
    assert info["textured_fps"].shape == (8, 3) and np.array_equal(info["textured_fps"], want)
    assert len(info["short_views"]) == 0
    paths = objinfo.write_obj_info(info, str(tmp_path), "ape")
    assert paths["SIFT_fps"].endswith("ape_SIFT_fps.txt") and "ORB_fps" not in paths
    assert np.array_equal(np.loadtxt(paths["SIFT_fps"], dtype=np.float32), info["textured_fps"])
    assert set(objinfo.write_obj_info(orb, str(tmp_path / "orb"), "ape")) == {"corners", "radius", "center", "fps",
                                                                              "ORB_fps"}


def test_short_view_is_skipped():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    radius = objinfo.get_r(objinfo.get_3D_bbox(xyz)) * np.float32(40)
    cloud, n_points, short = objinfo.textured_kp3ds(table, 0, radius=radius, extractor="SIFT")
    assert short.all() and int(n_points[0]) == 0


def test_graph_replay_equals_eager():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(xyz)))
    mesh_idx = torch.zeros((9, 1), dtype=torch.int32, device="cuda")
    RT32 = torch.from_numpy(poses[:, None, :3, :].astype(np.float32)).cuda()
    lab = torch.ones((9, 1), dtype=torch.uint8, device="cuda")
    Kd = torch.tensor([700.0, 700.0, 320.0, 240.0], dtype=torch.float64, device="cuda")
    RTd = torch.from_numpy(poses[:, :3, :]).cuda()

    def step():
        depth, img, _ = F.render_rgbd(table, mesh_idx, RT32, lab, Kd, 480, 640)
        count, pt = F.sift_detect(img, check=False)[:2]
        return F.sift_lift(count, pt, depth, Kd, RTd, 9), count, pt.shape[1]

    (eager, n_eager), count, cap = step()
    assert int(count.max()) <= cap
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                                   # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        (out, n_out), _, _ = step()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(n_out, n_eager)
    n = int(n_eager[0])
    assert torch.equal(out[:, :n], eager[:, :n])
