"""GPU: the textured keypoint pipeline (DESIGN.md §4.32) -- ``render_rgbd`` -> ``orb_detect`` -> ``orb_lift`` of the
ape's sphere of views -- equals the oracle composition bit for bit; ``gen_obj_info(mesh=...)``'s ``textured_fps``
equals ``farthest_point_sampling`` of the oracle's cloud; a view below 500 drawn pixels is skipped and flagged; one
CUDA-graph capture of detect + lift replays without a host sync and equals the eager call."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import objinfo
from ffb6d_b200.render import RenderMeshTable
from oracle import orb_oracle as O
import orb_cases as OC

pytestmark = pytest.mark.gpu

K = objinfo.TOOL_K


def oracle_cloud(depth, rgb, poses):
    pts = []
    for b in range(len(poses)):
        if np.count_nonzero(depth[b] > 1e-8) < O.MIN_RENDER_PIXELS:
            continue
        d = O.detect(rgb[b])
        pts.append(O.lift(d["pt"], depth[b], K, poses[b])[0])
    return np.concatenate(pts).astype(np.float32) if pts else np.zeros((0, 3), np.float32)


def test_ape_pipeline_matches_oracle():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    cloud, n_points, short = objinfo.textured_kp3ds(table, 0)
    radius = objinfo.get_r(objinfo.get_3D_bbox(xyz))
    poses = objinfo.sphere_poses(radius)
    # the oracle composition from the device's renders (the renderer is pinned by tests/test_gpu_render.py)
    depth, img, _ = F.render_rgbd(table, np.zeros((9, 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                                  np.ones((9, 1), np.uint8), K, 480, 640)
    want = oracle_cloud(depth.cpu().numpy(), img.cpu().numpy(), poses)
    n = int(n_points[0])
    assert not short.any() and n == len(want) and n > 100
    assert np.array_equal(cloud[0, :n].cpu().numpy().view(np.uint32), want.view(np.uint32))


def test_gen_obj_info_textured_fps():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    info = objinfo.gen_obj_info(xyz, 8, start=0, mesh=table, textured_start=3)
    plain = objinfo.gen_obj_info(xyz, 8, start=0)
    assert set(plain) == {"corners", "radius", "center", "fps"}
    for k in plain:
        assert np.array_equal(info[k], plain[k])
    cloud, n_points, _ = objinfo.textured_kp3ds(table, 0)
    want = F.farthest_point_sampling(cloud[0, :int(n_points[0])].cpu().numpy(), 8, start=3)
    assert info["textured_fps"].shape == (8, 3) and info["textured_fps"].dtype == np.float32
    assert np.array_equal(info["textured_fps"], want)
    assert len(info["short_views"]) == 0


def test_short_view_is_skipped(tmp_path):
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    # a sphere 40 times farther out: the ape covers a few dozen pixels in every view
    radius = objinfo.get_r(objinfo.get_3D_bbox(xyz)) * np.float32(40)
    cloud, n_points, short = objinfo.textured_kp3ds(table, 0, radius=radius)
    assert short.all() and int(n_points[0]) == 0
    info = dict(corners=np.zeros((8, 3)), radius=1.0, center=np.zeros(3), fps=np.zeros((8, 3)),
                textured_fps=np.ones((8, 3), np.float32))
    paths = objinfo.write_obj_info(info, str(tmp_path), "ape")
    assert np.array_equal(np.loadtxt(paths["ORB_fps"], dtype=np.float32), np.ones((8, 3), np.float32))


def test_graph_replay_equals_eager():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(xyz)))
    depth, img, _ = F.render_rgbd(table, np.zeros((9, 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                                  np.ones((9, 1), np.uint8), K, 480, 640)
    Kd = torch.tensor([700.0, 700.0, 320.0, 240.0], dtype=torch.float64, device="cuda")
    RTd = torch.from_numpy(poses[:, :3, :]).cuda()
    eager = F.orb_lift(*F.orb_detect(img)[:2], depth, Kd, RTd, 9)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        F.orb_lift(*F.orb_detect(img)[:2], depth, Kd, RTd, 9)          # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        count, pt, _, _ = F.orb_detect(img)
        out = F.orb_lift(count, pt, depth, Kd, RTd, 9)
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[1], eager[1])
    n = int(eager[1][0])
    assert torch.equal(out[0][:, :n], eager[0][:, :n])
