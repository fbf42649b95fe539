"""GPU: the textured rasteriser (DESIGN.md §4.35) is its oracle's bit for bit -- the example cracker box at the tool's
nine views, seeded noise and checker textures of 2048^2 at distances that reach deep levels and the last one, several
instances per frame (two of one mesh), per-frame cameras, inactive frames, ``out=``, 1 x 1 and odd frames, faces in
the drain queue -- its depth and labels are a vertex-coloured table's, its mip chains are the oracle's (up to the
16384-texel side limit), and one CUDA-graph capture replays equal to eager."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import objinfo
from ffb6d_b200.render import RenderMeshTable, TexturedMeshTable
from oracle import render_oracle as R
from oracle import textured_render_oracle as T
import textured_cases as TC

pytestmark = pytest.mark.gpu


def _kvec(K):
    K = np.asarray(K, np.float64)
    return np.stack([K[..., 0, 0], K[..., 1, 1], K[..., 0, 2], K[..., 1, 2]], -1)


def _check(table, meshes, mesh_idx, RTs, label, K, H, W, active=None):
    depth, rgb, lab = F.render_rgbd(table, mesh_idx, RTs, label, K, H, W, active=active)
    d, c, l = T.render(meshes, mesh_idx, RTs, label, _kvec(K), H, W, active=active)
    got = depth.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), d.view(np.uint32))
    assert np.array_equal(lab.cpu().numpy(), l)
    bad = np.nonzero((rgb.cpu().numpy() != c).any(-1))
    assert len(bad[0]) == 0, "%d pixels differ, first at %s" % (len(bad[0]), [b[:3] for b in bad])
    return depth, rgb, lab


def _pose(R3, t):
    return np.concatenate([np.asarray(R3, np.float64), np.reshape(t, (3, 1))], 1).astype(np.float32)


def _rot(ax, ay):
    cx, sx, cy, sy = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])


def test_box_at_the_tools_views():
    mesh = TC.box_mesh()
    table = TexturedMeshTable([mesh])
    pts = TC.GOLDEN["points"]
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(pts)), centre=np.mean(pts.astype(np.float64), 0))
    RT = poses[:, None, :3, :].astype(np.float32)
    depth, rgb, _ = _check(table, [mesh], np.zeros((9, 1), np.int32), RT, np.ones((9, 1), np.uint8), objinfo.TOOL_K,
                           480, 640)
    assert (torch.count_nonzero(depth > 0, dim=(1, 2)) > 2000).all()
    # depth and labels are a vertex-coloured table's of the same geometry
    flat = RenderMeshTable([(mesh[0], mesh[1], np.full(mesh[0].shape, 50, np.uint8))])
    d2, _, l2 = F.render_rgbd(flat, np.zeros((9, 1), np.int32), RT, np.ones((9, 1), np.uint8), objinfo.TOOL_K, 480, 640)
    assert torch.equal(depth.view(torch.int32), d2.view(torch.int32))


@pytest.mark.parametrize("kind", ["noise", "checker"])
def test_2048_textures_at_every_distance(kind):
    tex = TC.noise_texture(2048, 11) if kind == "noise" else TC.checker_texture(2048, 16)
    xyz, faces, uv, _ = TC.cuboid((-0.05, -0.05, -0.05), (0.05, 0.05, 0.05), tex, n=2)
    mesh = (xyz, faces, uv, tex)
    table = TexturedMeshTable([mesh])
    for l, lv in enumerate(T.mip_chain(tex)):
        assert np.array_equal(table.level(0, l).cpu().numpy(), lv), l
    # near (magnified) to far (a few pixels: the last levels), turned so each side is slanted
    dist = [0.12, 0.3, 1.0, 3.0, 12.0, 60.0]
    RT = np.stack([_pose(_rot(0.5 + 0.1 * k, 0.7 - 0.05 * k), (0.0, 0.0, z)) for k, z in enumerate(dist)])[:, None]
    K = np.array([[500.0, 0, 47.5], [0, 500.0, 40.0], [0, 0, 1]])
    _check(table, [mesh], np.zeros((len(dist), 1), np.int32), RT, np.full((len(dist), 1), 5, np.uint8), K, 81, 96)


def test_instances_cameras_inactive_and_out():
    box = TC.box_mesh(4)
    tex = TC.noise_texture(300, 2)[:300, :200]
    quad = (*TC.cuboid((-0.04, -0.03, -0.01), (0.04, 0.03, 0.01), tex, n=3)[:3], tex)
    meshes = [box, quad]
    table = TexturedMeshTable(meshes)
    B, M = 4, 3
    mesh_idx = np.array([[0, 1, 0], [1, -1, 1], [0, 0, 0], [-1, -1, 1]], np.int32)
    rng = np.random.default_rng(0)
    RT = np.stack([[_pose(_rot(*rng.uniform(-1, 1, 2)), (rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05),
                                                         rng.uniform(0.35, 0.6))) for _ in range(M)]
                   for _ in range(B)])
    label = np.arange(1, B * M + 1, dtype=np.uint8).reshape(B, M)
    K = np.stack([np.array([[600.0 + 10 * b, 0, 63.5 + b], [0, 590.0, 48.0 - b], [0, 0, 1]]) for b in range(B)])
    active = np.array([True, True, False, True])
    _check(table, meshes, mesh_idx, RT, label, K, 97, 129, active=active)
    # out=: dpt_mm, written in place; the inactive frame keeps what it held
    dev = table.device
    out = (torch.full((B, 97, 129), 7, dtype=torch.uint16, device=dev),
           torch.full((B, 97, 129, 3), 7, dtype=torch.uint8, device=dev),
           torch.full((B, 97, 129), 7, dtype=torch.uint8, device=dev))
    F.render_rgbd(table, mesh_idx, RT, label, K, 97, 129, active=active, out=out)
    d, c, l = T.render(meshes, mesh_idx, RT, label, _kvec(K), 97, 129)
    on = active
    assert np.array_equal(out[0].cpu().numpy()[on], R.dpt_mm(d)[on]) and (out[0][2] == 7).all()
    assert np.array_equal(out[1].cpu().numpy()[on], c[on]) and np.array_equal(out[2].cpu().numpy()[on], l[on])


@pytest.mark.parametrize("H, W", [(1, 1), (3, 7), (45, 1), (33, 65)])
def test_small_and_odd_frames_and_the_drain_queue(H, W):
    # a screen-filling quad: both faces' boxes hold more than 256 pixels at 33 x 65, so they are drawn by the drain
    tex = TC.noise_texture(64, 9)[:40, :64]
    xyz, faces, uv = TC.screen_quad(W, H, x0=-0.75, y0=-0.625, x1=W - 0.25, y1=H - 0.375, uv0=(-0.3, 0.2),
                                    uv1=(1.7, 2.9))
    mesh = (xyz, faces, uv, tex)
    table = TexturedMeshTable([mesh])
    K = np.eye(3)
    _check(table, [mesh], np.zeros((2, 1), np.int32), np.stack([TC.IDENTITY, TC.IDENTITY])[:, None],
           np.ones((2, 1), np.uint8), K, H, W)


def test_side_limit_table():
    side = F._lib.RND_MAX_TEX_SIDE
    rng = np.random.default_rng(21)
    texs = [rng.integers(0, 256, (4, side, 3), dtype=np.uint8), rng.integers(0, 256, (side, 3, 3), dtype=np.uint8)]
    meshes = [(*TC.screen_quad(40, 30)[:3], texs[0]), (*TC.screen_quad(40, 30, x1=2.5, y1=30.5)[:3], texs[1])]
    table = TexturedMeshTable(meshes)
    assert table.max_tex_side == side
    for m, tex in enumerate(texs):
        chain = T.mip_chain(tex)
        assert len(chain) == F._lib.RND_MAX_TEX_LEVELS
        for l, lv in enumerate(chain):
            assert np.array_equal(table.level(m, l).cpu().numpy(), lv), (m, l)
    _check(table, meshes, np.array([[0], [1]], np.int32), np.stack([TC.IDENTITY] * 2)[:, None],
           np.ones((2, 1), np.uint8), np.eye(3), 30, 40)


def test_graph_replay_equals_eager():
    mesh = TC.box_mesh()
    table = TexturedMeshTable([mesh])
    pts = TC.GOLDEN["points"]
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(pts)), centre=pts.astype(np.float64).mean(0))
    mesh_idx = torch.zeros((9, 1), dtype=torch.int32, device="cuda")
    RT = torch.from_numpy(poses[:, None, :3, :].astype(np.float32)).cuda()
    lab = torch.ones((9, 1), dtype=torch.uint8, device="cuda")
    Kd = torch.tensor([700.0, 700.0, 320.0, 240.0], dtype=torch.float64, device="cuda")
    eager = F.render_rgbd(table, mesh_idx, RT, lab, Kd, 480, 640)
    out = tuple(torch.zeros_like(t) for t in (eager[0].to(torch.uint16), eager[1], eager[2]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        F.render_rgbd(table, mesh_idx, RT, lab, Kd, 480, 640, out=out)
    torch.cuda.current_stream().wait_stream(s)
    for t in out:
        t.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        F.render_rgbd(table, mesh_idx, RT, lab, Kd, 480, 640, out=out)
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out[0].cpu().numpy(), R.dpt_mm(eager[0].cpu().numpy()))
    assert torch.equal(out[1], eager[1]) and torch.equal(out[2], eager[2])
