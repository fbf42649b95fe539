"""GPU: ``render_rgbd`` (``ffb6d_render_rgbd``, DESIGN.md §4.31) equals oracle/render_oracle.py bit for bit: the
reference's example ape mesh at several poses with shared and per-frame cameras, several instances per frame,
full-screen and close-up faces (the raster queue), vertices on pixel samples and edges, empty, culled and odd-sized
frames, inactive frames; the ``dpt_mm`` output; repeatability; a call at each checked limit."""
import os

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import GOLDEN
from ffb6d_b200 import _lib
from ffb6d_b200.render import RenderMeshTable
from ffb6d_b200.synthetic import INTRINSICS
from oracle import render_oracle as R

pytestmark = pytest.mark.gpu

H, W = 480, 640
EYE = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
K_SMALL = np.array([[143.1, 0.0, 80.3], [0.0, 143.4, 60.5], [0.0, 0.0, 1.0]])      # LineMOD's camera at 1/4 size


def ape():
    z = np.load(os.path.join(GOLDEN, "render_ape.npz"))
    return z["xyz"] / np.float32(1000.0), z["faces"], z["rgb"]


def fxfy(K):
    K = np.asarray(K, np.float64)
    return np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])


def rotation(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    a, b, c, d = q
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def pose(rs, z, spread=0.05):
    t = np.array([rs.uniform(-spread, spread), rs.uniform(-spread, spread), z])
    return np.concatenate([rotation(rs), t[:, None]], 1).astype(np.float32)


def check(meshes, mesh_idx, RTs, label, K, h=H, w=W, z_near=0.01, active=None):
    """render_rgbd against the oracle, both outputs; returns the depth map."""
    table = RenderMeshTable(meshes)
    mesh_idx = np.asarray(mesh_idx, np.int32)
    Kd = fxfy(K) if np.ndim(K) == 2 else np.stack([fxfy(k) for k in K])
    want = R.render(meshes, mesh_idx, RTs, label, Kd, h, w, z_near, active)
    midx = torch.from_numpy(mesh_idx).cuda()
    got = F.render_rgbd(table, midx, np.asarray(RTs, np.float32), np.asarray(label, np.uint8), K, h, w,
                        z_near=z_near, active=active)
    for g, wnt, name in zip(got, want, ("depth", "rgb", "labels")):
        g = g.cpu().numpy()
        assert g.dtype == wnt.dtype and np.array_equal(g.view(np.uint8), wnt.view(np.uint8)), \
            (name, int((g != wnt).sum()))
    B = mesh_idx.shape[0]
    out = (torch.zeros((B, h, w), dtype=torch.uint16, device="cuda"),
           torch.zeros((B, h, w, 3), dtype=torch.uint8, device="cuda"),
           torch.zeros((B, h, w), dtype=torch.uint8, device="cuda"))
    r = F.render_rgbd(table, midx, RTs, label, K, h, w, z_near=z_near, active=active, out=out)
    assert all(a is b for a, b in zip(r, out))
    assert np.array_equal(out[0].cpu().numpy(), R.dpt_mm(want[0]))
    assert torch.equal(out[1], got[1]) and torch.equal(out[2], got[2])
    return want[0]


def test_ape_at_several_poses_shared_and_per_frame_K(cuda):
    rs = np.random.RandomState(0)
    B = 4
    RTs = np.stack([pose(rs, z) for z in (0.3, 0.5, 0.8, 1.2)])[:, None]
    K = INTRINSICS["linemod"]
    d = check([ape()], np.zeros((B, 1)), RTs, np.ones((B, 1)), K)
    assert all((d[b] > 0).sum() > 500 for b in range(B))
    Ks = np.stack([INTRINSICS["linemod"], INTRINSICS["ycb_K1"], INTRINSICS["ycb_K2"], INTRINSICS["linemod"]])
    xyz, faces, rgb = ape()
    # column-major arrays are packed row-major by the table
    check([(np.asfortranarray(xyz), np.asfortranarray(faces), np.asfortranarray(rgb))], np.zeros((B, 1)), RTs,
          np.ones((B, 1)), Ks)


def test_several_instances_per_frame(cuda):
    rs = np.random.RandomState(1)
    xyz, faces, rgb = ape()
    box = (np.array([[-1, -1, 0], [1, -1, 0], [1, 1, 0], [-1, 1, 0]], np.float32) * np.float32(0.06),
           np.array([[0, 1, 2], [0, 2, 3]]), np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0]], np.uint8))
    B, M = 3, 4
    mesh_idx = np.array([[0, 0, 1, -1], [1, 0, -1, 0], [-1, -1, 0, 1]])
    RTs = np.stack([np.stack([pose(rs, rs.uniform(0.4, 0.7), 0.03) for _ in range(M)]) for _ in range(B)])
    d = check([(xyz, faces, rgb), box], mesh_idx, RTs, np.arange(1, B * M + 1).reshape(B, M), INTRINSICS["linemod"])
    assert all((d[b] > 0).any() for b in range(B))
    # indices outside the table, read on the device, draw nothing for their slot
    bad = np.array([[0, 7, -5, 2], [2, 2, 2, 2], [1, -1, 0, 99]])
    want = R.render([(xyz, faces, rgb), box], bad, RTs, np.ones((B, M)), fxfy(INTRINSICS["linemod"]), H, W)
    got = F.render_rgbd(RenderMeshTable([(xyz, faces, rgb), box]), torch.from_numpy(bad.astype(np.int32)).cuda(), RTs,
                        np.ones((B, M), np.uint8), INTRINSICS["linemod"], H, W)
    assert not got[0][1].any()
    assert all(np.array_equal(g.cpu().numpy(), wnt) for g, wnt in zip(got, want))


def test_full_screen_and_close_up_faces(cuda):
    # a quad larger than the frame at 2 m and the ape at 8 cm: faces far beyond the queue threshold
    rs = np.random.RandomState(2)
    quad = (np.array([[-3, -3, 0], [3, -3, 0.5], [3, 3, 1.0], [-3, 3, 0]], np.float32),
            np.array([[0, 1, 2], [0, 2, 3]]), np.array([[250, 10, 10], [10, 250, 10], [10, 10, 250], [90, 90, 90]],
                                                       np.uint8))
    RTs = np.stack([np.stack([pose(rs, 0.08, 0.0), EYE]), np.stack([EYE, EYE])])
    RTs[1, 1, 2, 3] = 2.0
    RTs[0, 1, 2, 3] = 2.0
    d = check([ape(), quad], [[0, 1], [-1, 1]], RTs, [[1, 2], [1, 2]], INTRINSICS["linemod"])
    assert (d[1] > 0).all()
    assert (d[0] < 0.5).sum() > 20000


def test_vertices_on_pixel_samples_and_edges(cuda):
    # a 12 x 12 grid of cells whose vertices lie on pixel samples and half-pixel edges, random depths
    rs = np.random.RandomState(3)
    K = np.array([[256.0, 0, 0], [0, 256.0, 0], [0, 0, 1]])
    n = 12
    gu, gv = np.linspace(4, 40, n + 1), np.linspace(3, 33, n + 1)
    uv = np.stack(np.meshgrid(gu, gv), -1).reshape(-1, 2)
    z = rs.uniform(0.5, 2.0, len(uv)).astype(np.float32).astype(np.float64)
    xyz = np.stack([uv[:, 0] / 256 * z, uv[:, 1] / 256 * z, z], 1).astype(np.float32)
    faces = []
    for r in range(n):
        for c in range(n):
            a, b, e, f = r * (n + 1) + c, r * (n + 1) + c + 1, (r + 1) * (n + 1) + c, (r + 1) * (n + 1) + c + 1
            faces += [[a, b, f], [a, f, e]] if (r + c) % 2 else [[a, b, e], [b, f, e]]
    faces = np.array(faces)
    faces[::3] = faces[::3, ::-1]
    mesh = (xyz, faces, rs.randint(0, 256, (len(uv), 3)).astype(np.uint8))
    d = check([mesh], [[0], [0]], np.stack([EYE, EYE])[:, None], [[1], [2]], K, h=37, w=45)
    assert (d[0] > 0).sum() == 36 * 30


def test_empty_culled_and_odd_frames(cuda):
    rs = np.random.RandomState(4)
    behind = pose(rs, -0.5)                           # every vertex behind the near plane
    aside = pose(rs, 0.5)
    aside[0, 3] = 100.0                               # every vertex outside the guard band
    RTs = np.stack([pose(rs, 0.5), behind, aside, pose(rs, 0.6)])[:, None]
    d = check([ape()], [[-1], [0], [0], [0]], RTs, np.ones((4, 1)), K_SMALL, h=121, w=161)
    assert not d[:3].any() and d[3].any()
    check([ape()], [[0], [0]], RTs[[0, 3]], np.ones((2, 1)), INTRINSICS["linemod"], h=1, w=1)
    check([ape()], [[0]], RTs[[0]], np.ones((1, 1)), INTRINSICS["linemod"], h=481, w=641, z_near=0.4)


def test_non_finite_vertices_and_poses_cull_their_faces(cuda):
    # faces in view, one vertex made infinite or NaN per face; a pose with an infinite translation culls everything
    rs = np.random.RandomState(7)
    xyz, faces, rgb = ape()
    bad = xyz.copy()
    bad[faces[::5, 0], 2] = np.inf
    bad[faces[1::5, 1], 0] = -np.inf
    bad[faces[2::5, 2], 1] = np.nan
    RTs = np.stack([pose(rs, 0.5), pose(rs, 0.6), pose(rs, 0.4)])[:, None]
    RTs[2, 0, 2, 3] = np.inf
    d = check([(bad, faces, rgb)], np.zeros((3, 1)), RTs, np.ones((3, 1)), INTRINSICS["linemod"])
    assert d[0].any() and d[1].any() and not d[2].any()


def test_inactive_frames_are_untouched(cuda):
    rs = np.random.RandomState(5)
    B = 4
    RTs = np.stack([pose(rs, 0.5) for _ in range(B)])[:, None]
    active = np.array([True, False, True, False])
    check([ape()], np.zeros((B, 1)), RTs, np.ones((B, 1)), INTRINSICS["linemod"], active=active)
    table = RenderMeshTable([ape()])
    g = torch.Generator(device="cuda").manual_seed(0)
    out = (torch.randint(0, 65535, (B, H, W), dtype=torch.int32, device="cuda", generator=g).to(torch.uint16),
           torch.randint(0, 255, (B, H, W, 3), dtype=torch.uint8, device="cuda", generator=g),
           torch.randint(0, 255, (B, H, W), dtype=torch.uint8, device="cuda", generator=g))
    before = [t.clone() for t in out]
    want = R.render([ape()], np.zeros((B, 1), np.int32), RTs, np.ones((B, 1)), fxfy(INTRINSICS["linemod"]), H, W)
    for act in (active, torch.from_numpy(active).cuda()):
        F.render_rgbd(table, np.zeros((B, 1), np.int32), RTs, np.ones((B, 1), np.uint8), INTRINSICS["linemod"], H, W,
                      active=act, out=out)
        for b in range(B):
            if active[b]:
                assert np.array_equal(out[0][b].cpu().numpy(), R.dpt_mm(want[0][b]))
                assert np.array_equal(out[1][b].cpu().numpy(), want[1][b])
            else:
                assert all(torch.equal(t[b], u[b]) for t, u in zip(out, before)), b


def test_two_calls_are_bitwise_equal(cuda):
    rs = np.random.RandomState(6)
    table = RenderMeshTable([ape()])
    B, M = 8, 3
    RTs = np.stack([np.stack([pose(rs, rs.uniform(0.2, 0.6), 0.04) for _ in range(M)]) for _ in range(B)])
    args = (table, np.zeros((B, M), np.int32), RTs, np.ones((B, M), np.uint8), INTRINSICS["linemod"], H, W)
    a, b = F.render_rgbd(*args), F.render_rgbd(*args)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def _point_mesh(n_faces=1):
    """A triangle that draws one pixel at the image origin, and ``n_faces - 1`` zero-area copies."""
    xyz = np.array([[-0.001, -0.001, 1], [0.002, -0.001, 1], [-0.001, 0.002, 1]], np.float32)
    faces = np.zeros((n_faces, 3), np.int32)
    faces[0] = [0, 1, 2]
    return xyz, faces, np.full((3, 3), 200, np.uint8)


def test_each_checked_limit_is_admitted(cuda):
    K = np.array([[256.0, 0, 0], [0, 256.0, 0], [0, 0, 1]])

    def run(B, M, h, w, mesh, mesh_idx=None):
        table = RenderMeshTable([mesh])
        mi = torch.zeros((B, M), dtype=torch.int32, device="cuda") if mesh_idx is None else mesh_idx
        RTs = torch.from_numpy(EYE).cuda().expand(B, M, 3, 4).contiguous()
        lab = torch.ones((B, M), dtype=torch.uint8, device="cuda")
        out = (torch.empty((B, h, w), dtype=torch.uint16, device="cuda"),
               torch.empty((B, h, w, 3), dtype=torch.uint8, device="cuda"),
               torch.empty((B, h, w), dtype=torch.uint8, device="cuda"))
        F.render_rgbd(table, mi, RTs, lab, K, h, w, z_near=0.001, out=out)
        return out

    d, c, l = run(_lib.RND_MAX_FRAMES, 1, 1, 1, _point_mesh())
    assert (d.to(torch.int32) == 1000).all() and (c == 200).all() and (l == 1).all()
    del d, c, l
    d, c, l = run(1, 1, 1, _lib.RND_MAX_FRAME_PIXELS, _point_mesh())
    assert d[0, 0, 0].item() == 1000
    assert not d[0, 0, 1:1 << 20].to(torch.int32).any() and not d[0, 0, -(1 << 20):].to(torch.int32).any()
    del d, c, l
    torch.cuda.empty_cache()
    # the most slots, and the most faces per frame (slots x the largest mesh's faces = 2^32): one slot draws, the
    # others are empty
    mi = torch.full((1, _lib.RND_MAX_SLOTS), -1, dtype=torch.int32, device="cuda")
    mi[0, -1] = 0
    n_faces = _lib.RND_MAX_FRAME_FACES // _lib.RND_MAX_SLOTS
    d, c, l = run(1, _lib.RND_MAX_SLOTS, 4, 4, _point_mesh(n_faces), mi)
    assert d[0, 0, 0].item() == 1000 and (d.to(torch.int32) > 0).sum().item() == 1 and l[0, 0, 0].item() == 1
    torch.cuda.synchronize()
