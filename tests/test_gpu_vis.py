"""GPU: pose and label drawing (``ffb6d_project_p3d``, ``ffb6d_draw_p2ds`` and ``ffb6d_b200.vis``) bitwise against
the numpy restatement of oracle/vis_oracle.py and the reference's outputs in tests/golden/vis_cases.npz."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import vis_cases as VC
from oracle import vis_oracle as O

pytestmark = pytest.mark.gpu

I32_MIN = np.iinfo(np.int32).min


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "vis_cases.npz"))
    return {k: z[k] for k in z.files}


def _t(a, dev, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dev) if dtype is None else \
        torch.as_tensor(np.ascontiguousarray(a)).to(dev, dtype)


def _project(cuda, p, cs, K, pose):
    n = len(p)
    one = lambda v: torch.tensor([v], dtype=torch.int32, device=cuda)        # noqa: E731
    pt = _t(pose[None], cuda, torch.float64) if pose is not None else None
    return F_ops().project_p3d(_t(p, cuda), one(0), one(n), n, _t(K, cuda, torch.float64), cs, pt)[0].cpu().numpy()


def F_ops():
    from ffb6d_b200 import ops
    return ops


def test_projection_cases(cuda, golden):
    from ffb6d_b200 import vis
    for name, (p, cs, K, pose) in VC.proj_cases().items():
        want = O.project_p3d(p, cs, K, pose)
        got = _project(cuda, p, cs, K, pose)
        assert np.array_equal(got, want), name
        key = "proj:" + name
        assert VC.sha(got) == str(golden[key + ":sha256"]) if key + ":sha256" in golden else \
            np.array_equal(got, golden[key]), name
        if pose is None:
            assert np.array_equal(vis.project_p3d(p, cs, K).cpu().numpy(), want), name
            assert np.array_equal(vis.project_p3d(_t(p, cuda), cs, K).cpu().numpy(), want), name


def test_projection_set_table(cuda):
    """Several sets in one call: per-set K and scale, poses, padding, disabled sets and bad rows."""
    ops = F_ops()
    rs = np.random.RandomState(1)
    table = np.concatenate([VC.mesh(rs, n, np.float64) for n in (40, 7, 100, 1)])
    start = np.array([0, 40, 47, 147, 140, -1, 100, 0], np.int32)
    count = np.array([40, 7, 100, 1, 10, 3, 60, 0], np.int32)
    enable = np.array([1, 1, 1, 1, 1, 1, 0, 1], np.uint8)
    S, max_rows = len(start), 100
    K = np.stack([VC.K_YCB, VC.K_LM] * 4)
    cs = np.array([1.0, 0.5, 2.0, 1.0, 1.0, 1.0, 1.0, 1.0])
    poses = np.stack([VC.pose_in_front(rs) for _ in range(S)])
    for f64 in (True, False):
        tab = table if f64 else table.astype(np.float32)
        for with_pose in (True, False):
            got = ops.project_p3d(_t(tab, cuda), _t(start, cuda), _t(count, cuda), max_rows, _t(K, cuda), _t(cs, cuda),
                                  _t(poses, cuda) if with_pose else None, _t(enable, cuda)).cpu().numpy()
            for s in range(S):
                ok = enable[s] and start[s] >= 0 and start[s] + count[s] <= len(tab) and count[s] <= max_rows
                n = count[s] if ok else 0
                if n:
                    want = O.project_p3d(tab[start[s]:start[s] + n], cs[s], K[s], poses[s] if with_pose else None)
                    assert np.array_equal(got[s, :n], want), (s, f64, with_pose)
                assert (got[s, n:] == I32_MIN).all(), s
    # count beyond max_rows: the set is empty
    got = ops.project_p3d(_t(table, cuda), _t(start[:1], cuda), _t(count[:1], cuda), 39, _t(VC.K_YCB, cuda), 1.0)
    assert (got.cpu().numpy() == I32_MIN).all()


def test_projection_nonfinite_and_far(cuda):
    rs = np.random.RandomState(2)
    p = rs.normal(0, 1, (3000, 3)) * 10.0 ** rs.randint(-12, 14, (3000, 1))
    p[rs.rand(3000) < 0.05, 0] = np.nan
    p[rs.rand(3000) < 0.05, 2] = np.inf
    p[rs.rand(3000) < 0.05, 2] = 0.0
    p[rs.rand(3000) < 0.05, 2] *= -1
    for dt in (np.float32, np.float64):
        q = p.astype(dt)
        for pose in (None, VC.pose_in_front(rs)):
            with np.errstate(all="ignore"):
                want = O.project_p3d(q, 1.0, VC.K_YCB, pose)
            got = _project(cuda, q, 1.0, VC.K_YCB, pose)
            assert np.array_equal(got, want), (dt, pose is None)
            assert (got == I32_MIN).any() and (got != I32_MIN).any()


def test_golden_drawing(cuda, golden):
    from ffb6d_b200 import vis
    for name, (bg, sets) in VC.draw_cases().items():
        img = _t(bg, cuda)
        for p2ds, r, cols in sets:
            vis.draw_p2ds(img, p2ds, r, list(cols))
        assert np.array_equal(img.cpu().numpy(), golden["draw:" + name]), name
        if name.startswith("overlap"):            # the same sets in one call: per-row colours, set order kept
            ops = F_ops()
            S, max_rows = len(sets), max(len(p) for p, _, _ in sets)
            p2ds = np.zeros((S, max_rows, 2), np.int32)
            col = np.zeros((S, max_rows, 3), np.uint8)
            for s, (p, _, c) in enumerate(sets):
                p2ds[s, :len(p)] = p
                col[s, :len(p)] = np.broadcast_to(np.asarray(c, np.uint8).reshape(-1, 3), (len(p), 3))
            count = np.array([len(p) for p, _, _ in sets], np.int32)
            img = _t(bg, cuda)[None].contiguous()
            ops.draw_p2ds(img, _t(p2ds, cuda), torch.zeros(S, dtype=torch.int32, device=cuda),
                          torch.zeros(S, dtype=torch.int32, device=cuda), _t(count, cuda), max_rows,
                          _t(np.array([r for _, r, _ in sets], np.int32), cuda), _t(col, cuda))
            assert np.array_equal(img[0].cpu().numpy(), golden["draw:" + name]), name


def _random_sets(rs, B, H, W, S, max_rows, radii):
    p2ds = np.stack((rs.randint(-8, W + 8, (S, max_rows)), rs.randint(-8, H + 8, (S, max_rows))), -1).astype(np.int32)
    p2ds[rs.rand(S, max_rows) < 0.05] = I32_MIN
    p2ds[rs.rand(S, max_rows) < 0.05, 0] = W
    p2ds[rs.rand(S, max_rows) < 0.05, 1] = H
    frame = rs.randint(0, B, S).astype(np.int32)
    count = rs.randint(0, max_rows + 1, S).astype(np.int32)
    radius = np.asarray(radii, np.int32)[rs.randint(0, len(radii), S)]
    return p2ds, frame, count, radius


def test_drawing_against_oracle(cuda):
    ops = F_ops()
    rs = np.random.RandomState(3)
    B, H, W, S, max_rows = 3, 37, 53, 24, 30
    for trial in range(6):
        p2ds, frame, count, radius = _random_sets(rs, B, H, W, S, max_rows, (0, 1, 2, 3, 4, 64) if trial < 3 else
                                                  (0, 1, 2, 3, 4))
        start = np.zeros(S, np.int32)
        enable = (rs.rand(S) > 0.2).astype(np.uint8)
        bad = rs.rand(S) < 0.15
        frame[rs.rand(S) < 0.05] = B                  # a frame out of range draws nothing
        radius[rs.rand(S) < 0.05] = 65                # so does a radius out of range
        start[bad] = rs.choice([-1, 5, 10 ** 6], bad.sum())
        n_rows = max_rows + 5
        per_row = trial % 2 == 1
        col = rs.randint(0, 256, (S, max_rows, 3) if per_row else (S, 3)).astype(np.uint8)
        bg = rs.randint(0, 256, (B, H, W, 3)).astype(np.uint8)
        img = _t(bg, cuda)
        ops.draw_p2ds(img, _t(p2ds, cuda), _t(frame, cuda), _t(start, cuda), _t(count, cuda), n_rows,
                      _t(radius, cuda), _t(col, cuda), _t(enable, cuda))
        sets = []
        for s in range(S):
            ok = enable[s] and 0 <= start[s] and start[s] + count[s] <= n_rows and 0 <= frame[s] < B and \
                radius[s] <= 64
            if ok:
                sets.append((frame[s], p2ds[s, :count[s]], radius[s], col[s, :count[s]] if per_row else col[s]))
        want = O.draw_sets(bg.copy(), sets)
        assert np.array_equal(img.cpu().numpy(), want), trial


def test_size_limits(cuda):
    ops = F_ops()
    rs = np.random.RandomState(4)
    for H, W in ((1, 16384), (16384, 1), (480, 640)):
        B, S, max_rows = 1, 3, 50
        p2ds, frame, count, _ = _random_sets(rs, B, H, W, S, max_rows, (0,))
        radius = np.array([64, 3, 1], np.int32)
        col = rs.randint(0, 256, (S, 3)).astype(np.uint8)
        img = torch.zeros((B, H, W, 3), dtype=torch.uint8, device=cuda)
        ops.draw_p2ds(img, _t(p2ds, cuda), _t(frame, cuda), torch.zeros(S, dtype=torch.int32, device=cuda),
                      _t(count, cuda), max_rows, _t(radius, cuda), _t(col, cuda))
        want = O.draw_sets(np.zeros((B, H, W, 3), np.uint8),
                           [(frame[s], p2ds[s, :count[s]], radius[s], col[s]) for s in range(S)])
        assert np.array_equal(img.cpu().numpy(), want), (H, W)


def test_no_allocation(cuda):
    ops = F_ops()
    rs = np.random.RandomState(5)
    B, H, W, S, max_rows = 2, 48, 64, 5, 40
    p2ds, frame, count, radius = _random_sets(rs, B, H, W, S, max_rows, (1, 3))
    args = [_t(a, cuda) for a in (p2ds, frame, np.zeros(S, np.int32), count)]
    img = torch.zeros((B, H, W, 3), dtype=torch.uint8, device=cuda)
    rad, col = _t(radius, cuda), _t(rs.randint(0, 256, (S, 3)).astype(np.uint8), cuda)
    ws = ops.draw_p2ds_workspace(img)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(cuda)
    ops.draw_p2ds(img, *args, max_rows, rad, col, ws=ws)
    assert torch.cuda.memory_allocated(cuda) == before


# ------------------------------------------------------------------------------------------- demo and debug views
def test_golden_demo_and_view_labels(cuda, golden):
    from ffb6d_b200 import pose, vis
    for ds, f in VC.demo_frames().items():
        table = pose.MeshTable(f["mesh_pts"], cuda, torch.float64)
        n_cls = 22
        present = torch.zeros((1, n_cls), dtype=torch.bool, device=cuda)
        poses = torch.zeros((1, n_cls, 3, 4), dtype=torch.float64, device=cuda)
        if ds == "ycb":
            for c, P in zip(f["pred_cls_ids"], f["pred_pose_lst"]):
                present[0, c] = True
                poses[0, c] = _t(P, cuda)
            colors = [vis.get_label_color(c, n_obj=22, mode=2) for c in range(n_cls)]
            img = _t(f["rgb"].astype(np.uint8).transpose(1, 2, 0)[:, :, ::-1], cuda)[None].contiguous()
            vis.draw_poses(img, table, _t(f["cls_ids"][None], cuda), present, poses, f["K"], colors)
        else:
            present[0, 1] = True
            poses[0, 1] = _t(f["pred_pose_lst"][0], cuda)
            colors = [(0, 0, 0), vis.get_label_color(f["obj_id"], n_obj=22, mode=2)] + [(0, 0, 0)] * 20
            mesh_ids = torch.full((n_cls,), -1, dtype=torch.long, device=cuda)
            mesh_ids[1] = f["obj_id"]
            img = _t(f["rgb"].astype(np.uint8).transpose(1, 2, 0), cuda)[None].contiguous()
            vis.draw_poses(img, table, _t(f["cls_ids"][None], cuda), present, poses, f["K"], colors,
                           mesh_ids=mesh_ids)
            img = img.flip(-1)
        assert VC.sha(img[0].cpu().numpy()) == str(golden["demo:%s:sha256" % ds]), ds
    cld, labels = VC.view_labels_frame()
    out = vis.view_labels(torch.zeros((1, 3, 480, 640), device=cuda), _t(cld[None], cuda), _t(labels[None], cuda),
                          VC.K_YCB)
    assert VC.sha(out[0].cpu().numpy()) == str(golden["view_labels:sha256"])


def _net_batch(cuda, B, seed, dataset):
    from ffb6d_b200.synthetic import make_pose_batch
    pb = make_pose_batch(seed, B, n_points=8192, n_objects=4)
    rs = np.random.RandomState(seed)
    n_cls, N = 22, pb["mask"].shape[1]
    segs = np.full((B, n_cls, N), -1.0, np.float32)
    np.put_along_axis(segs, pb["mask"][:, None, :], 1.0, axis=1)
    ep = {"pred_rgbd_segs": _t(segs, cuda), "pred_ctr_ofs": _t(pb["ctr_of"], cuda), "pred_kp_ofs": _t(pb["kp_of"], cuda)}
    cld = np.concatenate((pb["pcld"].transpose(0, 2, 1), rs.uniform(0, 1, (B, 6, N)).astype(np.float32)), 1)
    ids = np.zeros((B, 22, 1), np.int32)
    for b in range(B):
        if dataset == "ycb":
            cls = [c for c in np.unique(pb["mask"][b]) if c] + [21 if 21 not in pb["mask"][b] else 20]
            ids[b, :len(cls), 0] = rs.permutation(cls)
        else:
            ids[b, 0, 0] = 1
    item = {"rgb": _t(rs.randint(0, 256, (B, 3, 480, 640)).astype(np.float32), cuda), "cld_rgb_nrm": _t(cld, cuda),
            "cls_ids": _t(ids, cuda)}
    meshes = {c: VC.mesh(rs, 2621, np.float32) for c in range(1, n_cls)}
    return pb, ep, item, meshes


class _Net(torch.nn.Module):
    def __init__(self, ep):
        super().__init__()
        self.ep = ep

    def forward(self, item):
        return self.ep


def test_cal_view_pred_pose_ycb(cuda):
    from ffb6d_b200 import pose, vis
    B = 3
    pb, ep, item, meshes = _net_batch(cuda, B, 31, "ycb")
    got = vis.cal_view_pred_pose(_Net(ep), item, dataset="ycb", mesh_pts=meshes, mesh_kps=pb["mesh"],
                                 cls_radius=pb["cls_radius"], K=VC.K_YCB).cpu().numpy()
    pcld = item["cld_rgb_nrm"][:, :3].permute(0, 2, 1).contiguous()
    mask = ep["pred_rgbd_segs"].argmax(1)
    for b in range(B):
        ids, poses, _ = pose.cal_frame_poses(pcld[b], mask[b], ep["pred_ctr_ofs"][b], ep["pred_kp_ofs"][b], True, 22,
                                             True, mesh_kps=pb["mesh"], cls_radius=pb["cls_radius"])
        want = O.demo_draw(item["rgb"][b].cpu().numpy(), item["cls_ids"][b].cpu().numpy(), ids, poses, meshes,
                           VC.K_YCB, "ycb")
        assert np.array_equal(got[b], want), b
        assert (got[b] != item["rgb"][b].cpu().numpy().astype(np.uint8).transpose(1, 2, 0)[:, :, ::-1]).any()


def test_cal_view_pred_pose_linemod(cuda):
    from ffb6d_b200 import pose, vis
    B, obj = 3, 5
    pb, ep, item, meshes = _net_batch(cuda, B, 32, "linemod")
    lm_mesh = {obj: meshes[obj].astype(np.float64) * 1.1}
    got = vis.cal_view_pred_pose(_Net(ep), item, dataset="linemod", mesh_pts=lm_mesh, mesh_kps=pb["mesh"][1],
                                 K=VC.K_LM, obj_id=obj).cpu().numpy()
    pcld = item["cld_rgb_nrm"][:, :3].permute(0, 2, 1).contiguous()
    mask = ep["pred_rgbd_segs"].argmax(1)
    for b in range(B):
        poses = pose.cal_frame_poses_lm(pcld[b], mask[b], ep["pred_ctr_ofs"][b], ep["pred_kp_ofs"][b], True, 22,
                                        False, obj, mesh_kps=pb["mesh"][1])
        want = O.demo_draw(item["rgb"][b].cpu().numpy(), item["cls_ids"][b].cpu().numpy(), None, poses, lm_mesh,
                           VC.K_LM, "linemod", obj)
        assert np.array_equal(got[b], want), b
    with pytest.raises(ValueError):
        vis.cal_view_pred_pose(_Net(ep), item, dataset="linemod", mesh_pts=lm_mesh, mesh_kps=pb["mesh"][1],
                               K=VC.K_LM)


def test_cal_view_pred_pose_errors(cuda):
    from ffb6d_b200 import vis
    pb, ep, item, meshes = _net_batch(cuda, 1, 33, "ycb")
    kps = {c: k for c, k in pb["mesh"].items() if c != int(np.unique(pb["mask"][0])[1])}
    with pytest.raises(ValueError):
        vis.cal_view_pred_pose(_Net(ep), item, dataset="ycb", mesh_pts=meshes, mesh_kps=kps,
                               cls_radius=pb["cls_radius"], K=VC.K_YCB)


def test_view_labels_batched(cuda):
    from ffb6d_b200 import vis
    rs = np.random.RandomState(6)
    from ffb6d_b200.synthetic import make_frame
    clds = np.stack([make_frame(s, n_points=3000, intrinsics="linemod")["cld"].T for s in (1, 2)])
    labels = rs.randint(0, 3, (2, 3000))
    out = vis.view_labels(torch.zeros((2, 3, 480, 640), device=cuda), _t(clds, cuda), _t(labels, cuda), VC.K_LM,
                          n_objects=2).cpu().numpy()
    for b in range(2):
        assert np.array_equal(out[b], O.view_labels(480, 640, clds[b].T, labels[b], VC.K_LM, 2)), b
    with pytest.raises(ValueError):
        vis.view_labels(torch.zeros((2, 3, 480, 640), device=cuda), _t(clds, cuda), _t(labels + 1, cuda), VC.K_LM,
                        n_objects=2)


def test_graph_replay(cuda):
    from ffb6d_b200 import pose, vis
    B = 2
    pb, ep, item, meshes = _net_batch(cuda, B, 34, "ycb")
    table = pose.MeshTable(meshes, cuda, torch.float64)
    vt = pose.VoteTable(pb["mesh"], 22, pb["cls_radius"], cuda)
    pcld = item["cld_rgb_nrm"][:, :3].permute(0, 2, 1).contiguous()
    mask = ep["pred_rgbd_segs"].argmax(1)
    K = _t(VC.K_YCB, cuda, torch.float64)
    colors = _t(np.array([vis.get_label_color(c, n_obj=22, mode=2) for c in range(22)], np.uint8), cuda)
    base = item["rgb"].to(torch.uint8).permute(0, 2, 3, 1).contiguous()

    def step(ws=None):
        present, _, _, poses = pose.cal_batch_poses(pcld, mask, ep["pred_ctr_ofs"], ep["pred_kp_ofs"], True, 22,
                                                    True, mesh_kps=vt)
        img = base.clone()
        return vis.draw_poses(img, table, item["cls_ids"], present, poses, K, colors, ws=ws)

    eager = step().cpu().numpy()
    ws = F_ops().draw_p2ds_workspace(base)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(ws)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step(ws)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), eager)
    assert (eager != base.cpu().numpy()).any()
