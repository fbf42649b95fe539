"""GPU: the batched voting (``ops.vote_poses`` / ``pose.cal_batch_poses``) against the restatement in
oracle/pose_oracle.py and the reference's golden frame, bitwise against the per-object loop of
``mean_shift_fit`` / ``best_fit_transform`` and against its own B = 1 calls, through a CUDA graph, on bad input, at
its size limits, and inside ``TorchEval``."""
import os

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import GOLDEN
from ffb6d_b200 import ops, pose as P
from ffb6d_b200.synthetic import make_pose_batch, make_pose_frame
from oracle import pose_oracle as PO

pytestmark = pytest.mark.gpu
N_CLS = 5


def _same(a, b):
    """Bitwise equality of two tensors, NaN rows included."""
    a, b = a.contiguous().cpu(), b.contiguous().cpu()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _stack(frames):
    return [torch.from_numpy(np.stack([f[k] for f in frames])).cuda() for k in ("pcld", "mask", "ctr_of", "kp_of")]


def _mesh(mesh, n_kps, use_ctr):
    return {c: m if use_ctr else m[:n_kps] for c, m in mesh.items()}


def _lists(out, table, b, n_kps):
    present, count, kps, poses = (t[b].cpu().numpy() for t in out)
    return P._frame_lists(present, count, kps, poses, table.has_mesh.cpu().numpy(), n_kps)


def _edge_frames():
    """Frames at the rules' edges, all of make_pose_frame's 2 150 points: all background; one class with every
    centre vote NaN (no centre label is set); frames with other object sets (class 2 or classes 1 and 4 dropped)."""
    out = []
    fr = make_pose_frame(11)
    fr["mask"] = np.zeros_like(fr["mask"])
    out.append(fr)
    fr = make_pose_frame(12)
    fr["ctr_of"] = fr["ctr_of"].copy()
    fr["ctr_of"][0, fr["mask"] == 3] = np.nan
    out.append(fr)
    fr = make_pose_frame(13)
    fr["mask"] = np.where(fr["mask"] == 2, 0, fr["mask"])
    out.append(fr)
    fr = make_pose_frame(14)
    fr["mask"] = np.where((fr["mask"] == 1) | (fr["mask"] == 4), 0, fr["mask"])
    out.append(fr)
    return out


@pytest.fixture(scope="module")
def frames():
    return [make_pose_frame(s) for s in (1, 2, 3)] + _edge_frames()


def _oracle_want(fr, mesh, use_ctr, flt, drop=()):
    """The oracle's frame without the classes ``drop`` (whose fit numpy's SVD refuses: NaN keypoints)."""
    args = [fr[k] for k in ("pcld", "mask", "ctr_of", "kp_of")]
    fit = PO.best_fit_transform
    PO.best_fit_transform = lambda A, B: fit(A, B) if np.isfinite(B).all() else np.full((3, 4), np.nan)
    try:
        ids, poses, kps = PO.cal_frame_poses(*args, use_ctr, flt, mesh, fr["cls_radius"])
    finally:
        PO.best_fit_transform = fit
    keep = [k for k, c in enumerate(ids) if c not in drop]
    return dict(ids=np.asarray(ids, np.int64)[keep], poses=np.stack(poses)[keep] if keep else np.zeros((0, 3, 4)),
                **{"kps_%d" % ids[k]: kps[k] for k in keep})


@pytest.mark.parametrize("variant", PO.FRAME_VARIANTS, ids=[v[0] for v in PO.FRAME_VARIANTS])
def test_batch_vs_oracle(cuda, frames, variant):
    """Every frame of one batch against oracle/pose_oracle.cal_frame_poses, with check_frame_poses' tolerances
    (every frame fitted to the first frame's mesh keypoints)."""
    name, use_ctr, flt = variant
    n_kps, mesh = frames[0]["kp_of"].shape[0], frames[0]["mesh"]
    table = P.VoteTable(_mesh(mesh, n_kps, use_ctr), N_CLS, frames[0]["cls_radius"])
    out = P.cal_batch_poses(*_stack(frames), use_ctr, N_CLS, flt, mesh_kps=table)
    for b, fr in enumerate(frames):
        ids, poses, kps = _lists(out, table, b, n_kps)
        nan_cls = (3,) if b == 4 else ()
        PO.check_frame_poses([c for c in ids if c not in nan_cls], [p for c, p in zip(ids, poses) if c not in nan_cls],
                             [k for c, k in zip(ids, kps) if c not in nan_cls],
                             _oracle_want(fr, mesh, use_ctr, flt, nan_cls), mesh, n_kps, use_ctr)
        if b == 3:                                      # all background
            assert len(ids) == 0 and not out[0][b].any() and not out[3][b].any()


@pytest.mark.parametrize("use_ctr", [True, False])
def test_empty_centre_labels_keep_first_point(cuda, frames, use_ctr):
    """All centre votes of class 3 NaN: no centre label is set, so the class's keypoint sets are fitted from its
    first point alone (the reference's ``ctr_labels[0] = 1``): each keypoint is that point's vote, exactly."""
    fr = frames[4]
    n_kps = fr["kp_of"].shape[0]
    table = P.VoteTable(_mesh(fr["mesh"], n_kps, use_ctr), N_CLS, fr["cls_radius"])
    out = P.cal_batch_poses(*_stack([fr]), use_ctr, N_CLS, True, mesh_kps=table)
    first = int(np.flatnonzero(fr["mask"] == 3)[0])
    want = fr["pcld"][first][None] - fr["kp_of"][:, first]
    assert out[1][0, 3].item() == (fr["mask"] == 3).sum()
    assert np.array_equal(out[2][0, 3, :n_kps].cpu().numpy(), want)
    assert torch.isnan(out[2][0, 3, n_kps:]).all() if use_ctr else torch.isfinite(out[3][0, 3]).all()


def test_lm_batch_vs_oracle(cuda, frames):
    """LineMOD: class 1 of every frame, n_cls = 2 and no refinement, against oracle cal_frame_poses_lm."""
    fr0 = frames[0]
    table = P.VoteTable({1: fr0["mesh"][1]}, 2)
    pc, mask, ctr, kp = _stack(frames)
    for flt in (True, False):
        present, _, _, poses = P.cal_batch_poses(pc, mask == 1, ctr, kp, True, 2, flt, mesh_kps=table)
        for b, fr in enumerate(frames):
            w = PO.cal_frame_poses_lm(*[fr[k] for k in ("pcld", "mask", "ctr_of", "kp_of")], True, flt,
                                      fr0["mesh"][1])[0]
            if not present[b, 1]:
                assert np.array_equal(w, np.identity(4)[:3]) and not poses[b, 1].any()
                continue
            m = np.asarray(fr0["mesh"][1], np.float64)
            T = poses[b, 1].cpu().numpy()
            assert np.linalg.norm(m @ T[:, :3].T + T[:, 3] - (m @ w[:, :3].T + w[:, 3]), axis=1).mean() < 2e-4
            got = P.cal_frame_poses_lm(*[torch.from_numpy(fr[k]).cuda() for k in ("pcld", "mask", "ctr_of", "kp_of")],
                                       True, 2, flt, 1, mesh_kps=fr0["mesh"][1])
            assert np.array_equal(got[0], T)


@pytest.mark.parametrize("variant", PO.FRAME_VARIANTS, ids=[v[0] for v in PO.FRAME_VARIANTS])
def test_batch_vs_reference_golden(cuda, variant):
    """The reference's own frame (tests/golden/pose_frame_cases.npz), voted as frame 1 of a batch of three."""
    name, use_ctr, flt = variant
    gold = PO.load_frame_golden(os.path.join(GOLDEN, "pose_frame_cases.npz"))
    fr = make_pose_frame(int(gold["seed"]))
    assert PO.frame_input_sha256(fr) == str(gold["input_sha256"])
    n_kps = fr["kp_of"].shape[0]
    table = P.VoteTable(_mesh(fr["mesh"], n_kps, use_ctr), N_CLS, fr["cls_radius"])
    out = P.cal_batch_poses(*_stack([make_pose_frame(5), fr, make_pose_frame(6)]), use_ctr, N_CLS, flt,
                            mesh_kps=table)
    ids, poses, kps = _lists(out, table, 1, n_kps)
    PO.check_frame_poses(ids, poses, kps, gold[name], fr["mesh"], n_kps, use_ctr)


def test_batch_equals_single_frames(cuda, frames):
    """Frame b of a batch is bitwise a B = 1 call on frame b, in every variant."""
    n_kps = frames[0]["kp_of"].shape[0]
    batch = _stack(frames)
    for name, use_ctr, flt in PO.FRAME_VARIANTS:
        table = P.VoteTable(_mesh(frames[0]["mesh"], n_kps, use_ctr), N_CLS, frames[0]["cls_radius"])
        out = P.cal_batch_poses(*batch, use_ctr, N_CLS, flt, mesh_kps=table)
        again = P.cal_batch_poses(*batch, use_ctr, N_CLS, flt, mesh_kps=table)
        for b in range(len(frames)):
            one = P.cal_batch_poses(*(t[b:b + 1] for t in batch), use_ctr, N_CLS, flt, mesh_kps=table)
            for x, y, z in zip(out, one, again):
                assert _same(x[b], y[0]) and _same(x[b], z[b]), (name, b)


# ----------------------------------------------------------------------------- the per-object loop, restated
def _loop_frame(pcld, mask, ctr_of, kp_of, use_ctr, flt, mesh, thr):
    """One frame the way the parent voted it, one object at a time through ``mean_shift_fit`` and
    ``best_fit_transform``, with the refinement in the reference's difference form (numpy, float32).  Returns the
    batched op's four rows and the smallest |distance - threshold| of a refinement decision."""
    n_kps, N = kp_of.shape[:2]
    n_cls, R = thr.shape[0], n_kps + int(use_ctr)
    pred_ctr, pred_kp = pcld - ctr_of[0], pcld[None] - kp_of
    ids = torch.unique(mask[mask > 0]).tolist()
    present = torch.zeros(n_cls, dtype=torch.bool)
    present[ids] = True
    margin = np.inf
    if flt and ids:
        msks = torch.stack([mask == c for c in ids])
        ctrs, _, _ = F.mean_shift_fit(pred_ctr[None].expand(len(ids), N, 3).contiguous(), msks, 0.04, 300)
        pc, cc = pred_ctr.cpu().numpy(), ctrs.cpu().numpy()
        d = np.sqrt(((pc[:, None, :] - cc[None]) ** 2).sum(2, dtype=np.float32))
        j = d.argmin(1)
        near = np.asarray(ids)[j]
        dmin = d[np.arange(N), j]
        obj = mask.cpu().numpy() > 0
        margin = float(np.abs(dmin - thr[near])[obj].min())
        mask = torch.where(torch.from_numpy(obj & (dmin < thr[near])).cuda(), torch.from_numpy(near).cuda(), mask)
    count = torch.zeros(n_cls, dtype=torch.int32)
    kps = torch.zeros(n_cls, R, 3)
    poses = torch.zeros(n_cls, 3, 4, dtype=torch.float64)
    for c in ids:
        msk = mask == c
        count[c] = int(msk.sum())
        if count[c] == 0:
            poses[c] = torch.eye(3, 4, dtype=torch.float64)
            continue
        ctr, lab, _ = F.mean_shift_fit(pred_ctr[None], msk, 0.04, 300)
        lab = lab[0]
        if flt and not lab.any():
            lab[int(torch.nonzero(msk)[0])] = True
        kp, _, _ = F.mean_shift_fit(pred_kp, lab if flt else msk, 0.04, 300)
        kpc = torch.cat((kp, ctr)) if use_ctr else kp
        kps[c] = kpc.cpu()
        poses[c] = F.best_fit_transform(torch.as_tensor(mesh[c][:R], dtype=torch.float32).cuda(), kpc).cpu()
    return (present, count, kps, poses), margin


def _check_vs_loop(batch, mesh, cls_radius, n_cls):
    n_kps = batch[3].shape[1]
    for name, use_ctr, flt in PO.FRAME_VARIANTS:
        table = P.VoteTable(_mesh(mesh, n_kps, use_ctr), n_cls, cls_radius)
        thr = table.refine_thr.cpu().numpy()
        out = P.cal_batch_poses(*batch, use_ctr, n_cls, flt, mesh_kps=table)
        for b in range(batch[0].shape[0]):
            want, margin = _loop_frame(*(t[b] for t in batch), use_ctr, flt, _mesh(mesh, n_kps, use_ctr), thr)
            assert margin > 1e-5, (name, b, margin)         # no refinement decision within 1e-5 m of a threshold
            for k, (x, w) in enumerate(zip(out, want)):
                assert _same(x[b], w.to(x.dtype)), (name, b, k)


def test_equals_object_loop_2000_points(cuda, frames):
    """Bitwise the parent's per-object loop on make_pose_frame frames (2 150 points, 5 classes)."""
    fr = frames[0]
    _check_vs_loop(_stack([frames[i] for i in (0, 1, 2, 5, 6)]), fr["mesh"], fr["cls_radius"], N_CLS)


def test_equals_object_loop_full_size(cuda):
    """Bitwise the parent's per-object loop at N = 12288 with 22 classes, 5 objects per frame."""
    bt = make_pose_batch(3, 2)
    batch = [torch.from_numpy(bt[k]).cuda() for k in ("pcld", "mask", "ctr_of", "kp_of")]
    _check_vs_loop(batch, bt["mesh"], bt["cls_radius"], 22)


def test_cuda_graph_replay(cuda, frames):
    """One call captured, replayed on a second batch of the same shapes: bitwise an eager call on it."""
    table = P.VoteTable(frames[0]["mesh"], N_CLS, frames[0]["cls_radius"])
    first, second = _stack(frames[:3]), _stack([frames[5], frames[4], frames[6]])
    static = [t.clone() for t in first]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        P.cal_batch_poses(*static, True, N_CLS, True, mesh_kps=table)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = P.cal_batch_poses(*static, True, N_CLS, True, mesh_kps=table)
    for src in (first, second):
        for t, v in zip(static, src):
            t.copy_(v)
        g.replay()
        torch.cuda.synchronize()
        want = P.cal_batch_poses(*src, True, N_CLS, True, mesh_kps=table)
        assert all(_same(x, y) for x, y in zip(out, want))


def test_bad_mask_id_and_missing_mesh(cuda, frames):
    """A mask id outside [0, n_cls) makes its frame NaN (present and count 0) and a present class without mesh
    keypoints its row NaN; every other row is bitwise unchanged, and the frame wrappers raise ValueError."""
    fr = frames[0]
    table = P.VoteTable(fr["mesh"], N_CLS, fr["cls_radius"])
    batch = _stack(frames[:3])
    clean = P.cal_batch_poses(*batch, True, N_CLS, True, mesh_kps=table)
    for bad in (N_CLS, -1):
        m = batch[1].clone()
        m[1, 7] = bad
        out = P.cal_batch_poses(batch[0], m, batch[2], batch[3], True, N_CLS, True, mesh_kps=table)
        assert torch.isnan(out[2][1]).all() and torch.isnan(out[3][1]).all()
        assert not out[0][1].any() and not out[1][1].any()
        for x, y in zip(out, clean):
            assert _same(x[0], y[0]) and _same(x[2], y[2])
        with pytest.raises(ValueError, match="outside"):
            P.cal_frame_poses(batch[0][1], m[1], batch[2][1], batch[3][1], True, N_CLS, True, mesh_kps=fr["mesh"],
                              cls_radius=fr["cls_radius"])
    no2 = {c: v for c, v in fr["mesh"].items() if c != 2}
    out = P.cal_batch_poses(*batch, True, N_CLS, True, mesh_kps=P.VoteTable(no2, N_CLS, fr["cls_radius"]))
    assert torch.isnan(out[2][:, 2]).all() and torch.isnan(out[3][:, 2]).all()
    rows = [c for c in range(N_CLS) if c != 2]
    for x, y in zip(out, clean):
        assert _same(x[:, rows], y[:, rows])
    with pytest.raises(ValueError, match="no mesh"):
        P.cal_frame_poses(*(t[0] for t in batch), True, N_CLS, True, mesh_kps=no2, cls_radius=fr["cls_radius"])


def test_limits(cuda):
    """B = 0; the largest n_kps and n_cls, N at FFB6D_VOTE_MAX_POINTS and a set table of FFB6D_VOTE_MAX_SETS."""
    dev = cuda
    z = ops.vote_poses(torch.zeros(0, 5, 3, device=dev), torch.zeros(0, 5, dtype=torch.int64, device=dev),
                       torch.zeros(0, 1, 5, 3, device=dev), torch.zeros(0, 8, 5, 3, device=dev),
                       torch.zeros(3, 9, 3, device=dev), torch.ones(3, dtype=torch.uint8, device=dev))
    assert [tuple(t.shape) for t in z] == [(0, 3), (0, 3), (0, 3, 9, 3), (0, 3, 3, 4)]

    def run(B, N, C, K, n_obj_pts):
        g = torch.Generator(device=dev).manual_seed(B + N + C + K)
        pc = torch.rand(B, N, 3, device=dev, generator=g)
        mask = torch.zeros(B, N, dtype=torch.int64, device=dev)
        mask[0, :n_obj_pts] = C - 1
        ctr = pc[:, None] - 0.5 + torch.rand(B, 1, N, 3, device=dev, generator=g) * 1e-3
        kp = pc[:, None] - torch.rand(B, K, 1, 3, device=dev, generator=g) + torch.rand(B, K, N, 3, device=dev,
                                                                                    generator=g) * 1e-3
        mk = torch.rand(C, K + 1, 3, device=dev, generator=g)
        out = ops.vote_poses(pc, mask, ctr, kp, mk, torch.ones(C, dtype=torch.uint8, device=dev))
        assert out[0][0, C - 1] and out[1][0, C - 1].item() == n_obj_pts and torch.isfinite(out[3][0, C - 1]).all()
        assert out[0].sum().item() == 1
        return out

    run(2, 300, 3, F._lib.VOTE_MAX_KPS, 200)
    run(2, 300, F._lib.VOTE_MAX_CLASSES, 8, 200)
    run(1, F._lib.VOTE_MAX_POINTS, 2, 1, 300)
    B = F._lib.VOTE_MAX_SETS // F._lib.VOTE_MAX_CLASSES // F._lib.VOTE_MAX_KPS
    run(B, 1, F._lib.VOTE_MAX_CLASSES, F._lib.VOTE_MAX_KPS, 1)
    with pytest.raises(F._lib.FFB6DError):
        run(B + 1, 1, F._lib.VOTE_MAX_CLASSES, F._lib.VOTE_MAX_KPS, 1)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------- TorchEval
def _eval_batch(n_frames):
    frs = [make_pose_frame(40 + f) for f in range(n_frames)]
    n_obj, n_kps = 6, frs[0]["kp_of"].shape[0]
    cls_ids = np.zeros((n_frames, n_obj, 1), np.int64)
    RTs = np.zeros((n_frames, n_obj, 3, 4), np.float32)
    gt_kps = np.zeros((n_frames, n_obj, n_kps, 3), np.float32)
    for b, fr in enumerate(frs):
        for i, c in enumerate((1, 2, 3, 4)[: 4 - b % 2]):
            cls_ids[b, i, 0], RTs[b, i] = c, fr["poses"][c]
            gt_kps[b, i] = (fr["mesh"][c] @ fr["poses"][c][:, :3].T + fr["poses"][c][:, 3])[:n_kps]
    t = {k: torch.from_numpy(np.stack([f[k] for f in frs])).cuda() for k in ("pcld", "mask", "ctr_of", "kp_of")}
    return frs, t, torch.from_numpy(cls_ids).cuda(), torch.from_numpy(RTs).cuda(), torch.from_numpy(gt_kps).cuda()


def test_torch_eval_batch_equals_single_frames(cuda):
    """A B = 8 eval_pose_parallel gives exactly the lists of eight B = 1 calls, for YCB and LineMOD."""
    frs, t, cls_ids, RTs, gt_kps = _eval_batch(8)
    rs = np.random.RandomState(3)
    meshes = {c: rs.uniform(-0.08, 0.08, (500, 3)).astype(np.float32) for c in range(1, N_CLS)}
    for ds in ("ycb", "linemod"):
        te8 = P.TorchEval(meshes, frs[0]["mesh"], frs[0]["cls_radius"], (3,), n_cls=N_CLS)
        te1 = P.TorchEval(meshes, frs[0]["mesh"], frs[0]["cls_radius"], (3,), n_cls=N_CLS)
        kw = dict(obj_id=1, ds=ds)
        te8.eval_pose_parallel(t["pcld"], None, t["mask"], t["ctr_of"], None, None, 0, cls_ids, RTs, t["kp_of"],
                               gt_kps, None, **kw)
        for b in range(8):
            s = slice(b, b + 1)
            te1.eval_pose_parallel(t["pcld"][s], None, t["mask"][s], t["ctr_of"][s], None, None, 0, cls_ids[s],
                                   RTs[s], t["kp_of"][s], gt_kps[s], None, **kw)
        assert te8.cls_add_dis == te1.cls_add_dis and te8.cls_adds_dis == te1.cls_adds_dis
        assert te8.pred_kp_errs == te1.pred_kp_errs
        assert len(te8.pred_id2pose_lst) == len(te1.pred_id2pose_lst)
        for x, y in zip(te8.pred_id2pose_lst, te1.pred_id2pose_lst):
            assert x.keys() == y.keys() and all(np.array_equal(x[k], y[k]) for k in x)
        assert sum(len(v) for v in te8.cls_add_dis[1:]) == (28 if ds == "ycb" else 8)
