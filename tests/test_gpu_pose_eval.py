"""GPU: ADD / ADD-S of a batch in one launch (ops.pose_add_adds) against float64 (oracle/pose_eval_oracle.py) and the
reference's own values (tests/golden/pose_eval_cases.npz, inputs rebuilt by tests/pose_eval_cases.py); NaN and out-of-range rows, graph replay and the size
limits; the reference-named mirrors (eval_metric(_lm), TorchEval) against the reference's runs.

Bound: |got - f64| <= 2e-6 m * max(1, s), s the largest transformed coordinate in metres (DESIGN.md §4.24).  The
largest measured |got - f64| / max(1, s), over the 137 float64 checks of the tile-size, golden and ragged-batch tests,
was 1.1e-7 on an H100 80GB HBM3 (700 W power limit)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from ffb6d_b200 import _lib, ops, pose
from oracle import pose_eval_oracle as PO
import pose_eval_cases as PC

pytestmark = pytest.mark.gpu

TOL = 2e-6
TILE_SIZES = sorted({1, 7, 8, 9} | {t + d for t in (256, 512, 1024) for d in (-1, 0, 1)} | {2000, 2621, 40000})


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "pose_eval_cases.npz"))
    return {k: z[k] for k in z.files}


def golden_cases(golden):
    i, out = 0, []
    while "adds:%d:n" % i in golden:
        k = "adds:%d:" % i
        n = int(golden[k + "n"])
        mesh = PC.adds_mesh(n) if n else golden["adds:ring"]
        out.append((str(golden[k + "kind"]), mesh, golden[k + "pred"], golden[k + "gt"],
                    float(golden[k + "add"]), float(golden[k + "adds"])))
        i += 1
    return out


def scale(mesh, pred, gt):
    x = mesh.astype(np.float64)
    s = max(np.abs(x @ np.asarray(T, np.float64)[:, :3].T + np.asarray(T, np.float64)[:, 3]).max() for T in (pred, gt))
    return max(1.0, float(s))


def run(mesh_list, cls, pred, gt, max_points=None):
    """ops.pose_add_adds over a table of ``mesh_list``; returns numpy (add, adds)."""
    off = np.concatenate(([0], np.cumsum([len(m) for m in mesh_list]))).astype(np.int32)
    pts = torch.as_tensor(np.concatenate(mesh_list).astype(np.float32)).cuda()
    mp = max_points or max(len(m) for m in mesh_list)
    add, adds = ops.pose_add_adds(pts, torch.as_tensor(off).cuda(), torch.as_tensor(np.asarray(cls, np.int32)).cuda(),
                                  torch.as_tensor(np.asarray(pred, np.float32)).cuda(),
                                  torch.as_tensor(np.asarray(gt, np.float32)).cuda(), mp)
    return add.cpu().numpy(), adds.cpu().numpy()


def check_f64(mesh, pred, gt, add, adds):
    a64, s64 = PO.add_adds_f64(mesh, pred, gt)
    s = scale(mesh, pred, gt)
    err = max(abs(add - a64), abs(adds - s64)) / s
    assert err <= TOL, (len(mesh), add, a64, adds, s64, s)


@pytest.mark.parametrize("n", TILE_SIZES)
def test_against_f64(golden, n):
    """Every pose kind of the golden file, in one batch, on a mesh of n points."""
    kinds = [c for c in golden_cases(golden) if len(c[1]) == 2621]
    mesh = np.random.RandomState(n).uniform(-0.1, 0.1, (n, 3)).astype(np.float32)
    pred = np.stack([c[2] for c in kinds])
    gt = np.stack([c[3] for c in kinds])
    add, adds = run([mesh], [0] * len(kinds), pred, gt)
    for m in range(len(kinds)):
        check_f64(mesh, pred[m], gt[m], add[m], adds[m])


def test_against_reference_golden(golden):
    cases = golden_cases(golden)
    for kind, mesh, pred, gt, ref_add, ref_adds in cases:
        add, adds = run([mesh], [0], pred[None], gt[None])
        s = scale(mesh, pred, gt)
        for got, ref in ((add[0], ref_add), (adds[0], ref_adds)):
            assert abs(got - ref) <= TOL * s + 1e-5 * abs(ref), (kind, len(mesh), got, ref)
        check_f64(mesh, pred, gt, add[0], adds[0])


def test_exact_cases(golden):
    for kind, mesh, pred, gt, _, _ in golden_cases(golden):
        if kind == "identical":
            add, adds = run([mesh], [0], pred[None], gt[None])
            assert add[0] == 0.0 and adds[0] == 0.0, (len(mesh), add, adds)
        if kind == "symmetric":
            add, adds = run([mesh], [0], pred[None], gt[None])
            a64, s64 = PO.add_adds_f64(mesh, pred, gt)
            assert add[0] > 0.03 and abs(add[0] - a64) <= TOL
            assert adds[0] <= s64 + TOL and abs(adds[0] - s64) <= TOL


def ragged(seed=3):
    rs = np.random.RandomState(seed)
    meshes = [rs.uniform(-0.1, 0.1, (int(rs.randint(1, 3000)), 3)).astype(np.float32) for _ in range(21)]
    cls, pred, gt = [], [], []
    for _ in range(8):
        for _ in range(int(rs.randint(1, 7))):
            cls.append(int(rs.randint(0, 21)))
            R = np.linalg.qr(rs.normal(size=(3, 3)))[0]
            t = rs.uniform(-0.3, 0.3, 3) + [0, 0, 1]
            G = np.concatenate((R, t[:, None]), 1)
            gt.append(G)
            pred.append(G + rs.normal(0, 0.01, (3, 4)))
    return meshes, cls, np.asarray(pred, np.float32), np.asarray(gt, np.float32)


def test_ragged_batch_equals_single_calls():
    meshes, cls, pred, gt = ragged()
    add, adds = run(meshes, cls, pred, gt)
    add2, adds2 = run(meshes, cls, pred, gt)
    assert add.tobytes() == add2.tobytes() and adds.tobytes() == adds2.tobytes()
    for m, c in enumerate(cls):
        a1, s1 = run([meshes[c]], [0], pred[m:m + 1], gt[m:m + 1])
        assert a1[0].tobytes() == add[m].tobytes() and s1[0].tobytes() == adds[m].tobytes(), m
        if m % 7 == 0:
            check_f64(meshes[c], pred[m], gt[m], add[m], adds[m])


def test_bad_values_give_nan_rows():
    meshes, cls, pred, gt = ragged(5)
    clean_add, clean_adds = run(meshes, cls, pred, gt)
    p, g = pred.copy(), gt.copy()
    p[0, 1, 2] = np.nan
    g[2, 0, 3] = np.inf
    p[4, 2, 0] = -np.inf
    add, adds = run(meshes, cls, p, g)
    bad = {0, 2, 4}
    for m in range(len(cls)):
        if m in bad:
            assert np.isnan(add[m]) and np.isnan(adds[m]), m
        else:
            assert add[m].tobytes() == clean_add[m].tobytes() and adds[m].tobytes() == clean_adds[m].tobytes()
    # a NaN point poisons the objects scored on its mesh only
    mm = [m.copy() for m in meshes]
    c0 = cls[1]
    mm[c0][len(mm[c0]) // 2, 1] = np.nan
    add, adds = run(mm, cls, pred, gt)
    for m, c in enumerate(cls):
        assert np.isnan(add[m]) == (c == c0) and np.isnan(adds[m]) == (c == c0)
        if c != c0:
            assert add[m] == clean_add[m] and adds[m] == clean_adds[m]


def test_out_of_range_rows_give_nan():
    rs = np.random.RandomState(9)
    meshes = [rs.uniform(-0.1, 0.1, (n, 3)).astype(np.float32) for n in (100, 600, 40, 700)]
    off = np.concatenate(([0], np.cumsum([len(m) for m in meshes]))).astype(np.int32)
    pts = torch.as_tensor(np.concatenate(meshes)).cuda()
    G = np.concatenate((np.eye(3), [[0], [0], [1]]), 1).astype(np.float32)
    P = G + np.float32(0.01)
    M = 8
    pr = torch.as_tensor(np.stack([P] * M)).cuda()
    gt = torch.as_tensor(np.stack([G] * M)).cuda()

    def call(cls, o, mp=700):
        a, s = ops.pose_add_adds(pts, torch.as_tensor(o).cuda(), torch.as_tensor(np.asarray(cls, np.int32)).cuda(),
                                 pr, gt, mp)
        return a.cpu().numpy(), s.cpu().numpy()

    cls = [0, 1, 2, 3, 0, 1, 2, 3]
    ref_add, ref_adds = call(cls, off)
    for m, c in enumerate(cls):
        check_f64(meshes[c], P, G, ref_add[m], ref_adds[m])
    # class ids out of [0, n_meshes)
    add, adds = call([0, -1, 2, 4, 0, 1, 2 ** 31 - 1, 3], off)
    assert np.isnan(add[[1, 3, 6]]).all() and np.isnan(adds[[1, 3, 6]]).all()
    keep = [0, 2, 4, 5, 7]
    assert (add[keep] == ref_add[keep]).all() and (adds[keep] == ref_adds[keep]).all()
    # a negative offset (mesh 0), a decreasing pair (mesh 2), and a mesh longer than max_points (mesh 3 at 650)
    o = off.copy()
    o[0] = -5
    o[3] = o[2] - 1
    add, adds = call(cls, o, mp=650)
    nan_rows = [m for m, c in enumerate(cls) if c in (0, 1, 2, 3) and c != 1]
    assert np.isnan(add[nan_rows]).all() and np.isnan(adds[nan_rows]).all()
    ok = [m for m, c in enumerate(cls) if c == 1]
    assert (add[ok] == ref_add[ok]).all() and (adds[ok] == ref_adds[ok]).all()


def test_graph_replay_is_bitwise():
    meshes, cls, pred, gt = ragged(11)
    off = np.concatenate(([0], np.cumsum([len(m) for m in meshes]))).astype(np.int32)
    pts = torch.as_tensor(np.concatenate(meshes)).cuda()
    o, c = torch.as_tensor(off).cuda(), torch.as_tensor(np.asarray(cls, np.int32)).cuda()
    pr, g = torch.as_tensor(pred).cuda(), torch.as_tensor(gt).cuda()
    mp = max(len(m) for m in meshes)
    eager = ops.pose_add_adds(pts, o, c, pr, g, mp)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.pose_add_adds(pts, o, c, pr, g, mp)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.pose_add_adds(pts, o, c, pr, g, mp)
    for _ in range(3):
        out[0].zero_()
        out[1].zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
    pr.copy_(torch.as_tensor(gt))                   # new inputs in the captured buffers: identical poses
    graph.replay()
    torch.cuda.synchronize()
    assert (out[0] == 0).all() and (out[1] == 0).all()


def test_limits():
    M = _lib.POSE_EVAL_MAX_OBJECTS
    rs = np.random.RandomState(13)
    meshes = [rs.uniform(-0.1, 0.1, (n, 3)).astype(np.float32) for n in (1, 2, 3)]
    cls = rs.randint(0, 3, M)
    R = np.linalg.qr(rs.normal(size=(3, 3)))[0]
    gt = np.concatenate((R, [[0.1], [0.0], [1.0]]), 1).astype(np.float32)
    pred = (gt[None] + rs.normal(0, 0.01, (M, 3, 4))).astype(np.float32)
    add, adds = run(meshes, cls, pred, np.repeat(gt[None], M, 0))
    for m in list(range(0, M, 4099)) + [M - 1]:
        check_f64(meshes[cls[m]], pred[m], gt, add[m], adds[m])
    n = _lib.POSE_EVAL_MAX_POINTS
    free, _ = torch.cuda.mem_get_info()
    if free < 1 << 30:
        pytest.skip("the largest mesh's check needs 1 GB of free device memory, %d bytes are free" % free)
    big = rs.uniform(-0.1, 0.1, (n, 3)).astype(np.float32)
    P2 = (gt + rs.normal(0, 0.002, (3, 4))).astype(np.float32)
    add, adds = run([big], [0], P2[None], gt[None], max_points=n)
    check_f64(big, P2, gt, add[0], adds[0])
    x = torch.zeros(4, 3, device="cuda")
    o = torch.tensor([0, 4], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        ops.pose_add_adds(x, o, torch.zeros(M + 1, dtype=torch.int32, device="cuda"),
                          torch.zeros(M + 1, 3, 4, device="cuda"), torch.zeros(M + 1, 3, 4, device="cuda"), 4)
    with pytest.raises(ValueError):
        ops.pose_add_adds(x, o, torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, 3, 4, device="cuda"),
                          torch.zeros(1, 3, 4, device="cuda"), n + 1)


def test_single_object_mirrors(golden):
    for kind, mesh, pred, gt, ref_add, ref_adds in golden_cases(golden)[::5]:
        p3 = torch.as_tensor(mesh).cuda()
        a = pose.cal_add_cuda(torch.as_tensor(pred).cuda(), torch.as_tensor(gt).cuda(), p3)
        s = pose.cal_adds_cuda(torch.as_tensor(pred).cuda(), torch.as_tensor(gt).cuda(), p3)
        assert a.dim() == 0 and a.is_cuda and s.dim() == 0
        add, adds = run([mesh], [0], pred[None], gt[None])
        assert a.item() == add[0] and s.item() == adds[0]


def unflatten(golden, key, n_cls=22):
    out = [[] for _ in range(n_cls)]
    for c, v in zip(golden[key + ":cls"], golden[key + ":val"]):
        out[int(c)].append(float(v))
    return out


def close_lists(got, want, tol):
    assert [len(x) for x in got] == [len(x) for x in want]
    for g, w in zip(got, want):
        assert np.allclose(g, w, rtol=0, atol=tol), (g, w)


def test_eval_metric_mirrors(golden):
    table = pose.MeshTable(PC.ycb_meshes())
    ids = torch.as_tensor(golden["metric:ids"]).cuda()
    res = pose.eval_metric(ids, list(golden["metric:pred_pose_lst"]), golden["metric:pred_cls_ids"],
                           torch.as_tensor(golden["metric:RTs"]).cuda(), None, None,
                           torch.as_tensor(golden["metric:gt_kps"]).cuda(), None, list(golden["metric:pred_kpc_lst"]),
                           mesh_table=table)
    tol = TOL * 1.5 + 1e-5 * 1.1
    close_lists(res[0], unflatten(golden, "metric:add"), tol)
    close_lists(res[1], unflatten(golden, "metric:adds"), tol)
    close_lists(res[2], unflatten(golden, "metric:kp_err"), 1e-12)
    lm = pose.MeshTable({PC.LM_OBJ: PC.lm_mesh()})
    res = pose.eval_metric_lm(None, [golden["metric_lm:pred"]], torch.as_tensor(golden["metric_lm:RTs"]).cuda(), None,
                              None, PC.LM_OBJ, mesh_table=lm)
    close_lists(res[0], unflatten(golden, "metric_lm:add"), tol)
    close_lists(res[1], unflatten(golden, "metric_lm:adds"), tol)


def on_device(golden, key, batch):
    """The rebuilt batch on the GPU, after checking it is the one the reference was run on."""
    np.testing.assert_allclose(PC.frame_fingerprint(batch), golden[key], rtol=1e-9, atol=1e-9)
    return {k: torch.as_tensor(np.ascontiguousarray(v)).cuda() for k, v in batch.items()}


def test_torch_eval_end_to_end_ycb(golden):
    frs, kps, radius = PC.frames()
    te = pose.TorchEval(PC.ycb_meshes(), kps, radius, PC.YCB_SYM)
    b = on_device(golden, "te:fingerprint", PC.ycb_batch(frs))
    te.eval_pose_parallel(b["pclds"], None, b["masks"], b["pred_ctr_ofs"], None, None, 0, b["cls_ids"], b["RTs"],
                          b["pred_kp_ofs"], b["gt_kps"], b["gt_ctrs"])
    r = te.cal_auc()
    for name in ("add_dis_lst", "adds_dis_lst"):
        want = unflatten(golden, "te:" + name)
        for g, w in zip(r[name], want):
            assert len(g) == len(w)
        close_lists(r[name], want, 1e-4)
    close_lists(r["pred_kp_errs"], unflatten(golden, "te:pred_kp_errs"), 2e-4)
    for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        assert np.allclose(r[name], golden["te:" + name], rtol=0, atol=0.1), name
    assert len(te.pred_id2pose_lst) == 3


def test_torch_eval_end_to_end_linemod(golden):
    batch, kps = PC.lm_batch()
    te = pose.TorchEval({PC.LM_OBJ: PC.lm_mesh()}, {PC.LM_OBJ: kps}, sym_cls_ids=PC.LM_SYM)
    b = on_device(golden, "telm:fingerprint", batch)
    te.eval_pose_parallel(b["pclds"], None, b["masks"], b["pred_ctr_ofs"], None, None, 0, b["cls_ids"], b["RTs"],
                          b["pred_kp_ofs"], b["gt_kps"], b["gt_ctrs"], obj_id=PC.LM_OBJ, ds="linemod")
    r = te.cal_lm_add(PC.LM_OBJ, PC.LM_DIAMETER)
    close_lists(r["add_dis_lst"], unflatten(golden, "telm:add_dis_lst"), 1e-4)
    close_lists(r["adds_dis_lst"], unflatten(golden, "telm:adds_dis_lst"), 1e-4)
    for name in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        assert np.allclose(r[name], golden["telm:" + name], rtol=0, atol=0.1), name
    assert r["add"] == golden["telm:add"] and r["adds"] == golden["telm:adds"]
