"""GPU: the test run's device record and summary (``ops.eval_record`` / ``ops.eval_auc``, DESIGN.md §4.29) and
:class:`ffb6d_b200.GraphedTestStep`.

The record's rows against the numpy restatement (oracle/eval_record_oracle.py) and its summary against
``TorchEval.cal_auc`` / ``cal_lm_add`` on the same votes; the summary of a large hand-made table against the
restatement; ``GraphedTestStep`` against the eager chain (``build_ffb6d_item``, the eval forward and loss,
``TorchEval.eval_pose_parallel``) over three seeded batches for YCB (one camera matrix per frame) and LineMOD, with a
replay under the CUDA sync debug mode, ``reset()`` and a second run, and an overflowing batch; a capture in the
middle of a run; and the ``-test_gt`` sanity check of the reference's README.  Frames are 120x160 with 4096 points."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib, ops, pose
from ffb6d_b200.graphed import _tensors
from ffb6d_b200.item import pose_gt_objects
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D
from ffb6d_b200.synthetic import INTRINSICS, make_item_frame, make_pose_frame
from oracle import eval_record_oracle as O

pytestmark = pytest.mark.gpu

B, H, W, N, N_KPS = 2, 120, 160, 4096, 8
N_CLS = {"ycb": 4, "linemod": 2}
CAM_SCALE = {"ycb": 10000.0, "linemod": 1000.0}
K_OF = {"ycb": INTRINSICS["ycb_K1"], "linemod": INTRINSICS["linemod"]}
OBJ = 3                     # the LineMOD object's class id
SYM = (2,)
DIAMETER = 172.0


def _same(got, want, tol=1e-9):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    np.testing.assert_allclose(got[ok], want[ok], rtol=0, atol=tol)


# ------------------------------------------------------------------------------------------ record and summary
def _vote_batch(n_frames=6):
    frs = [make_pose_frame(60 + f) for f in range(n_frames)]
    n_obj, n_kps = 5, frs[0]["kp_of"].shape[0]
    cls_ids = np.zeros((n_frames, n_obj, 1), np.int32)
    RTs = np.zeros((n_frames, n_obj, 3, 4), np.float32)
    gt_kps = np.zeros((n_frames, n_obj, n_kps, 3), np.float32)
    for b, fr in enumerate(frs):
        for i, c in enumerate((1, 2, 3, 4)[: 4 - b % 2]):
            cls_ids[b, i, 0], RTs[b, i] = c, fr["poses"][c]
            gt_kps[b, i] = (fr["mesh"][c] @ fr["poses"][c][:, :3].T + fr["poses"][c][:, 3])[:n_kps]
    t = {k: torch.from_numpy(np.stack([f[k] for f in frs])).cuda() for k in ("pcld", "mask", "ctr_of", "kp_of")}
    rs = np.random.RandomState(3)
    meshes = {c: rs.uniform(-0.08, 0.08, (500, 3)).astype(np.float32) for c in range(1, 5)}
    return frs, t, torch.from_numpy(cls_ids).cuda(), torch.from_numpy(RTs).cuda(), torch.from_numpy(gt_kps).cuda(), \
        meshes


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_record_and_summary_against_torch_eval(cuda, dataset):
    frs, t, cls_ids, RTs, gt_kps, meshes = _vote_batch()
    n_cls = 5
    obj = 1 if dataset == "linemod" else 0
    te = pose.TorchEval(meshes, frs[0]["mesh"], frs[0]["cls_radius"], SYM, n_cls=n_cls)
    te.eval_pose_parallel(t["pcld"], None, t["mask"], t["ctr_of"], None, None, 0, cls_ids, RTs, t["kp_of"], gt_kps,
                          None, obj_id=obj, ds=dataset)
    bs, n_obj = RTs.shape[:2]
    rows = torch.full((bs * n_obj + 7, _lib.EVAL_ROW_WORDS), 12345, dtype=torch.int32, device="cuda")
    state = torch.zeros(4, dtype=torch.int64, device="cuda")
    if dataset == "ycb":
        votes, ids, pred, add, adds = pose._ycb_scores(te.mesh_table, te.vote_table, t["pcld"], t["mask"], t["ctr_of"],
                                                       t["kp_of"], cls_ids, RTs, True, True)
        pose._ycb_record(rows, state, votes, ids, pred, add, adds, gt_kps)
        want = O.record(ids.cpu().numpy(), votes[0].cpu().numpy(), pred.reshape(bs, n_obj, 3, 4).cpu().numpy(),
                        add.cpu().numpy(), adds.cpu().numpy(), kps=votes[2].cpu().numpy(), gt_kps=gt_kps.cpu().numpy())
    else:
        votes, pred, add, adds = pose._lm_scores(te.mesh_table, te.lm_tables[obj], obj, t["pcld"], t["mask"],
                                                 t["ctr_of"], t["kp_of"], RTs, True, True)
        pose._lm_record(rows, state, votes, obj, n_obj, pred, add, adds)
        want = O.record(np.zeros((bs, n_obj), np.int32), votes[0].cpu().numpy(), pred.cpu().numpy(),
                        add.cpu().numpy(), adds.cpu().numpy(), obj_id=obj)
    got = rows.cpu().numpy()
    assert state.tolist() == [bs * n_obj, bs, 0, 0]
    assert (got[bs * n_obj:] == 12345).all()                   # nothing past the batch
    got = got[:bs * n_obj]
    cols = [c for c in range(_lib.EVAL_ROW_WORDS) if c != 5]
    np.testing.assert_array_equal(got[:, cols], want[:, cols])
    np.testing.assert_allclose(got.view(np.float32)[:, 5], want.view(np.float32)[:, 5], rtol=4e-7, atol=0)
    # the summary, against TorchEval's on the lists it built from the same launch's rows
    lm_thr = DIAMETER / 1000.0 * 0.1
    auc, pct, kp = (x.cpu().numpy() for x in ops.eval_auc(rows, state, n_cls, torch.tensor(
        [c in SYM for c in range(n_cls)], device="cuda"), lm_thr))
    o_auc, o_pct, o_kp = O.summary(got, len(got), n_cls, SYM, lm_thr)
    _same(auc, o_auc)
    _same(pct, o_pct, 0)
    _same(kp, o_kp, 1e-12)
    if dataset == "ycb":
        r = te.cal_auc()
        for m, name in enumerate(("add_auc_lst", "adds_auc_lst", "add_s_auc_lst")):
            _same(auc[m], r[name])
        assert kp[1] == sum(map(len, r["pred_kp_errs"]))
        _same(kp[0] / kp[1], r["mean_kp_err"], 1e-12)
        assert sum(len(x) for x in te.cls_add_dis[1:]) == 21
    else:
        r = te.cal_lm_add(obj, DIAMETER)
        for m, name in enumerate(("add_auc_lst", "adds_auc_lst", "add_s_auc_lst")):
            _same([auc[m, obj]], r[name])
        assert pct[0, obj] == r["add"] and pct[1, obj] == r["adds"]
    flat = got.view(np.float32)
    keep = got[:, 0] != -1
    assert te.cls_add_dis[0] == [float(x) for x in flat[keep, 3]]     # the lists are the rows, bit for bit
    assert te.cls_adds_dis[0] == [float(x) for x in flat[keep, 4]]


def test_summary_of_a_large_table(cuda):
    """20 000 rows over 22 classes with ties, misses, inf, a NaN class and a count below the capacity; twice, for the
    same bits."""
    rs = np.random.RandomState(11)
    n, n_cls, cap = 20000, 22, 20500
    d = np.round(rs.uniform(0, 0.14, (n, 2)), 3).astype(np.float32)     # rounded: many ties, some above 0.1
    d[rs.rand(n) < 0.01] = np.inf
    cls = rs.randint(0, n_cls, (n // 10, 10)).astype(np.int32)
    cls[:, 0] = np.maximum(cls[:, 0], 1)
    rows = O.record(cls, rs.rand(n // 10, n_cls) < 0.5, rs.normal(size=(n // 10, 10, 3, 4)), d[:, 0], d[:, 1],
                    kps=rs.uniform(-0.1, 0.1, (n // 10, n_cls, 9, 3)).astype(np.float32),
                    gt_kps=rs.uniform(-0.1, 0.1, (n // 10, 10, 8, 3)).astype(np.float32))
    rows.view(np.float32)[rows[:, 0] == 7, 3] = np.nan
    full = np.concatenate([rows, np.tile(rows[:1], (cap - n, 1))])       # rows past the count are not read
    sym = (13, 16, 19, 20, 21)
    sym_d = torch.tensor([c in sym for c in range(n_cls)], device="cuda")
    rows_d = torch.from_numpy(full).cuda()
    state = torch.tensor([n, n // 10, 0, 0], dtype=torch.int64, device="cuda")
    first = [x.cpu().numpy() for x in ops.eval_auc(rows_d, state, n_cls, sym_d, 0.0172)]
    again = [x.cpu().numpy() for x in ops.eval_auc(rows_d, state, n_cls, sym_d, 0.0172)]
    for a, b in zip(first, again):
        assert a.tobytes() == b.tobytes()
    auc, pct, kp = first
    o_auc, o_pct, o_kp = O.summary(rows, n, n_cls, sym, 0.0172)
    _same(auc, o_auc)
    _same(pct, o_pct, 0)
    _same(kp, o_kp, 1e-9)
    assert np.isnan(auc[0, 7]) and np.isnan(auc[0, 0]) and not np.isnan(auc[1, 7])
    add, adds, add_s, _ = O.class_lists(rows, n, n_cls, sym)
    for c in (0, 1, 13):
        _same([auc[1, c], auc[2, c]], [pose.cal_auc(adds[c]), pose.cal_auc(add_s[c])])


# ------------------------------------------------------------------------------------------ GraphedTestStep
def _mesh_kps(dataset, seed=5):
    rs = np.random.RandomState(seed)
    ids = (OBJ,) if dataset == "linemod" else range(1, N_CLS["ycb"])
    return {c: np.concatenate([rs.uniform(-0.08, 0.08, (N_KPS, 3)), rs.uniform(-0.01, 0.01, (1, 3))]) for c in ids}


def _mesh_pts(dataset, seed=6):
    rs = np.random.RandomState(seed)
    ids = (OBJ,) if dataset == "linemod" else range(1, N_CLS["ycb"])
    return {c: rs.uniform(-0.08, 0.08, (700, 3)).astype(np.float32) for c in ids}


def _test_batch(seed, dataset, per_frame_K=False):
    """B frames whose objects use the meshes of ``_mesh_kps`` (so that ``-test_gt`` can recover their poses)."""
    ycb = dataset == "ycb"
    cls = (1, 2, 3) if ycb else (1,)
    mk = _mesh_kps(dataset)
    key = (lambda c: c) if ycb else (lambda c: OBJ)
    fr = [make_item_frame(seed * 31 + i, h=H, w=W, dataset=dataset, n_kps=N_KPS, cls_ids=cls, blobs=cls)
          for i in range(B)]
    objs = [pose_gt_objects(f["poses"], list(cls), [mk[key(c)][:-1] for c in cls], [mk[key(c)][-1] for c in cls],
                            4 if ycb else 2, N_KPS, dataset=dataset) for f in fr]
    batch = {"dpt": np.stack([f["raw"] for f in fr]), "rgb": np.stack([f["rgb"] for f in fr]),
             "labels": np.stack([f["labels"] for f in fr]), "nrm_map": np.stack([f["nrm"] for f in fr])}
    batch.update({k: np.stack([o[k] for o in objs]) for k in objs[0]})
    batch = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in batch.items()}
    if per_frame_K:
        batch["K"] = torch.from_numpy(np.stack([INTRINSICS[("ycb_K1", "ycb_K2")[i % 2]] for i in range(B)])).cuda()
    return batch


def _kw(dataset, **extra):
    kw = dict(dataset=dataset, cam_scale=CAM_SCALE[dataset], K=K_OF[dataset], mesh_pts=_mesh_pts(dataset),
              mesh_kps=_mesh_kps(dataset), sym_cls_ids=SYM, n_points=N, capacity=3 * B)
    if dataset == "ycb":
        kw["cls_radius"] = [0.08] * 21
    else:
        kw["obj_id"] = OBJ
    kw.update(extra)
    return kw


def _model(dataset):
    torch.manual_seed(0)
    return FFB6D(n_classes=N_CLS[dataset], n_pts=N, n_kps=N_KPS).cuda().eval()


def _eager(model, batch, te, dataset, test_gt=False):
    """The eager chain of one test batch, as model_fn runs it."""
    K = batch["K"].cpu().numpy() if "K" in batch else K_OF[dataset]
    item = F.build_ffb6d_item(batch["dpt"], CAM_SCALE[dataset], K, batch["rgb"], batch["labels"], batch["nrm_map"],
                              batch, N, seed=0, fill=dataset == "ycb")
    item["rgb"] = item["rgb"].float()
    with torch.no_grad():
        ep = model(item)
        loss, info = ffb6d_loss(ep, item, valid=item["valid"])
        cld = item["cld_rgb_nrm"][:, :3, :].permute(0, 2, 1).contiguous()
        if test_gt:
            mask, ctr = item["labels"], item["ctr_targ_ofst"].unsqueeze(2).permute(0, 2, 1, 3)
            kp = item["kp_targ_ofst"].permute(0, 2, 1, 3)
        else:
            mask, ctr, kp = torch.max(ep["pred_rgbd_segs"], 1)[1], ep["pred_ctr_ofs"], ep["pred_kp_ofs"]
        te.eval_pose_parallel(cld, item["rgb"], mask, ctr, item["ctr_targ_ofst"], item["labels"], 0, item["cls_ids"],
                              item["RTs"], kp, item["kp_3ds"], item["ctr_3ds"], min_cnt=1, use_ctr_clus_flter=True,
                              use_ctr=True, obj_id=OBJ if dataset == "linemod" else 0, ds=dataset)
    return ep, loss, info


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.reshape(-1).view(torch.uint8),
                                                                     b.reshape(-1).view(torch.uint8))


def _check_summary(got, te, dataset, infos):
    if dataset == "ycb":
        want = te.cal_auc()
        assert got["pred_kp_errs"] == want["pred_kp_errs"]
        _same(got["mean_kp_err"], want["mean_kp_err"], 1e-12)
        for k in ("add_auc_mean", "adds_auc_mean", "add_s_auc_mean"):
            _same(got[k], want[k])
        assert len(got["pred_id2pose_lst"]) == len(te.pred_id2pose_lst)
        for x, y in zip(got["pred_id2pose_lst"], te.pred_id2pose_lst):
            assert sorted(x) == sorted(y) and all(np.array_equal(x[k], y[k]) for k in x)
    else:
        want = te.cal_lm_add(OBJ, DIAMETER)
        assert got["add"] == want["add"] and got["adds"] == want["adds"]
        assert got["pred_id2pose_lst"] == []
    assert got["add_dis_lst"] == want["add_dis_lst"] and got["adds_dis_lst"] == want["adds_dis_lst"]
    for k in ("add_auc_lst", "adds_auc_lst", "add_s_auc_lst"):
        _same(got[k], want[k])
    for k in infos[0]:
        v = [i[k] for i in infos]
        _same(got["mean_eval_dict"][k], np.array(v).mean() * (100 if "acc" in k else 1), 1e-12)
    _same(got["mean_eval_dict"]["loss_target"], np.mean([i["loss_all"] for i in infos]), 1e-12)


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_graphed_equals_eager(cuda, dataset):
    """Three batches against the eager chain: outputs bit for bit, the summary as TorchEval's; a replay issues no
    package launch, and one runs under the sync debug mode; reset() and a second run give the same summary; a batch
    past the capacity leaves the table as it is and makes summary() raise."""
    model = _model(dataset)
    seq = [_test_batch(s, dataset, per_frame_K=dataset == "ycb") for s in (1, 2, 3)]
    step = F.GraphedTestStep(model, seq[0], **_kw(dataset))
    te = pose.TorchEval(_mesh_pts(dataset), _mesh_kps(dataset), [0.08] * 21 if dataset == "ycb" else None, SYM,
                        n_cls=N_CLS["ycb"] if dataset == "ycb" else 22)
    infos = []
    for i, batch in enumerate(seq):
        n0 = _lib.launch_count()
        if i == 1:
            torch.cuda.set_sync_debug_mode("error")
        try:
            ep, loss, info = step(batch)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert _lib.launch_count() == n0, "a replay called the library"
        got = [(path, t.clone()) for path, t in _tensors((ep, loss, info))]
        eager = _eager(model, batch, te, dataset)
        want = _tensors(eager)
        assert [p for p, _ in got] == [p for p, _ in want]
        for (path, g), (_, w) in zip(got, want):
            assert _bits_equal(g, w), "batch %d: %s differs" % (i, path)
        infos.append({k: v.item() for k, v in eager[2].items()})
    first = step.summary(DIAMETER)
    _check_summary(first, te, dataset, infos)
    step.reset()
    for batch in seq:
        step(batch)
    second = step.summary(DIAMETER)
    assert repr(second) == repr(first)
    assert step.captures == 1
    if dataset == "ycb":
        before = step._rows.clone()
        step(seq[0])                                             # a fourth batch: past the capacity of 3 batches
        torch.cuda.synchronize()
        assert torch.equal(step._rows, before) and step._state[2].item() == 1
        with pytest.raises(RuntimeError, match="did not fit"):
            step.summary()
        step.reset()
        step(seq[1])
        assert len(step.summary()["add_dis_lst"][0]) == 3 * B


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_test_gt_recovers_the_poses(cuda, dataset):
    """-test_gt: the vote from the labels and target offsets gives an ADD(-S) AUC of at least 99.99 for every class
    present (the reference README's check of the evaluation code)."""
    model = _model(dataset)
    seq = [_test_batch(s, dataset) for s in (4, 5, 6)]
    step = F.GraphedTestStep(model, seq[0], test_gt=True, **_kw(dataset))
    for batch in seq:
        step(batch)
    r = step.summary(DIAMETER)
    classes = (OBJ,) if dataset == "linemod" else (1, 2, 3)
    for c in classes:
        assert len(r["add_dis_lst"][c]) > 0
        auc = r["add_s_auc_lst"][0 if dataset == "linemod" else c]
        assert auc >= 99.99, (c, auc, r["add_dis_lst"][c])


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_capture_in_the_middle_of_a_run(cuda, dataset):
    """A parameter re-pointed at an equal clone changes the baked key but no value: the next call captures again, and
    its warm-up leaves the run's table and sums as they were, so the summary is that of a step that never captured
    again."""
    model = _model(dataset)
    seq = [_test_batch(s, dataset) for s in (1, 2, 3)]
    once = F.GraphedTestStep(model, seq[0], **_kw(dataset))
    for batch in seq:
        once(batch)
    want = once.summary(DIAMETER)
    step = F.GraphedTestStep(model, seq[0], **_kw(dataset))
    step(seq[0])
    step(seq[1])
    p = next(model.parameters())
    p.data = p.data.clone()
    step(seq[2])
    assert step.captures == 2 and once.captures == 1
    assert repr(step.summary(DIAMETER)) == repr(want)
