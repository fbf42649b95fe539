"""GPU: the depth-normal estimator (``ops.depth_normal``, DESIGN.md §4.30) and ``normals="device"``.

``depth_normal`` bit for bit against the numpy restatement (oracle/normal_oracle.py) on YCB- and LineMOD-shaped
480x640 frames with holes and per-frame camera matrices, all-zero and all-far maps, checkerboards around the difference
threshold, 1x1 frames and frames smaller than the stencil, widths off the tile, and k_size 1, 5 and the maximum; the
YCB millimetre map against numpy's cast; the item builders with ``normals="device"`` against the same call given the
oracle's map (YCB training: from the composed, completed depth); and the graphed steps with ``normals="device"``
against their eager compositions, replayed without a host synchronisation."""
import copy

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib, ops
from ffb6d_b200.graphed import _tensors
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.synthetic import INTRINSICS, make_item_frame
from frame_batches import CAM_SCALE, K_OF, make_train_batch
from oracle.normal_oracle import depth_normal as oracle_normal, depth_normal_K, ycb_mm

pytestmark = pytest.mark.gpu

FX, FY = 1066.778, 1067.487


def _bits(t):
    return t.contiguous().reshape(-1).view(torch.uint8)


def _check(D, fx=FX, fy=FY, **kw):
    """depth_normal of the uint16 map ``D`` ([H,W] or [B,H,W]) against the oracle, bit for bit."""
    B = 1 if D.ndim == 2 else D.shape[0]
    fxb, fyb = np.broadcast_to(np.float64(fx), (B,)), np.broadcast_to(np.float64(fy), (B,))
    intr = torch.tensor(np.stack([fxb, fyb, np.zeros(B), np.zeros(B)], 1), dtype=torch.float64, device="cuda")
    got = F.depth_normal(torch.from_numpy(np.ascontiguousarray(D)).cuda(), intr if B > 1 or D.ndim == 3 else intr[0],
                         **kw).cpu().numpy()
    want = oracle_normal(D, fxb if D.ndim == 3 else fxb[0], fyb if D.ndim == 3 else fyb[0], **kw)
    assert got.shape == want.shape and got.dtype == np.float32
    bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)).any(-1))
    assert bad.size == 0, "%d pixels differ, first %s: %s vs %s" % (bad.size, bad[0], got.reshape(-1, 3)[bad[0]],
                                                                     want.reshape(-1, 3)[bad[0]])
    return got


# ------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_dataset_frames(cuda, dataset):
    fr = [make_item_frame(s, dataset=dataset) for s in (3, 4, 5)]
    raw = np.stack([f["raw"] for f in fr])
    D = ycb_mm(raw.astype(np.float32)) if dataset == "ycb" else raw
    assert (D == 0).mean() > 0.05
    Ks = np.stack([INTRINSICS[n] for n in ("ycb_K1", "linemod", "ycb_K2")])
    for into in (False, True):
        want = depth_normal_K(D, Ks, point_into_surface=into)
        for K in (Ks, ops._frame_intrinsics(torch.from_numpy(Ks).cuda())):         # host matrices, device (fx,fy,cx,cy)
            got = F.depth_normal(torch.from_numpy(D).cuda(), K, point_into_surface=into).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (dataset, into)
        nz = (np.abs(want).sum(-1) > 0).mean()
        assert 0.2 < nz < 0.95, nz                   # both fitted and zero normals occur
    one = F.depth_normal(torch.from_numpy(D[1]).cuda(), Ks[1]).cpu().numpy()      # [H,W] with a [3,3] K
    assert np.array_equal(one.view(np.uint32), depth_normal_K(D[1], Ks[1]).view(np.uint32))


def test_empty_and_far_maps(cuda):
    assert not _check(np.zeros((2, 37, 45), np.uint16)).any()
    rs = np.random.RandomState(1)
    assert not _check(rs.randint(2000, 65536, (2, 37, 45)).astype(np.uint16)).any()
    assert not _check(np.full((30, 40), 65535, np.uint16), distance_threshold=65535).any()
    assert _check(np.full((30, 40), 65535, np.uint16), distance_threshold=65536).any()


@pytest.mark.parametrize("t", [19, 20, 21])
@pytest.mark.parametrize("cell", [1, 3, 5])
def test_checkerboards(cuda, t, cell):
    y, x = np.mgrid[:64, :96]
    D = (1000 + t * (((y // cell) + (x // cell)) % 2) + (x // 7)).astype(np.uint16)
    _check(D)
    _check(D, k_size=cell)


@pytest.mark.parametrize("hw", [(1, 1), (1, 700), (700, 1), (3, 4), (10, 10), (11, 11), (7, 40)])
def test_small_frames(cuda, hw):
    rs = np.random.RandomState(hw[0] * 1000 + hw[1])
    D = (800 + rs.randint(-12, 13, (2,) + hw)).astype(np.uint16)
    _check(D, fx=[FX, 572.4], fy=[FY, 573.6])
    _check(D, k_size=1)


@pytest.mark.parametrize("W", [1, 31, 33, 65, 100, 641])
@pytest.mark.parametrize("k_size", [1, 5, _lib.NRM_MAX_KSIZE])
def test_widths_and_k_sizes(cuda, W, k_size):
    rs = np.random.RandomState(W + k_size)
    H = 19
    y, x = np.mgrid[:H, :W]
    D = (1500 + 3 * x - 2 * y + rs.randint(-9, 10, (H, W))).astype(np.int64)
    D[rs.rand(H, W) < 0.1] = 0
    D[rs.rand(H, W) < 0.05] = 2100
    D = np.stack([D, D[::-1]]).astype(np.uint16)
    _check(D, fx=[FX, 572.4], fy=[FY, 573.6], k_size=k_size)
    _check(D, k_size=k_size, distance_threshold=1600, difference_threshold=7, point_into_surface=True)


def test_ycb_millimetres(cuda):
    fr = [make_item_frame(s) for s in (7, 8)]
    filled = F.fill_missing(torch.from_numpy(np.stack([f["raw"] for f in fr])).cuda(), 10000.0)
    assert torch.equal(ops.depth_to_mm(filled).cpu(), torch.from_numpy(ycb_mm(filled.cpu().numpy())))
    mm = np.arange(1, 6000, 7)
    k = mm.astype(np.float32) * 10
    v = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(1e9)), k + 9.999999,
                        np.float32([0.5, 9.9999995, 10.000001])]).astype(np.float32)
    got = ops.depth_to_mm(torch.from_numpy(v).cuda()).cpu().numpy()
    assert np.array_equal(got, ycb_mm(v))
    assert (got[len(k):2 * len(k)] == mm - 1).all()          # just below an integer millimetre


# ------------------------------------------------------------------------------------------ the item builders
N = 480 * 640 // 24


def _frames(dataset, per_frame_K):
    ycb = dataset == "ycb"
    fr = [make_item_frame(s, dataset=dataset, n_kps=8, cls_ids=(1, 5) if ycb else (1,), blobs=(1, 5) if ycb else (1,))
          for s in (21, 22)]
    b = {k: torch.from_numpy(np.stack([f[src] for f in fr])).cuda()
         for k, src in (("dpt", "raw"), ("rgb", "rgb"), ("labels", "labels"))}
    from ffb6d_b200.item import pose_gt_objects
    objs = [pose_gt_objects(f["poses"], f["cls_ids"] if ycb else [1], f["kps"], f["ctrs"], 6 if ycb else 2, 8,
                            dataset=dataset) for f in fr]
    K = np.stack([INTRINSICS["ycb_K1"], INTRINSICS["ycb_K2"]]) if per_frame_K else K_OF[dataset]
    return b, objs, K


def _oracle_map(dpt, dataset, K):
    """The normals the reference computes: YCB from the completed depth's millimetre map, LineMOD from dpt_mm."""
    if dataset == "ycb":
        D = ycb_mm(F.fill_missing(dpt, CAM_SCALE["ycb"]).cpu().numpy())
    else:
        D = dpt.cpu().numpy()
    K = np.broadcast_to(np.asarray(K, np.float64), (D.shape[0], 3, 3))
    return torch.from_numpy(depth_normal_K(D, K)).cuda()


@pytest.mark.parametrize("dataset,per_frame_K", [("ycb", False), ("ycb", True), ("linemod", False)])
def test_item_builders(cuda, dataset, per_frame_K):
    b, objs, K = _frames(dataset, per_frame_K)
    fill, cs = dataset == "ycb", CAM_SCALE[dataset]
    nrm = _oracle_map(b["dpt"], dataset, K)
    pairs = [(F.build_ffb6d_inputs(b["dpt"], cs, K, b["rgb"], None, N, seed=3, fill=fill, normals="device"),
              F.build_ffb6d_inputs(b["dpt"], cs, K, b["rgb"], nrm, N, seed=3, fill=fill)),
             (F.build_ffb6d_item(b["dpt"], cs, K, b["rgb"], b["labels"], None, objs, N, seed=3, fill=fill,
                                 normals="device"),
              F.build_ffb6d_item(b["dpt"], cs, K, b["rgb"], b["labels"], nrm, objs, N, seed=3, fill=fill))]
    for got, want in pairs:
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and torch.equal(_bits(got[k]), _bits(want[k])), k


def _integration_upto_depth(batch, dataset, seed):
    """INTEGRATION.md's trainer lines up to add_real_back: the image and the composed depth."""
    rgb = F.color_jitter(batch["rgb"], batch["jitter"].numpy(), active=batch["jittered"])
    rgb = F.rgb_add_noise(rgb, batch["plans"][:, 0].numpy(), seed=seed)
    rgb, dpt = F.add_real_back(rgb, batch["labels"], batch["dpt"], batch["back_rgb"], batch["back_labels"],
                               batch["back_dpt"], batch["apply_rgb"], dataset, active=batch["augment"])
    return F.rgb_add_noise(rgb, batch["plans"][:, 1].numpy(), seed=seed), dpt


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_train_item_from_composed_depth(cuda, dataset):
    H, W, n = 120, 160, 4096
    batch = make_train_batch(4, dataset, 4, H, W, 22 if dataset == "ycb" else 2, per_frame_K=dataset == "ycb")
    assert batch["augment"].any()
    dev_batch = {k: v for k, v in batch.items() if k != "nrm_map"}
    rgb, dpt = _integration_upto_depth(batch, dataset, 77)
    K = batch["K"].cpu().numpy() if "K" in batch else K_OF[dataset]
    nrm = _oracle_map(dpt, dataset, K)
    if dataset == "ycb":      # the background depth is composed before the completion: the normals change with it
        assert not torch.equal(nrm, _oracle_map(batch["dpt"], dataset, K))
    want = F.build_ffb6d_item(dpt, CAM_SCALE[dataset], K, rgb, batch["labels"], nrm, batch, n, seed=77,
                              fill=dataset == "ycb")
    want["rgb"] = want["rgb"].float()
    got = F.build_ffb6d_train_item(dev_batch, dataset=dataset, cam_scale=CAM_SCALE[dataset], K=K_OF[dataset],
                                   n_points=n, seed=77, normals="device")
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and torch.equal(_bits(got[k]), _bits(want[k])), (dataset, k)


# ------------------------------------------------------------------------------------------ the graphed steps
def _replay(step, *args, **kw):
    """One call under the CUDA sync debug mode, which must issue no library launch; its outputs cloned."""
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = step(*args, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.launch_count() == n0, "a replay called the library"
    return [(p, t.clone()) for p, t in _tensors(out)]


def _assert_same(got, want, when):
    want = _tensors(want)
    assert [p for p, _ in got] == [p for p, _ in want], when
    for (p, g), (_, w) in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and torch.equal(_bits(g), _bits(w)), (when, p)


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_graphed_pose_step(cuda, dataset):
    import test_gpu_estimate as E
    model = E.FFB6D(n_classes=E.N_CLS[dataset], n_pts=E.N, n_kps=E.N_KPS).to(cuda).eval()
    seq = []
    for s in ((31, 32), (33, 34)):
        f = E._batch(s, dataset, cuda, per_frame_K=dataset == "linemod")[0]
        del f["nrm_map"]
        seq.append(f)
    kw = E._kw(dataset)
    step = F.GraphedPoseStep(model, seq[0], seed=4, warmup=1, normals="device", **kw)
    for i in (0, 1, 0):
        got = _replay(step, seq[i])
        _assert_same(got, F.estimate_poses(model, seq[i], seed=4, normals="device", **kw), "%s batch %d" % (dataset, i))
    assert step.captures == 1


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_graphed_test_step(cuda, dataset):
    import test_gpu_test_step as T
    model = T._model(dataset)
    seq = []
    for s in (1, 2):
        b = T._test_batch(s, dataset, per_frame_K=dataset == "ycb")
        del b["nrm_map"]
        seq.append(b)
    step = F.GraphedTestStep(model, seq[0], normals="device", **T._kw(dataset))
    for i, b in enumerate(seq):
        got = _replay(step, b)
        K = b["K"].cpu().numpy() if "K" in b else T.K_OF[dataset]
        item = F.build_ffb6d_item(b["dpt"], T.CAM_SCALE[dataset], K, b["rgb"], b["labels"], None, b, T.N, seed=0,
                                  fill=dataset == "ycb", normals="device")
        item["rgb"] = item["rgb"].float()
        with torch.no_grad():
            ep = model(item)
            loss, info = ffb6d_loss(ep, item, valid=item["valid"])
        _assert_same(got, (ep, loss, info), "%s batch %d" % (dataset, i))
    assert step.captures == 1


def test_graphed_frame_train_step(cuda):
    import test_gpu_frame_step as S
    seq = []
    for s in (11, 12, 13):
        b = make_train_batch(s, "ycb", S.B, S.H, S.W, S.N_CLS, per_frame_K=True)
        del b["nrm_map"]
        seq.append(b)
    S.deterministic(True)
    try:
        model = S.make_model()
        twin = copy.deepcopy(model)
        opt, opt_e = S.adam(model), S.adam(twin)
        step = F.GraphedFrameTrainStep(model, opt, seq[0], warmup=1, normals="device", **S.KW)
        for i, (batch, seed) in enumerate(zip(seq, (5, 9, 6))):
            # the first call may wait for a staging slot; later ones must not synchronise
            got = _replay(step, batch, seed=seed) if i else [(p, t.clone()) for p, t in _tensors(step(batch, seed=seed))]
            item = F.build_ffb6d_train_item(batch, seed=seed, normals="device", **S.KW)
            opt_e.zero_grad(set_to_none=True)
            loss, info = ffb6d_loss(twin(item), item, valid=item["valid"])
            loss.backward()
            opt_e.step()
            _assert_same(got, (loss.detach(), info), "step %d" % i)
            S.assert_state_equal(model, opt, twin, opt_e, "step %d" % i)
        assert step.captures == 1
    finally:
        S.deterministic(False)
