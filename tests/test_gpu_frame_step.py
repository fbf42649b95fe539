"""GPU: training from decoded frames (:func:`ffb6d_b200.build_ffb6d_train_item`, :class:`GraphedFrameTrainStep`,
DESIGN.md §4.28).

The ``_dseed`` entry points against the by-value ones; ``build_ffb6d_train_item`` against INTEGRATION.md's trainer
lines for YCB and LineMOD; three graphed steps against three eager steps of a deep copy trained through
``build_ffb6d_train_item``, bit for bit under ``torch.use_deterministic_algorithms(True)``, with a bad record and a bad
plan rejected in between; a call under the CUDA sync debug mode; and the rejections.  Frames are 120x160 with 4096
points, as in test_gpu_graphed_step."""
import copy

import numpy as np
import pytest
import torch
import torch.distributed as dist

import ffb6d_b200 as F
from ffb6d_b200 import _lib, augment as A
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D, FFB6DFusionNet
from ffb6d_b200.synthetic import make_aug_frame
from frame_batches import CAM_SCALE, K_OF, integration_item, make_train_batch

pytestmark = pytest.mark.gpu

B, H, W, N, N_KPS, N_CLS = 3, 120, 160, 4096, 8, 4
LR = 1e-3
SEEDS = (0, 1, 2 ** 32 + 7, 2 ** 64 - 1)


def _dev_seed(s, dtype=torch.int64):
    return torch.tensor([s - (1 << 64) if s >= 1 << 63 else s], dtype=torch.int64, device="cuda").view(dtype)


def _bits(t):
    return t.contiguous().view(torch.uint8)


# ------------------------------------------------------------------------------------------------ seed on the device
@pytest.mark.parametrize("seed", SEEDS)
def test_dseed_equals_by_value(cuda, seed):
    rs = np.random.RandomState(5)
    depth = torch.from_numpy(np.where(rs.rand(2, 60, 70) < 0.3, 0, rs.rand(2, 60, 70)).astype(np.float32)).cuda()
    for n in (512, 5000):                                  # a subset, and the 'wrap' of fewer valid pixels
        want = F.sample_valid_pixels(depth, n, seed=seed, return_count=True)
        for dtype in (torch.int64, torch.uint64):
            got = F.sample_valid_pixels(depth, n, seed=_dev_seed(seed, dtype), return_count=True)
            assert all(torch.equal(g, w) for g, w in zip(got, want)), (seed, n, dtype)
    af = [make_aug_frame(s, h=40, w=45) for s in (1, 2)]
    rgb = torch.from_numpy(np.stack([f["rgb"] for f in af])).cuda()
    rec = np.stack([A.draw_rgb_noise(np.random.RandomState(8 + i), "ycb", pass_=i) for i in range(2)])
    rec[:, A.I_NOISE] = rec[:, A.I_FINAL] = 1
    want = F.rgb_add_noise(rgb, rec, seed)
    for dtype in (torch.int64, torch.uint64):
        assert torch.equal(F.rgb_add_noise(rgb, rec, _dev_seed(seed, dtype)), want), (seed, dtype)


def test_dseed_rejects_bad_seed_tensors(cuda):
    depth = torch.ones(1, 8, 8, device="cuda")
    for bad in (torch.zeros(2, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda"),
                torch.zeros(1, dtype=torch.int64)):
        with pytest.raises(ValueError, match="tensor seed"):
            F.sample_valid_pixels(depth, 16, seed=bad)


# ------------------------------------------------------------------------------------------------ the composition
@pytest.mark.parametrize("dataset,per_frame_K", [("ycb", True), ("ycb", False), ("linemod", False)])
def test_train_item_equals_integration(cuda, dataset, per_frame_K):
    batch = make_train_batch(4, dataset, 4, H, W, 22 if dataset == "ycb" else 2, per_frame_K=per_frame_K)
    assert batch["augment"].any() and not batch["augment"].all()
    assert batch["jittered"].any() and not batch["jittered"].all()
    assert (batch["apply_rgb"] & batch["augment"]).any() and (~batch["apply_rgb"] & batch["augment"]).any()
    want = integration_item(batch, dataset, K_OF[dataset], N, 77)
    for seed in (77, _dev_seed(77)):
        got = F.build_ffb6d_train_item(batch, dataset=dataset, cam_scale=CAM_SCALE[dataset], K=K_OF[dataset],
                                       n_points=N, seed=seed)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and torch.equal(_bits(got[k]), _bits(want[k])), (dataset, k)


def test_train_item_rejects(cuda):
    batch = make_train_batch(4, "ycb", 2, H, W, 22)
    kw = dict(cam_scale=1e4, K=K_OF["ycb"], n_points=N, seed=0)
    with pytest.raises(ValueError, match="dataset"):
        F.build_ffb6d_train_item(batch, dataset="coco", **kw)
    with pytest.raises(ValueError, match="lacks"):
        F.build_ffb6d_train_item({k: v for k, v in batch.items() if k != "plans"}, dataset="ycb", **kw)


# ------------------------------------------------------------------------------------------------ the graphed step
def deterministic(on):
    torch.use_deterministic_algorithms(on)
    torch.backends.cudnn.deterministic = on


def make_model():
    torch.manual_seed(3)
    model = FFB6D(n_classes=N_CLS, n_pts=N, n_kps=N_KPS, fused_image_head=True).cuda()
    for m in model.modules():
        if isinstance(m, torch.nn.modules.dropout._DropoutNd):
            m.p = 0.0                          # the runs are compared bit for bit
    return model.train()


def adam(model):
    return torch.optim.Adam(model.parameters(), lr=torch.tensor(LR, device="cuda"), capturable=True)


KW = dict(dataset="ycb", cam_scale=CAM_SCALE["ycb"], K=K_OF["ycb"], n_points=N)


def batches():
    return [make_train_batch(s, "ycb", B, H, W, N_CLS, per_frame_K=True) for s in (11, 12, 13)]


def eager_step(model, opt, batch, seed):
    item = F.build_ffb6d_train_item(batch, seed=seed, **KW)
    opt.zero_grad(set_to_none=True)
    loss, info = ffb6d_loss(model(item), item, valid=item["valid"])
    loss.backward()
    opt.step()
    return loss.detach(), info


def assert_state_equal(mg, og, me, oe, when, with_adam=True):
    pairs = list(zip(mg.parameters(), me.parameters())) + list(zip(mg.buffers(), me.buffers()))
    for pg, pe in zip(mg.parameters(), me.parameters()) if with_adam else ():
        sg, se = og.state.get(pg, {}), oe.state.get(pe, {})
        assert sorted(sg) == sorted(se), when
        pairs += [(sg[k], se[k]) for k in sg]
    diff = sum(not torch.equal(a, b) for a, b in pairs)
    assert diff == 0, "%s: %d of %d tensors differ" % (when, diff, len(pairs))


def test_graphed_equals_eager(cuda):
    seq = batches()
    seeds = (5, 2 ** 63 + 9, 6)
    deterministic(True)
    try:
        model = make_model()
        twin = copy.deepcopy(model)
        opt, opt_e = adam(model), adam(twin)
        step = F.GraphedFrameTrainStep(model, opt, seq[0], warmup=2, **KW)
        # the warm-up left no trace (its Adam state is zeroed; the eager twin has none before its first step)
        assert_state_equal(model, opt, twin, opt_e, "after the warm-up", with_adam=False)
        for i, (batch, seed) in enumerate(zip(seq, seeds)):
            if i == 2:
                # a bad jitter plan or noise record: FFB6DError before anything is copied; the step stays usable
                bad = dict(batch, jitter=batch["jitter"].clone())
                bad["jitter"][1, 7] = 0.7
                with pytest.raises(_lib.FFB6DError, match="color_jitter: frame 1: bad plan"):
                    step(bad, seed=99)
                bad = dict(batch, plans=batch["plans"].clone())
                bad["plans"][2, 1, A.I_GAUSS_K] = 4
                with pytest.raises(_lib.FFB6DError, match="rgb_add_noise: frame 2: bad record"):
                    step(bad, seed=99)
            loss, info = step(batch, seed=seed)
            loss_e, info_e = eager_step(twin, opt_e, batch, seed)
            assert torch.equal(loss, loss_e), "step %d: loss" % i
            assert sorted(info) == sorted(info_e)
            assert all(torch.equal(info[k], info_e[k]) for k in info), "step %d: info" % i
            assert_state_equal(model, opt, twin, opt_e, "step %d" % i)
            assert step.captures == 1
    finally:
        deterministic(False)


def test_no_host_sync_after_the_first_call(cuda):
    seq = batches()
    model = make_model()
    step = F.GraphedFrameTrainStep(model, adam(model), seq[0], warmup=1, **KW)
    step(seq[1], seed=1)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(3):                     # every staging slot, reused
            step(seq[i], seed=2 + i)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert step.captures == 1


def test_rejects_mismatched_batches(cuda):
    seq = batches()
    model = make_model()
    step = F.GraphedFrameTrainStep(model, adam(model), seq[0], warmup=1, **KW)
    b = seq[1]
    bad = [({k: v for k, v in b.items() if k != "back_dpt"}, "keys"),
           (dict(b, extra=b["dpt"]), "keys"),
           (dict(b, labels=b["labels"][:, :, :W // 2]), "captured for"),
           (dict(b, K=b["K"].float()), "captured for"),
           (dict(b, plans=b["plans"][:, :, :512]), "captured for"),
           (dict(b, jittered=b["jittered"].to(torch.uint8)), "captured for"),
           (dict(b, jitter=b["jitter"].cuda()), "on the host"),
           (dict(b, dpt=b["dpt"].cpu()), "on the device")]
    for batch, what in bad:
        with pytest.raises(ValueError, match=what):
            step(batch, seed=3)
    for seed in (-1, 1 << 64, 1.5, torch.zeros(2, dtype=torch.int64, device="cuda")):
        with pytest.raises(ValueError):
            step(b, seed=seed)
    loss, _ = step(b, seed=3)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item() and step.captures == 1


def test_rejects_what_cannot_be_captured(cuda, monkeypatch, tmp_path):
    assert not _lib.lib.ffb6d_check_indices_enabled()
    batch = batches()[0]
    fusion = FFB6DFusionNet(n_classes=N_CLS, n_pts=N, n_kps=N_KPS).cuda().train()
    with pytest.raises(ValueError, match="FFB6DFusionNet"):
        F.GraphedFrameTrainStep(fusion, adam(fusion), batch, **KW)
    model = make_model()
    model.eval()
    with pytest.raises(ValueError, match="eval mode"):
        F.GraphedFrameTrainStep(model, adam(model), batch, **KW)
    model.train()
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="FFB6D_CHECK_INDICES"):
        F.GraphedFrameTrainStep(model, adam(model), batch, **KW)
    monkeypatch.delenv("FFB6D_CHECK_INDICES")
    dist.init_process_group("gloo", init_method="file://%s" % (tmp_path / "store"), rank=0, world_size=1)
    try:
        ddp = torch.nn.parallel.DistributedDataParallel(model)
        with pytest.raises(ValueError, match="DataParallel"):
            F.GraphedFrameTrainStep(ddp, adam(model), batch, **KW)
    finally:
        dist.destroy_process_group()
    torch.cuda.synchronize()
