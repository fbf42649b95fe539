"""GPU: FFB6D's training loss (ffb6d_b200.loss over csrc/loss.cu) against the reference's own models/loss.py as
recorded in tests/golden/loss_cases.npz, and against oracle/loss_oracle.py at training sizes: masks, label types,
out-of-range labels, determinism, CUDA-graph capture, and the whole item -> network -> loss -> backward chain."""
import numpy as np
import pytest
import torch

from ffb6d_b200 import loss as L
from oracle import loss_oracle as O
from test_loss_oracle import KEYS, _case_names, alpha_of, case, rel

pytestmark = pytest.mark.gpu


def dev(a, cuda, grad=False):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return t.requires_grad_(True) if grad else t


def bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


# --------------------------------------------------------------------------- against the reference's fixture
@pytest.mark.parametrize("label_dtype", [np.int64, np.int32])
@pytest.mark.parametrize("name", _case_names("focal"))
def test_focal_fixture(cuda, name, label_dtype):
    c = case("focal", name)
    x = dev(c["logits"], cuda, True)
    crit = L.FocalLoss(gamma=float(c["gamma"]), alpha=alpha_of(c), size_average=bool(c["size_average"]))
    loss = crit(x, dev(c["labels"].astype(label_dtype), cuda))
    loss.backward(torch.tensor(float(c["g"]), device=cuda))
    want64, _, grad64 = O.focal_loss(c["logits"], c["labels"], float(c["gamma"]), alpha_of(c),
                                     bool(c["size_average"]), grad_loss=float(c["g"]))
    assert rel(loss.item(), c["loss"]) <= 1e-5
    assert rel(loss.item(), want64) <= 2e-6
    assert np.abs(x.grad.cpu().numpy() - c["grad"]).max() <= 1e-6 * abs(float(c["g"]))


@pytest.mark.parametrize("label_dtype", [np.int32, np.int64])
@pytest.mark.parametrize("name", _case_names("of"))
def test_of_fixture(cuda, name, label_dtype):
    c = case("of", name)
    p = dev(c["pred"], cuda, True)
    out = L.OFLoss()(p, dev(c["targ"], cuda), dev(c["labels"].astype(label_dtype), cuda))
    out.backward(dev(c["g"], cuda))
    got = out.detach().cpu().numpy()
    want64 = O.of_l1_loss(c["pred"], c["targ"], c["labels"])
    assert np.all(np.abs(got - c["out"]) <= 1e-5 * np.abs(c["out"]))
    assert np.all(np.abs(got - want64) <= 2e-6 * np.abs(want64))
    assert np.array_equal(bits(p.grad), c["grad"].view(np.uint32))


@pytest.mark.parametrize("name", _case_names("model"))
def test_model_block_fixture(cuda, name):
    c = case("model", name)
    ep = {k: dev(c[k], cuda, True) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    item = {k: dev(c[k], cuda) for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst", "valid")}
    loss, info = L.ffb6d_loss(ep, item, valid=item["valid"])
    loss.backward()
    want64 = O.ffb6d_loss({k: c[k] for k in ep}, {k: c[k] for k in item}, valid=c["valid"])
    for k in KEYS:
        assert info[k].is_cuda and info[k].dim() == 0
        assert rel(info[k].item(), c[k]) <= 1e-5, k
        assert rel(info[k].item(), want64[k]) <= 2e-6, k
    assert loss.item() == info["loss_all"].item()
    for k in ("pred_kp_ofs", "pred_ctr_ofs"):
        assert np.array_equal(bits(ep[k].grad), c["grad_" + k].view(np.uint32)), k
    assert np.abs(ep["pred_rgbd_segs"].grad.cpu().numpy() - c["grad_pred_rgbd_segs"]).max() <= 1e-6


# --------------------------------------------------------------------------- training sizes against the oracle
def training_batch(cuda, B, C, K, N, seed):
    rs = np.random.RandomState(seed)
    labels = rs.randint(0, C, (B, N))
    labels[rs.rand(B, N) < 0.6] = 0
    a = dict(pred_rgbd_segs=(rs.randn(B, C, N) * 3).astype(np.float32),
             pred_kp_ofs=rs.randn(B, K, N, 3).astype(np.float32), pred_ctr_ofs=rs.randn(B, 1, N, 3).astype(np.float32),
             labels=labels.astype(np.int32), kp_targ_ofst=rs.randn(B, N, K, 3).astype(np.float32),
             ctr_targ_ofst=rs.randn(B, N, 3).astype(np.float32))
    return a


MASKS = {"all": [1] * 8, "mixed": [1, 0, 1, 1, 0, 0, 1, 1], "one": [0, 0, 0, 0, 0, 1, 0, 0], "none": [0] * 8}


@pytest.mark.parametrize("mask", sorted(MASKS))
@pytest.mark.parametrize("C", [2, 22])
def test_training_size_against_oracle(cuda, C, mask):
    B, K, N = 8, 8, 12288
    a = training_batch(cuda, B, C, K, N, seed=C + len(mask))
    valid = np.asarray(MASKS[mask], bool)
    ep = {k: dev(a[k], cuda, True) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    item = {k: dev(a[k], cuda) for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst")}
    v = dev(valid, cuda)
    loss, info = L.ffb6d_loss(ep, item, valid=v)
    loss.backward()
    want64 = O.ffb6d_loss({k: a[k] for k in ep}, {k: a[k] for k in item}, valid=valid)
    for k in KEYS:
        w = want64[k]
        assert abs(info[k].item() - w) <= 2e-6 * abs(w), (k, info[k].item(), w)
    if not valid.any():
        assert all(info[k].item() == 0 for k in KEYS)
        for t in ep.values():
            assert not t.grad.any()
        return
    # the reference's float32 torch ops on the sub-batch x[valid], on the same GPU
    ep_ref = {k: t.detach().clone().requires_grad_(True) for k, t in ep.items()}
    ref_loss, ref_info = O.ffb6d_loss_torch(ep_ref, item, valid=v)
    ref_loss.backward()
    for k in KEYS:
        assert rel(info[k].item(), ref_info[k].item()) <= 1e-5, k
    for k in ("pred_kp_ofs", "pred_ctr_ofs"):
        assert torch.equal(ep[k].grad, ep_ref[k].grad), k
    g = ep["pred_rgbd_segs"].grad
    assert (g - ep_ref["pred_rgbd_segs"].grad).abs().max().item() <= 1e-6
    assert not g[~v].any() and not ep["pred_kp_ofs"].grad[~v].any()


@pytest.mark.parametrize("C", [2, 22])
def test_focal_gradient_against_oracle(cuda, C):
    a = training_batch(cuda, 4, C, 1, 12288, seed=3)
    x = dev(a["pred_rgbd_segs"], cuda, True)
    valid = np.array([1, 0, 1, 1], bool)
    loss = L.FocalLoss(gamma=2)(x, dev(a["labels"].astype(np.int64), cuda), valid=dev(valid, cuda))
    loss.backward()
    want, _, grad = O.focal_loss(a["pred_rgbd_segs"], a["labels"], 2.0, valid=valid)
    assert rel(loss.item(), want) <= 2e-6
    assert np.abs(x.grad.cpu().numpy() - grad).max() <= 1e-6


def test_int32_and_int64_labels_agree(cuda):
    a = training_batch(cuda, 8, 22, 8, 12288, seed=9)
    res = []
    for dt in (torch.int32, torch.int64):
        ep = {k: dev(a[k], cuda, True) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
        item = {k: dev(a[k], cuda) for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst")}
        item["labels"] = item["labels"].to(dt)
        loss, info = L.ffb6d_loss(ep, item, valid=dev(np.array(MASKS["mixed"], bool), cuda))
        loss.backward()
        res.append([info[k] for k in KEYS] + [t.grad for t in ep.values()])
    for x, y in zip(*res):
        assert torch.equal(x, y)


def test_reduce_and_rows_input(cuda):
    a = training_batch(cuda, 4, 22, 8, 1000, seed=5)
    p, t, lab = dev(a["pred_kp_ofs"], cuda), dev(a["kp_targ_ofst"], cuda), dev(a["labels"], cuda)
    v = np.array([0, 1, 1, 0], bool)
    got = L.of_l1_loss(p, t, lab, reduce=True, valid=dev(v, cuda)).item()
    assert rel(got, O.of_l1_loss(a["pred_kp_ofs"], a["kp_targ_ofst"], a["labels"])[v].mean()) <= 2e-6
    assert rel(L.of_l1_loss(p, t, lab, reduce=True).item(),
               O.of_l1_loss(a["pred_kp_ofs"], a["kp_targ_ofst"], a["labels"]).mean()) <= 2e-6
    rows = a["pred_rgbd_segs"][0].T.copy()                      # [M, C]
    x = dev(rows, cuda, True)
    loss = L.FocalLoss(gamma=2)(x, dev(a["labels"][0], cuda))
    loss.backward()
    want, _, grad = O.focal_loss(rows, a["labels"][0], 2.0)
    assert rel(loss.item(), want) <= 2e-6 and np.abs(x.grad.cpu().numpy() - grad).max() <= 1e-6


def test_out_of_range_labels_give_nan(cuda):
    """Labels outside [0, C) are never read through: their terms and gradient rows are NaN, the rest stay finite."""
    a = training_batch(cuda, 2, 22, 8, 4096, seed=11)
    lab = a["labels"].astype(np.int64)
    lab[0, 7], lab[1, 100], lab[1, 4095] = 22, -1, 1 << 40
    x = dev(a["pred_rgbd_segs"], cuda, True)
    loss = L.FocalLoss(gamma=2)(x, dev(lab, cuda))
    loss.backward()
    assert torch.isnan(loss)
    g = x.grad.cpu().numpy()
    bad = np.zeros(lab.shape, bool)
    bad[0, 7] = bad[1, 100] = bad[1, 4095] = True
    assert np.isnan(g.transpose(0, 2, 1)[bad]).all() and np.isfinite(g.transpose(0, 2, 1)[~bad]).all()
    alpha = L.FocalLoss(gamma=2, alpha=[0.5] * 22)(x.detach(), dev(lab, cuda))
    assert torch.isnan(alpha)


# --------------------------------------------------------------------------- determinism and CUDA graphs
def _run(ep0, item, v):
    ep = {k: t.detach().clone().requires_grad_(True) for k, t in ep0.items()}
    loss, info = L.ffb6d_loss(ep, item, valid=v)
    loss.backward()
    return [info[k] for k in KEYS] + [t.grad for t in ep.values()]


def test_repeated_runs_are_bitwise_identical(cuda):
    a = training_batch(cuda, 8, 2, 8, 12288, seed=1)
    ep = {k: dev(a[k], cuda) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    item = {k: dev(a[k], cuda) for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst")}
    v = dev(np.array(MASKS["mixed"], bool), cuda)
    first = _run(ep, item, v)
    for _ in range(3):
        for x, y in zip(first, _run(ep, item, v)):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_graph_capture_and_replay(cuda):
    """The loss, its backward and info in one CUDA graph; replays on new inputs equal eager runs bitwise."""
    B, C, K, N = 8, 22, 8, 12288
    a = training_batch(cuda, B, C, K, N, seed=2)
    ep = {k: dev(a[k], cuda, True) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    item = {k: dev(a[k], cuda) for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst")}
    v = dev(np.array(MASKS["mixed"], bool), cuda)

    def step():
        for t in ep.values():
            t.grad = None
        loss, info = L.ffb6d_loss(ep, item, valid=v)
        loss.backward()
        return [info[k] for k in KEYS] + [t.grad for t in ep.values()]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    for seed in (2, 3):
        b = training_batch(cuda, B, C, K, N, seed=seed)
        with torch.no_grad():
            for k in ep:
                ep[k].copy_(torch.from_numpy(b[k]))
            for k in item:
                item[k].copy_(torch.from_numpy(b[k]))
        graph.replay()
        torch.cuda.synchronize()
        want = _run(ep, item, v)
        for x, y in zip(outs, want):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_deterministic_mode_runs_without_warnings(cuda):
    a = training_batch(cuda, 2, 22, 8, 2048, seed=4)
    ep = {k: dev(a[k], cuda) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    item = {k: dev(a[k], cuda) for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst")}
    eager = _run(ep, item, None)
    torch.use_deterministic_algorithms(True)
    try:
        det = _run(ep, item, None)
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y in zip(eager, det):
        assert torch.equal(x, y)


# --------------------------------------------------------------------------- item -> network -> loss
@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_item_network_loss_backward(cuda, dataset):
    """build_ffb6d_item on synthetic frames (one below 400 valid pixels) -> FFB6DFusionNet in training mode ->
    ffb6d_loss(valid=item["valid"]) -> backward.  The loss and the gradients reaching end_points equal the
    reference's loss evaluated on the valid sub-batch of the same end_points."""
    import ffb6d_b200 as F
    from ffb6d_b200.model import FFB6DFusionNet
    from ffb6d_b200.synthetic import INTRINSICS
    from test_gpu_item import _item_inputs, _seeded_batch
    n_classes = 22 if dataset == "ycb" else 2
    frames, objs, _ = _seeded_batch(3, 480, 640, 12288, 8, 41, dataset=dataset)
    raw = frames[1]["raw"]
    if dataset == "ycb":
        raw[:] = 0                      # fill_missing would complete a sparse frame: no depth at all
    else:
        keep = np.random.RandomState(1).choice(np.flatnonzero(raw), 300, replace=False)
        sparse = np.zeros_like(raw).reshape(-1)
        sparse[keep] = raw.reshape(-1)[keep]
        frames[1]["raw"] = sparse.reshape(raw.shape)
    x = _item_inputs(frames, objs, cuda)
    K = INTRINSICS["ycb_K1" if dataset == "ycb" else "linemod"]
    item = F.build_ffb6d_item(x["dpt"], 10000.0 if dataset == "ycb" else 1000.0, K, x["rgb"], x["labels"],
                              x["nrm_map"], objs, 12288, fill=dataset == "ycb")
    assert item["valid"].tolist() == [True, False, True]
    torch.manual_seed(0)
    net = FFB6DFusionNet(n_classes=n_classes).to(cuda).train()
    g = torch.Generator(device=cuda).manual_seed(0)
    feats = [torch.randn(s, generator=g, device=cuda) for s in FFB6DFusionNet.rgb_feature_shapes(3)]
    end_points = net(item, rgb_feats=feats)
    for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs"):
        end_points[k].retain_grad()
    loss, info = L.ffb6d_loss(end_points, item, valid=item["valid"])
    loss.backward()
    ep_ref = {k: end_points[k].detach().clone().requires_grad_(True)
              for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    ref_loss, ref_info = O.ffb6d_loss_torch(ep_ref, item, valid=item["valid"])
    ref_loss.backward()
    for k in KEYS:
        assert rel(info[k].item(), ref_info[k].item()) <= 1e-5, k
    for k in ("pred_kp_ofs", "pred_ctr_ofs"):
        assert torch.equal(end_points[k].grad, ep_ref[k].grad), k
    assert (end_points["pred_rgbd_segs"].grad - ep_ref["pred_rgbd_segs"].grad).abs().max().item() <= 1e-6
    for k in ep_ref:
        assert not end_points[k].grad[1].any()
    assert all(p.grad is None or torch.isfinite(p.grad).all() for p in net.parameters())
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in net.parameters())
