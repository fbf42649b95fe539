"""GPU: training through the restructured pixel fusion (W . cat(rgb, p[idx]) = W1 . rgb + (W2 . p)[idx], SURVEY.md
§8f-3).  The segment sum -- the backward of the gathered addend -- against torch's index_add_ in float64, and its
determinism under repeated calls and CUDA-graph replay; Conv2d.forward_interp in its three modes against the
reference composition in float64; the whole FFB6DFusionNet(restructured=True) against the float64 restatement of
tests/test_gpu_model.py; and the activation memory the restructured path saves.  Inputs come from seeds."""
import copy
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F_

import test_gpu_model
from test_gpu_train import away_from_kink, close_fp32
from ffb6d_b200 import fusion, ops
from ffb6d_b200 import tables as T
from ffb6d_b200.model import FFB6DFusionNet
from ffb6d_b200.modules import Conv2d
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu

N_LEVEL = [T.set_size(("cld", i)) for i in range(5)]
# the seven p2r stages at 480x640: (name, index key, C_r, h, w, N')
STAGES = [("ds%d" % i, "p2r_ds_nei_idx%d" % i, T.DS_RGB_OC[i], 480 // T.RGB_DS_SR[i], 640 // T.RGB_DS_SR[i],
           N_LEVEL[i + 1]) for i in range(4)]
STAGES += [("up%d" % i, "p2r_up_nei_idx%d" % i, T.UP_RGB_OC[i], 480 // T.RGB_UP_SR[i], 640 // T.RGB_UP_SR[i],
            N_LEVEL[3 - i]) for i in range(3)]
STAGE_IDS = [s[0] for s in STAGES]

_indices = {}


def stage_indices(cuda, B=2):
    """The index tensors of ``B`` synthetic frames (10 % holes: every hole pixel maps to one point per stage)."""
    if B not in _indices:
        batch = make_batch(list(range(11, 11 + B)))
        _indices[B] = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(cuda),
                                          torch.from_numpy(batch["dpt_xyz"]).to(cuda))
    return _indices[B]


# ------------------------------------------------------------------ segment sum
def check_segment_sum(grad, idx, na, what):
    """ops.segment_sum against index_add_ in float64: per element within one fp32 ulp of the float64 sum, or
    2^-36 of the sum of |terms| where the terms cancel; segments no pixel maps to are exactly 0."""
    out = ops.segment_sum(grad, idx, na)
    B, C = grad.shape[0], grad.shape[1]
    g = grad.reshape(B, C, -1).double()
    ix = idx.reshape(B, -1).long()
    want = torch.zeros((B, C, na), dtype=torch.float64, device=grad.device)
    mag = torch.zeros_like(want)
    for b in range(B):
        want[b].index_add_(1, ix[b], g[b])
        mag[b].index_add_(1, ix[b], g[b].abs())
    w = want.cpu().numpy()
    ulp = np.spacing(np.abs(w).astype(np.float32)).astype(np.float64)
    bound = np.maximum(ulp, 2.0 ** -36 * mag.cpu().numpy())
    err = np.abs(out.double().cpu().numpy() - w)
    bad = err > bound
    assert not bad.any(), "%s: %d elements out of bound, worst err %.3e (bound %.3e)" % (
        what, int(bad.sum()), err[bad].max(), bound[bad][np.argmax(err[bad])])
    count = torch.zeros((B, na), dtype=torch.int64, device=grad.device)
    for b in range(B):
        count[b].index_add_(0, ix[b], torch.ones_like(ix[b]))
    empty = (count == 0).unsqueeze(1).expand(-1, C, -1)
    assert torch.equal(out[empty], torch.zeros_like(out[empty])), what + ": an empty segment is not 0.0"
    return out


@pytest.mark.parametrize("stage", STAGES, ids=STAGE_IDS)
def test_segment_sum_stage_shapes(cuda, stage):
    name, key, C, h, w, na = stage
    idx = stage_indices(cuda)[key]
    B = idx.shape[0]
    ix = idx.reshape(B, -1).long()
    # the hole pixels (depth 0, at the origin) all map to one point: the largest segment of the frame
    largest = max(int(torch.bincount(ix[b], minlength=na).max()) for b in range(B))
    assert largest > 256, "%s: no segment long enough to be split across warps (%d)" % (name, largest)
    g = torch.Generator(device=cuda).manual_seed(C * 31 + na)
    grad = torch.randn((B, C, h, w), generator=g, device=cuda)
    out = check_segment_sum(grad, idx, na, name)
    assert torch.equal(out, ops.segment_sum(grad, idx, na))


@pytest.mark.parametrize("case", ["all_one_segment", "unused_points", "na1", "p1", "ragged_i64_c1", "ragged_i64_c1024"])
def test_segment_sum_edge_cases(cuda, case):
    g = torch.Generator(device=cuda).manual_seed(len(case))
    B, C, P, na = {"all_one_segment": (2, 64, 76800, 768), "unused_points": (2, 40, 5000, 3000), "na1": (3, 5, 4099, 1),
                   "p1": (2, 33, 1, 7), "ragged_i64_c1": (3, 1, 7 * 13, 11), "ragged_i64_c1024": (3, 1024, 7 * 13, 11)}[case]
    if case == "all_one_segment":
        idx = torch.full((B, P, 1), 5, dtype=torch.int32, device=cuda)
    elif case == "unused_points":      # only the even points are hit
        idx = 2 * torch.randint(0, na // 2, (B, P), generator=g, device=cuda, dtype=torch.int32)
    else:
        idx = torch.randint(0, na, (B, P, 1), generator=g, device=cuda)
        if not case.startswith("ragged"):
            idx = idx.int()
    grad = torch.randn((B, C, P), generator=g, device=cuda)
    if case == "unused_points":        # cancelling sums: terms of both signs around a large offset
        grad = grad + 100.0 * torch.where(torch.rand((B, C, P), generator=g, device=cuda) < 0.5, -1.0, 1.0)
    if case.startswith("ragged"):
        grad = grad.reshape(B, C, 7, 13)
        assert idx.dtype == torch.int64
    check_segment_sum(grad, idx, na, case)


def test_segment_sum_bitwise_repeatable_and_graph_replay(cuda):
    idx = stage_indices(cuda)["p2r_up_nei_idx2"]            # 240x320 pixels onto 3072 points
    B, P = idx.shape[0], idx.shape[1]
    na = N_LEVEL[1]
    g = torch.Generator(device=cuda).manual_seed(5)
    grad = torch.randn((B, 64, P), generator=g, device=cuda)
    first = ops.segment_sum(grad, idx, na)
    plan = ops.segment_plan(idx, na)
    assert torch.equal(first, ops.segment_sum(grad, None, na, plan=plan))
    assert torch.equal(first, ops.segment_sum(grad, idx, na))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                          # warm up off the capture
        ops.segment_sum(grad, idx, na)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.segment_sum(grad, idx, na)               # plan and sum, both captured
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, first)


# ------------------------------------------------------------------ Conv2d.forward_interp
def make_layer(cuda, c_r, seed):
    torch.manual_seed(seed)
    layer = Conv2d(2 * c_r, c_r, kernel_size=(1, 1), bn=True).to(cuda)
    g = torch.Generator().manual_seed(seed)
    bn = layer.normlayer.bn
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c_r, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c_r, generator=g) * 0.1)
        bn.running_mean.copy_(torch.randn(c_r, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c_r, generator=g) + 0.5)
    return layer


def reference_composition(w, gamma, beta, rmean, rvar, x1, p, idx, train):
    """models/ffb6d.py:246-253 in torch ops: nearest_interpolation, cat, 1x1 conv, BatchNorm, ReLU.
    Returns (y, pre-activation)."""
    B, _, h, w_ = x1.shape
    up = torch.gather(p.squeeze(3), 2, idx.reshape(B, 1, -1).expand(-1, p.shape[1], -1).long()).view(B, -1, h, w_)
    z = torch.einsum("oc,bchw->bohw", w.reshape(w.shape[0], -1), torch.cat((x1, up), 1))
    pre = F_.batch_norm(z, rmean, rvar, gamma, beta, train, 0.1, 1e-5)
    return torch.relu(pre), pre


RAGGED = ("ragged", None, 48, 37, 53, 100)        # h * w = 1961, not a multiple of 128


def interp_inputs(cuda, stage):
    name, key, c_r, h, w, na = stage
    B = 2
    g = torch.Generator(device=cuda).manual_seed(c_r + h)
    if key is None:
        idx = torch.randint(0, na, (B, h * w, 1), generator=g, device=cuda, dtype=torch.int32)
    else:
        idx = stage_indices(cuda)[key]
    x1 = torch.randn((B, c_r, h, w), generator=g, device=cuda)
    p = torch.relu(torch.randn((B, c_r, na, 1), generator=g, device=cuda))
    return x1, p, idx


@pytest.mark.parametrize("mode", ["train", "eval_grad"])
@pytest.mark.parametrize("stage", STAGES + [RAGGED], ids=STAGE_IDS + ["ragged"])
def test_forward_interp_matches_reference_composition(cuda, stage, mode):
    """Train mode (batch statistics) and eval under autograd (frozen BatchNorm): y, the running statistics, dW
    (both halves), dgamma, dbeta, dx1 and dp against float64; 1e-5 of each tensor's scale or 4x torch fp32's error."""
    c_r = stage[2]
    train = mode == "train"
    layer = make_layer(cuda, c_r, seed=c_r)
    x1, p, idx = interp_inputs(cuda, stage)
    bn = layer.normlayer.bn
    refs = {}
    for dt in (torch.float64, torch.float32):
        leaves = [t.detach().to(dt).requires_grad_(True) for t in (layer.conv.weight, bn.weight, bn.bias, x1, p)]
        rm, rv = bn.running_mean.detach().to(dt).clone(), bn.running_var.detach().to(dt).clone()
        y, pre = reference_composition(leaves[0], leaves[1], leaves[2], rm, rv, leaves[3], leaves[4], idx, train)
        refs[dt] = (leaves, rm, rv, y, pre)
    layer.train(train)
    xg, pg = x1.clone().requires_grad_(True), p.clone().requires_grad_(True)
    y = layer.forward_interp(xg, pg, idx)
    gy = torch.randn(y.shape, generator=torch.Generator(device=cuda).manual_seed(2), device=cuda)
    gy = away_from_kink(gy, refs[torch.float64][4], 1)
    y.backward(gy)
    for dt in refs:
        refs[dt][3].backward(gy.to(dt))
    (l64, rm64, rv64, y64, _), (l32, rm32, rv32, y32, _) = refs[torch.float64], refs[torch.float32]
    what = "%s %s" % (stage[0], mode)
    close_fp32(y, y64, y32, what + " y")
    if train:
        close_fp32(bn.running_mean, rm64, rm32, what + " running_mean")
        close_fp32(bn.running_var, rv64, rv32, what + " running_var")
        assert int(bn.num_batches_tracked) == 1
    gw, gw64, gw32 = layer.conv.weight.grad.reshape(c_r, -1), l64[0].grad.reshape(c_r, -1), l32[0].grad.reshape(c_r, -1)
    close_fp32(gw[:, :c_r], gw64[:, :c_r], gw32[:, :c_r], what + " dW1")
    close_fp32(gw[:, c_r:], gw64[:, c_r:], gw32[:, c_r:], what + " dW2")
    close_fp32(bn.weight.grad, l64[1].grad, l32[1].grad, what + " dgamma")
    close_fp32(bn.bias.grad, l64[2].grad, l32[2].grad, what + " dbeta")
    close_fp32(xg.grad, l64[3].grad, l32[3].grad, what + " dx1")
    close_fp32(pg.grad, l64[4].grad, l32[4].grad, what + " dp")


@pytest.mark.parametrize("stage", [STAGES[3], STAGES[6], RAGGED], ids=["ds3", "up2", "ragged"])
def test_forward_interp_eval_is_the_restructured_stage(cuda, stage):
    """Eval without autograd: bitwise what fusion.FusionStage(restructured=True) computes with the same weights."""
    c_r, na = stage[2], stage[5]
    c_p = max(c_r // 2, 16)
    x1, _, idx = interp_inputs(cuda, stage)
    g = torch.Generator(device=cuda).manual_seed(7)
    p_emb0 = torch.randn((2, c_p, na, 1), generator=g, device=cuda)
    r2p_idx = torch.randint(0, x1.shape[2] * x1.shape[3], (2, na, 16), generator=g, device=cuda)
    torch.manual_seed(c_r)
    r2p_pre, r2p_fuse = Conv2d(c_r, c_p, bn=True).to(cuda).eval(), Conv2d(2 * c_p, c_p, bn=True).to(cuda).eval()
    p2r_pre, p2r_fuse = Conv2d(c_p, c_r, bn=True).to(cuda).eval(), make_layer(cuda, c_r, seed=3).eval()
    stage_ = fusion.FusionStage(*(fusion.FusedConv.from_module(m) for m in (r2p_pre, r2p_fuse, p2r_pre, p2r_fuse)))
    with torch.no_grad():
        want, _ = stage_(x1, p_emb0, idx, r2p_idx, restructured=True)
        got = p2r_fuse.forward_interp(x1, p2r_pre(p_emb0), idx)
        assert torch.equal(got, want)
        assert torch.equal(p2r_fuse.forward_interp(x1, p2r_pre(p_emb0), idx.long()), want)
        p2r_fuse.normlayer.bn.running_mean.add_(0.5)           # the cached split follows the BatchNorm statistics
        stage_ = fusion.FusionStage(*(fusion.FusedConv.from_module(m) for m in (r2p_pre, r2p_fuse, p2r_pre, p2r_fuse)))
        want2, _ = stage_(x1, p_emb0, idx, r2p_idx, restructured=True)
        assert torch.equal(p2r_fuse.forward_interp(x1, p2r_pre(p_emb0), idx), want2)
        assert not torch.equal(want2, want)


def test_forward_interp_rejects_bad_shapes(cuda):
    layer = make_layer(cuda, 16, seed=1).eval()
    x1 = torch.randn(2, 16, 4, 5, device=cuda)
    p = torch.randn(2, 16, 7, 1, device=cuda)
    idx = torch.zeros(2, 20, 1, dtype=torch.int32, device=cuda)
    with pytest.raises(ValueError, match="input channels"):
        layer.forward_interp(x1, p[:, :8], idx)
    with pytest.raises(ValueError, match="interp_idx"):
        layer.forward_interp(x1, p, idx[:, :19])
    with pytest.raises(ValueError, match="forward_interp expects"):
        layer.forward_interp(x1, p.squeeze(3), idx)
    with pytest.raises(RuntimeError, match="no CPU path"):
        layer.forward_interp(x1.cpu(), p, idx)


# ------------------------------------------------------------------ the whole network
class _Restructured(FFB6DFusionNet):
    def __init__(self, *args, **kw):
        super().__init__(*args, restructured=True, **kw)


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
def test_restructured_net_matches_torch_restatement(cuda, train, monkeypatch):
    """tests/test_gpu_model.py's comparison (outputs within 5e-5, every parameter gradient within max(4x torch
    fp32's error, 2e-3) of float64) with the model built restructured; every p2r fusion goes through
    forward_interp."""
    calls = []
    orig = Conv2d.forward_interp

    def spy(self, *args):
        calls.append(self.training)
        return orig(self, *args)

    monkeypatch.setattr(Conv2d, "forward_interp", spy)
    monkeypatch.setattr(test_gpu_model, "FFB6DFusionNet", _Restructured)
    test_gpu_model.test_fusion_net_matches_torch_restatement(cuda, train)
    assert calls == [train] * 7


def test_state_dicts_move_between_settings(cuda):
    torch.manual_seed(0)
    a = FFB6DFusionNet(restructured=True)
    b = FFB6DFusionNet(restructured=False)
    assert list(a.state_dict()) == list(b.state_dict())
    b.load_state_dict(a.state_dict(), strict=True)
    a.load_state_dict(b.state_dict(), strict=True)
    assert a.restructured and not b.restructured


def test_restructured_training_saves_the_interpolated_maps(cuda):
    """One training forward + backward at B = 2, 480x640: the seven interpolated maps (95.8 MB per frame, computed
    from the stage shapes) are no longer held for the backward, so the peak is at least 140 MB lower."""
    maps = sum(4 * c * h * w for _, _, c, h, w, _ in STAGES)
    assert abs(maps - 95.8e6) < 0.1e6
    B = 2
    inputs = dict(stage_indices(cuda, B))
    batch = make_batch(list(range(11, 11 + B)))
    inputs["choose"] = torch.from_numpy(batch["choose"]).to(cuda)
    inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(cuda)
    torch.manual_seed(0)
    model = FFB6DFusionNet().to(cuda).train()
    g = torch.Generator(device=cuda).manual_seed(0)
    feats = [torch.randn(s, generator=g, device=cuda).requires_grad_(True) for s in FFB6DFusionNet.rgb_feature_shapes(B)]
    peak = {}
    for restructured in (False, True, False, True):       # the second round is the one kept
        model.restructured = restructured
        model.zero_grad(set_to_none=True)
        for t in feats:
            t.grad = None
        gc.collect()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = model(inputs, feats)
        loss = sum(out[k].mean() for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")) + \
            sum(r.mean() for r in out["fused_rgb"])
        loss.backward()
        del out, loss
        torch.cuda.synchronize()
        peak[restructured] = torch.cuda.max_memory_allocated() - base
    saved = peak[False] - peak[True]
    assert saved >= 140e6, "peak %.1f MB (reference order) vs %.1f MB (restructured): %.1f MB saved" % (
        peak[False] / 1e6, peak[True] / 1e6, saved / 1e6)
