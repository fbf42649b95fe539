"""GPU: the attentive pooling of RandLA's Building_block on the fused training kernels (ops.lfa_train_fwd /
lfa_train_bwd, modules._LfaAttPool): against float64 autograd of the reference expression
    f_agg = sum_k x_k * softmax_k(W_fc . x_k),   x_k = cat(feature[:, idx[n, k]], f_xyz[:, n, k])
(models/RandLA/RandLANet.py:200-212, 243-248) at the shapes of FFB6D's encoder levels 0-2 and on edge cases; the
determinism of its backward; the routing of Building_block; and whole training steps of Dilated_res_block and
FFB6DFusionNet with ``fused_lfa`` off and on against their float64 restatement."""
import contextlib
import copy

import pytest
import torch

from ffb6d_b200 import modules, ops
from ffb6d_b200._lib import FFB6DError
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6DFusionNet
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_b200.synthetic import make_batch
from ffb6d_restatement import TorchRef, close, unit

pytestmark = pytest.mark.gpu

# (d/2, N) of encoder levels 0-2 at 12288 points (d_out = 32, 64, 128)
LEVELS = [(16, 12288), (32, 3072), (64, 768)]


@contextlib.contextmanager
def deterministic(on=True):
    saved = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(saved)


def neighbours(B, N, g, dev, dtype=torch.int32):
    """KNN-like rows: the point itself first, then random points, with the second half of every third row a copy of
    its first half (the duplicated neighbours of a wrap-padded frame)."""
    idx = torch.randint(0, N, (B, N, 16), generator=g, device=dev)
    idx[:, :, 0] = torch.arange(N, device=dev)
    idx[:, ::3, 8:] = idx[:, ::3, :8]
    return idx.to(dtype)


def inputs(B, Dh, N, seed, dev, logit=4.0, idx_dtype=torch.int32):
    g = torch.Generator(device=dev).manual_seed(seed)
    feature = torch.randn(B, Dh, N, 1, generator=g, device=dev)
    f_xyz = torch.randn(B, Dh, N, 16, generator=g, device=dev)
    w = torch.randn(2 * Dh, 2 * Dh, 1, 1, generator=g, device=dev) * (logit / (2 * Dh) ** 0.5 / 3.0)
    return feature, neighbours(B, N, g, dev, idx_dtype), f_xyz, w, torch.randn(B, 2 * Dh, N, 1, generator=g, device=dev)


def reference(feature, idx, f_xyz, w):
    """The reference expression with torch ops, in the dtype of its inputs."""
    B, Dh, N, _ = feature.shape
    K = idx.shape[2]
    gathered = torch.gather(feature.squeeze(3), 2, idx.long().reshape(B, 1, N * K).expand(-1, Dh, -1))
    x = torch.cat([gathered.reshape(B, Dh, N, K), f_xyz], 1)
    s = torch.softmax(torch.einsum("oc,bcnk->bonk", w.reshape(w.shape[0], -1), x), 3)
    return (x * s).sum(3, keepdim=True)


def run_reference(args, dtype):
    feature, idx, f_xyz, w, go = args
    leaves = [t.detach().to(dtype).requires_grad_(True) for t in (feature, f_xyz, w)]
    out = reference(leaves[0], idx, leaves[1], leaves[2])
    out.backward(go.to(dtype))
    return out.detach(), [t.grad for t in leaves]


def run_fused(args):
    feature, idx, f_xyz, w, go = args
    leaves = [t.detach().clone().requires_grad_(True) for t in (feature, f_xyz, w)]
    out = modules._LfaAttPool.apply(leaves[0], idx, leaves[1], leaves[2])
    out.backward(go)
    return out.detach(), [t.grad for t in leaves]


def check(got, want64, want32, what, rtol=2e-5, factor=4.0):
    """Element-wise: |got - want64| <= rtol * scale(want64) + factor * |torch fp32 - want64| (scale: the tensor's
    largest finite magnitude), NaN exactly where float64 has NaN."""
    nan = torch.isnan(want64)
    assert torch.equal(torch.isnan(got), nan), "%s: NaN at %d positions, float64 at %d" % (
        what, int(torch.isnan(got).sum()), int(nan.sum()))
    fin = ~nan
    g, w, w32 = got[fin].double(), want64[fin], want32[fin].double()
    if w.numel() == 0:
        return
    scale = max(w.abs().max().item(), 1e-6)
    tol = rtol * scale + factor * (w32 - w).abs()
    err = (g - w).abs()
    bad = err > tol
    assert not bad.any(), "%s: %d elements out of tolerance, worst err %.3e (tol %.3e) at scale %.3e" % (
        what, int(bad.sum()), err[bad].max().item(), tol[bad][int((err - tol)[bad].argmax())].item(), scale)


def compare(args, what, **kw):
    got, ggot = run_fused(args)
    want, gwant = run_reference(args, torch.float64)
    want32, gwant32 = run_reference(args, torch.float32)
    check(got, want, want32, what + " f_agg", **kw)
    for name, a, b, c in zip(("grad_feature", "grad_f_xyz", "grad_w_fc"), ggot, gwant, gwant32):
        check(a, b, c, "%s %s" % (what, name), **kw)


@pytest.mark.parametrize("Dh,N", LEVELS, ids=["level0", "level1", "level2"])
def test_encoder_levels_vs_float64(cuda, Dh, N):
    compare(inputs(8, Dh, N, 10 + Dh, cuda), "B=8 d/2=%d N=%d" % (Dh, N))


CASES = ["all_same_neighbour", "large_logits", "n_not_multiple", "batch_of_one", "int64_indices", "nan_feature"]


@pytest.mark.parametrize("Dh", [16, 32, 64])
@pytest.mark.parametrize("case", CASES)
def test_edge_cases_vs_float64(cuda, case, Dh):
    B, N = (1, 1000) if case == "batch_of_one" else (2, 997 if case == "n_not_multiple" else 512)
    args = list(inputs(B, Dh, N, 7 * Dh + CASES.index(case), cuda, logit=80.0 if case == "large_logits" else 4.0,
                       idx_dtype=torch.int64 if case == "int64_indices" else torch.int32))
    if case == "all_same_neighbour":        # every neighbour of every point the same point: 16 edges per row land there
        args[1] = torch.full_like(args[1], N // 3)
    if case == "nan_feature":
        args[0][0, 3, 17, 0] = float("nan")
    if case == "large_logits":
        want = run_reference(args, torch.float64)[0]
        assert torch.isfinite(want).all()
        logits = torch.einsum("oc,bcnk->bonk", args[3].reshape(2 * Dh, 2 * Dh).double(), torch.cat([
            torch.gather(args[0].squeeze(3), 2, args[1].long().reshape(B, 1, -1).expand(-1, Dh, -1)).reshape(
                B, Dh, N, 16), args[2]], 1).double())
        assert logits.abs().max().item() > 60.0, "the case must reach large logits"
    if case != "nan_feature":
        got, grads = run_fused(args)
        assert torch.isfinite(got).all() and all(torch.isfinite(t).all() for t in grads), case
    compare(args, "%s d/2=%d" % (case, Dh))


def test_unsupported_shapes_raise(cuda):
    f, idx, fx, w, _ = inputs(1, 16, 64, 1, cuda)
    with pytest.raises(FFB6DError, match="only K = 16"):
        ops.lfa_train_fwd(f, idx[..., :8], fx[..., :8], w)
    f, idx, fx, w, _ = inputs(1, 128, 64, 1, cuda)
    with pytest.raises(FFB6DError, match="fused for 16, 32, 64"):
        ops.lfa_train_fwd(f, idx, fx, w)
    f, idx, fx, w, _ = inputs(1, 8, 64, 1, cuda)
    with pytest.raises(FFB6DError, match="fused for 16, 32, 64"):
        ops.lfa_train_fwd(f, idx, fx, w)


@pytest.mark.parametrize("Dh,N", LEVELS, ids=["level0", "level1", "level2"])
def test_deterministic_backward_is_bitwise_reproducible(cuda, Dh, N):
    args = inputs(8, Dh, N, 30 + Dh, cuda)
    with deterministic():
        a, b = run_fused(args), run_fused(args)
    assert torch.equal(a[0], b[0])
    for name, x, y in zip(("grad_feature", "grad_f_xyz", "grad_w_fc"), a[1], b[1]):
        assert torch.equal(x, y), "%s differs between two deterministic runs" % name
    c = run_fused(args)      # default mode: the scatter of grad_feature adds with atomics, the rest is the same
    assert torch.equal(a[1][2], c[1][2]), "grad_w_fc differs between the deterministic and the default mode"
    assert torch.equal(a[1][1], c[1][1]), "grad_f_xyz differs between the deterministic and the default mode"
    torch.testing.assert_close(a[1][0], c[1][0], rtol=1e-5, atol=1e-5 * a[1][0].abs().max().item())


def count_fused(monkeypatch):
    calls = []
    real = ops.lfa_train_fwd

    def spy(*a, **kw):
        calls.append(a[0].shape[1])
        return real(*a, **kw)

    monkeypatch.setattr(ops, "lfa_train_fwd", spy)
    return calls


def block_inputs(B, d_in, N, K, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    xyz = torch.rand(B, N, 3, generator=g, device=dev)
    idx = torch.randint(0, N, (B, N, K), generator=g, device=dev, dtype=torch.int32)
    return torch.randn(B, d_in, N, 1, generator=g, device=dev), xyz, idx


@pytest.mark.parametrize("d_out,K,fused", [(32, 16, True), (64, 16, True), (128, 16, True), (256, 16, False),
                                           (32, 8, False), (32, 24, False)],
                         ids=["d32", "d64", "d128", "d256_per_op", "K8_per_op", "K24_per_op"])
def test_building_block_routing(cuda, monkeypatch, d_out, K, fused):
    calls = count_fused(monkeypatch)
    blk = modules.Dilated_res_block(16, d_out).to(cuda).train()
    feature, xyz, idx = block_inputs(2, 16, 256, K, cuda)
    blk(feature, xyz, idx).sum().backward()                     # flag off: never the fused kernels
    assert calls == []
    blk.lfa.fused_lfa = True
    blk(feature, xyz, idx).sum().backward()
    assert calls == ([d_out // 2] * 2 if fused else []), calls
    calls.clear()
    blk.lfa.fused_lfa = False
    blk(feature, xyz, idx, fused_lfa=True).sum().backward()     # the per-call override
    assert calls == ([d_out // 2] * 2 if fused else [])


def randomise_bn(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)


def grad_errors(named_grads, ref):
    """Per parameter: |grad - float64 grad| / the largest float64 gradient norm of its layer (tests/test_gpu_model.py)."""
    scale = {}
    for name in named_grads:
        scale[unit(name)] = max(scale.get(unit(name), 1e-12), ref.p[name].grad.norm().item())
    return {n: (g.double() - ref.p[n].grad).norm().item() / scale[unit(n)] for n, g in named_grads.items()}


def check_step_pair(off, on, ref, what, bound=2e-3, ref32=None):
    """``off`` / ``on``: (named grads, buffers); the fused path's gradients are no further from float64 than the
    per-op path's -- or, with ``ref32`` (the restatement in float32), than torch's own float32 -- (4x, or within
    ``bound`` of the layer's scale), and its running statistics agree with float64."""
    e_off, e_on = grad_errors(off[0], ref), grad_errors(on[0], ref)
    e_32 = {n: (ref32.p[n].grad.double() - ref.p[n].grad).norm().item() for n in e_on} if ref32 is not None else {}
    scale = {}
    for n in e_on:
        scale[unit(n)] = max(scale.get(unit(n), 1e-12), ref.p[n].grad.norm().item())
    for n in e_on:
        yard = max(e_off[n], e_32.get(n, 0.0) / scale[unit(n)])
        assert e_on[n] <= max(4 * yard, bound), "%s grad %s: fused %.3e of its layer's scale, per-op %.3e%s" % (
            what, n, e_on[n], e_off[n], ", torch fp32 %.3e" % (e_32[n] / scale[unit(n)]) if e_32 else "")
    for n, want in ref.after.items():
        for tag, bufs in (("per-op", off[1]), ("fused", on[1])):
            close(bufs[n], want, "%s %s running statistic %s" % (what, tag, n), 1e-5)


@pytest.mark.parametrize("d_in,d_out,N", [(8, 32, 4096), (64, 64, 1024), (128, 128, 256)],
                         ids=["level0", "level1", "level2"])
def test_dilated_res_block_step_off_and_on(cuda, d_in, d_out, N):
    torch.manual_seed(5)
    blk = modules.Dilated_res_block(d_in, d_out).to(cuda).train()
    randomise_bn(blk, 6)
    feature, xyz, _ = block_inputs(4, d_in, N, 16, cuda, seed=d_out)
    g = torch.Generator(device=cuda).manual_seed(8)
    idx = neighbours(4, N, g, cuda)
    sd = {"b." + k: v.clone() for k, v in blk.state_dict().items()}
    go = None
    results = {}
    for fused in (False, True):
        m = copy.deepcopy(blk)
        m.lfa.fused_lfa = fused
        f = feature.clone().requires_grad_(True)
        out = m(f, xyz, idx)
        if go is None:
            go = torch.randn(out.shape, generator=g, device=cuda)
        out.backward(go)
        grads = {"b." + n: p.grad for n, p in m.named_parameters()}
        grads["feature"] = f.grad
        results[fused] = (out.detach(), grads, {"b." + n: b for n, b in m.named_buffers()})
    ref = TorchRef(sd, True, 8)
    f64 = feature.double().requires_grad_(True)
    want = ref.block("b", f64, xyz.double(), idx)
    want.backward(go.double())
    ref.p["feature"] = f64
    e_out = {k: (results[k][0].double() - want).abs().max().item() for k in (False, True)}
    scale = want.abs().max().item()
    assert e_out[True] <= max(4 * e_out[False], 2e-5 * scale), (e_out, scale)
    check_step_pair(results[False][1:], results[True][1:], ref, "Dilated_res_block(%d, %d)" % (d_in, d_out))


def net_setup(cuda):
    B, h, w, n_pts, n_kps = 2, 120, 160, 4096, 8
    torch.manual_seed(3)
    model = FFB6DFusionNet(n_classes=5, n_pts=n_pts, n_kps=n_kps).cuda().train()
    randomise_bn(model, 9)
    batch = make_batch([3, 4], n_points=n_pts, h=h, w=w)
    inp = build_ffb6d_indices(torch.from_numpy(batch["cld"]).cuda(), torch.from_numpy(batch["dpt_xyz"]).cuda())
    inp["choose"] = torch.from_numpy(batch["choose"]).cuda()
    inp["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    rgb = [torch.randn(s, generator=g, device="cuda") for s in FFB6DFusionNet.rgb_feature_shapes(B, h, w)]
    item = {"labels": torch.randint(0, 5, (B, n_pts), generator=g, device="cuda", dtype=torch.int32),
            "kp_targ_ofst": torch.randn(B, n_pts, n_kps, 3, generator=g, device="cuda") * 0.05,
            "ctr_targ_ofst": torch.randn(B, n_pts, 3, generator=g, device="cuda") * 0.05}
    return model, inp, rgb, item


KEYS = ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")


def net_step(model, inp, rgb, item, fused):
    m = copy.deepcopy(model)
    m.fused_lfa = fused
    out = m(inp, rgb)
    for t in [out[k] for k in KEYS] + out["fused_rgb"]:
        t.retain_grad()
    loss = ffb6d_loss(out, item)[0]
    # the fused image maps feed the (absent) CNN stages: a small term keeps the layers that make them in the graph
    loss = loss + sum(r.mean() for r in out["fused_rgb"]) * 1e-3
    loss.backward()
    grads = {n: p.grad for n, p in m.named_parameters()}
    return out, loss.detach(), grads, {n: b for n, b in m.named_buffers()}


def test_fusion_net_step_off_and_on(cuda):
    model, inp, rgb, item = net_setup(cuda)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    off = net_step(model, inp, rgb, item, False)
    on = net_step(model, inp, rgb, item, True)
    assert not model.fused_lfa and model.state_dict().keys() == sd.keys()
    ref = TorchRef(sd, True, 8)
    want = ref.forward(inp, [t.double() for t in rgb])
    for k in KEYS:
        scale = want[k].abs().max().item()
        e = [(r[0][k].detach().double() - want[k]).abs().max().item() for r in (off, on)]
        assert e[1] <= max(4 * e[0], 5e-5 * scale), "%s: fused %.3e, per-op %.3e at scale %.3e" % (k, e[1], e[0], scale)
    # the loss of the float64 outputs, through the same loss kernels
    loss64 = ffb6d_loss({k: want[k].detach().float() for k in KEYS}, item)[0].double() + sum(
        r.detach().mean() for r in want["fused_rgb"]) * 1e-3
    for tag, r in (("per-op", off), ("fused", on)):
        assert abs(r[1].item() - loss64.item()) <= 1e-5 * abs(loss64.item()), (tag, r[1].item(), loss64.item())
    # float64 gradients of the same loss, linearised at the per-op step's output gradients
    pairs = [(want[k], off[0][k]) for k in KEYS] + list(zip(want["fused_rgb"], off[0]["fused_rgb"]))
    sum((w * o.grad.double()).sum() for w, o in pairs).backward()
    # and in float32 through torch: how far plain fp32 autograd of this 60-layer network lands from float64
    # (tests/test_gpu_model.py)
    ref32 = TorchRef(sd, True, 8, dtype=torch.float32)
    want32 = ref32.forward(inp, rgb)
    pairs = [(want32[k], off[0][k]) for k in KEYS] + list(zip(want32["fused_rgb"], off[0]["fused_rgb"]))
    sum((w * o.grad).sum() for w, o in pairs).backward()
    # Through ~60 layers of batch-statistics BatchNorm over as few as 32 positions and the max-pools of random_sample,
    # whose arg-max can flip under a reordered fp32 sum, round-off is amplified (tests/test_gpu_model.py), and the
    # atomics of the default backward make it vary from run to run.  Measured on an H100 in two runs: the encoder's
    # first layers (rndla_pre_stages.bn.bn.weight, rndla_ds_stages.0.mlp1.conv.weight) land 3.0e-3 and 8.9e-3 of
    # their layer's scale from float64 with the flag on, 6.7e-4 and 1.3e-3 with it off; the floor is 2e-2.
    check_step_pair(off[2:], on[2:], ref, "FFB6DFusionNet", bound=2e-2, ref32=ref32)


def test_fusion_net_step_on_under_deterministic_switch(cuda):
    model, inp, rgb, item = net_setup(cuda)
    on = net_step(model, inp, rgb, item, True)
    with deterministic():
        a = net_step(model, inp, rgb, item, True)
        b = net_step(model, inp, rgb, item, True)
    assert torch.equal(a[1], b[1])
    for n in a[2]:
        assert torch.equal(a[2][n], b[2][n]), "grad %s differs between two deterministic steps" % n
        torch.testing.assert_close(a[2][n], on[2][n], rtol=1e-3, atol=1e-3 * max(on[2][n].abs().max().item(), 1e-6))
