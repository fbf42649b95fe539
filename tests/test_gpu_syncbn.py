"""GPU: BatchNorm synchronised over ranks (a model converted with nn.SyncBatchNorm.convert_sync_batchnorm).

* The kernels, one process: a [B, C, P] batch split into three "virtual ranks" of 1, 2 and 3 frames, each running
  ffb6d_bn_sync_moments / _fwd / _bwd_sums / _bwd on its shard with the rows of all three stacked in rank order,
  against float64 BatchNorm and its autograd over the whole batch, at the shapes, activations, eps / momentum pairs
  and distributions of test_gpu_train.py::test_bn_train_vs_float64 and within its bounds.
* The modules, two processes over gloo on one GPU: a stack of converted layers (and forward_interp), and
  FFB6DFusionNet in both fusion orders, each rank holding half the batch, against one process holding the whole batch
  in float64.  Per-rank statistics miss these bounds by orders of magnitude.
* Two ranks over NCCL under DDP, when two GPUs are visible.
* A converted model without a process group is bitwise the unconverted one."""
import datetime
import os
import sys
import traceback

import pytest
import torch
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F_

from ffb6d_b200 import modules as M
from ffb6d_b200._lib import lib, check
from ffb6d_b200.ops import _stream
from conftest import ROOT
from test_gpu_train import BN_DISTS, BN_SHAPES, act_fn, away_from_kink, close_elementwise, close_fp32

pytestmark = pytest.mark.gpu

SHARDS = (1, 2, 3)          # frames per virtual rank


# ------------------------------------------------------------------ the kernels, virtual ranks in one process
@pytest.mark.parametrize("dist", BN_DISTS)
@pytest.mark.parametrize("eps,momentum", [(1e-5, 0.1), (1e-6, 0.99)], ids=["fusion", "randla"])
@pytest.mark.parametrize("act,slope", [(0, 0.0), (1, 0.0), (2, 0.2)], ids=["none", "relu", "leaky"])
@pytest.mark.parametrize("C,P", [(C, P) for _, C, P in BN_SHAPES])
def test_bn_sync_vs_float64(cuda, C, P, act, slope, eps, momentum, dist):
    B = sum(SHARDS)
    W = len(SHARDS)
    g = torch.Generator(device=cuda).manual_seed(C * 104729 + P + 31 * act + 1000 * BN_DISTS.index(dist))
    z = torch.randn(B, C, P, generator=g, device=cuda)
    if dist.startswith("offset"):
        std = torch.exp(torch.rand(C, generator=g, device=cuda) * 2 - 1)
        sign = torch.where(torch.rand(C, generator=g, device=cuda) < 0.5, -1.0, 1.0)
        z = z * std[:, None] + (sign * float(dist[6:]) * std)[:, None]
    cc = C - 1 if dist == "const" else None
    if cc is not None:
        z[:, cc] = 0.3
    gamma = 1 + 0.5 * torch.randn(C, generator=g, device=cuda)
    beta = 0.5 * torch.randn(C, generator=g, device=cuda)
    rm0 = torch.randn(C, generator=g, device=cuda)
    rv0 = torch.rand(C, generator=g, device=cuda) + 0.5
    gy = torch.randn(B, C, P, generator=g, device=cuda)
    f = act_fn(act, slope)

    z64 = z.double().requires_grad_(True)
    gam64, bet64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm64, rv64 = rm0.double(), rv0.double()
    pre64 = F_.batch_norm(z64, rm64, rv64, gam64, bet64, True, momentum, eps)
    y64 = f(pre64)
    gy = away_from_kink(gy, pre64, act)
    del pre64
    gz64, gg64, gb64 = torch.autograd.grad(y64, (z64, gam64, bet64), gy.double())
    y64 = y64.detach()
    with torch.no_grad():
        mean64 = z64.mean(dim=(0, 2))
        var64 = z64.var(dim=(0, 2), unbiased=False)
    del z64

    nbytes = int(lib.ffb6d_bn_workspace_bytes(C, P))
    st = _stream(cuda)
    lo = [sum(SHARDS[:r]) for r in range(W)]
    shard = [z[lo[r]:lo[r] + SHARDS[r]].contiguous() for r in range(W)]
    gshard = [gy[lo[r]:lo[r] + SHARDS[r]].contiguous() for r in range(W)]
    ws = [torch.empty(nbytes, dtype=torch.uint8, device=cuda) for _ in range(W)]
    rows = torch.empty(W, 2 * C + 1, dtype=torch.float64, device=cuda)
    for r in range(W):
        check(lib.ffb6d_bn_sync_moments(shard[r].data_ptr(), SHARDS[r], C, P, rows[r].data_ptr(), ws[r].data_ptr(), nbytes, st))
    stats = [torch.empty(C, 4, device=cuda) for _ in range(W)]
    count = [torch.empty(1, dtype=torch.float64, device=cuda) for _ in range(W)]
    rms, rvs = [rm0.clone() for _ in range(W)], [rv0.clone() for _ in range(W)]
    ys = [torch.empty_like(s) for s in shard]
    for r in range(W):
        check(lib.ffb6d_bn_sync_fwd(shard[r].data_ptr(), SHARDS[r], C, P, rows.data_ptr(), W, gamma.data_ptr(),
                                    beta.data_ptr(), eps, momentum, rms[r].data_ptr(), rvs[r].data_ptr(), act, slope,
                                    stats[r].data_ptr(), count[r].data_ptr(), ys[r].data_ptr(), st))
    brows = torch.empty(W, 2 * C, dtype=torch.float64, device=cuda)
    ggam = [torch.empty(C, device=cuda) for _ in range(W)]
    gbet = [torch.empty(C, device=cuda) for _ in range(W)]
    for r in range(W):
        check(lib.ffb6d_bn_sync_bwd_sums(shard[r].data_ptr(), gshard[r].data_ptr(), stats[r].data_ptr(), SHARDS[r], C, P,
                                         act, slope, brows[r].data_ptr(), ggam[r].data_ptr(), gbet[r].data_ptr(),
                                         ws[r].data_ptr(), nbytes, st))
    dzs = [torch.empty_like(s) for s in shard]
    for r in range(W):
        check(lib.ffb6d_bn_sync_bwd(shard[r].data_ptr(), gshard[r].data_ptr(), stats[r].data_ptr(), SHARDS[r], C, P,
                                    brows.data_ptr(), W, count[r].data_ptr(), act, slope, dzs[r].data_ptr(),
                                    ws[r].data_ptr(), nbytes, st))
    y, dz = torch.cat(ys), torch.cat(dzs)
    gg = sum(t.double() for t in ggam)
    gb = sum(t.double() for t in gbet)

    z32 = z.clone().requires_grad_(True)
    gam32, bet32 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    y32 = f(F_.batch_norm(z32, rm0.clone(), rv0.clone(), gam32, bet32, True, momentum, eps))
    gz32, gg32, gb32 = torch.autograd.grad(y32, (z32, gam32, bet32), gy)
    del z32

    what = "bn_sync %s over %s act=%d eps=%g %s" % ((B, C, P), SHARDS, act, eps, dist)
    for r in range(1, W):     # every rank combined the same rows in the same order
        assert torch.equal(stats[r], stats[0]) and torch.equal(rms[r], rms[0]) and torch.equal(rvs[r], rvs[0]), what
        assert torch.equal(count[r], count[0]), what
    assert count[0].item() == B * P, what
    stats, rm, rv = stats[0], rms[0], rvs[0]
    rest = slice(0, C if cc is None else cc)
    std64 = (var64 + eps).sqrt()
    dxhat = (2.0 ** -24 * mean64.abs() / std64)[rest]
    why = "2x what the fp32 mean's rounding moves it by"
    floor_y = 2 * (gamma.double()[rest].abs() * dxhat).max().item() if dxhat.numel() else 0.0
    floor_dz = 2 * (gamma.double()[rest].abs() / std64[rest] * dxhat * gg64[rest].abs() / (B * P)).max().item() if dxhat.numel() else 0.0
    floor_gg = 2 * (dxhat * gb64[rest].abs()).max().item() if dxhat.numel() else 0.0
    close_fp32(y[:, rest], y64[:, rest], y32[:, rest], what + " y", inherent=floor_y, why=why)
    close_elementwise(stats[:, 0], mean64, 1e-5 * std64 + 2.0 ** -24 * mean64.abs(), what + " stats mean")
    close_elementwise(stats[:, 1], 1 / std64, 1e-5 / std64, what + " stats invstd")
    close_elementwise(stats[:, 2], gamma.double() / std64, 1e-5 * (gamma.double() / std64).abs(), what + " stats gamma*invstd")
    assert torch.equal(stats[:, 3], beta), what + " stats beta"
    m = momentum
    close_elementwise(rm, rm64, 1e-5 * ((1 - m) * rm0.double().abs() + m * (mean64.abs() + std64)), what + " running_mean")
    close_elementwise(rv, rv64, 1e-5 * rv64.abs(), what + " running_var")
    close_fp32(dz[:, rest], gz64[:, rest], gz32[:, rest], what + " dz", inherent=floor_dz, why=why)
    close_fp32(gg, gg64, gg32, what + " grad_gamma", inherent=floor_gg, why=why)
    close_fp32(gb, gb64, gb32, what + " grad_beta")
    if cc is not None:
        # sigma^2 = 0 exactly: invstd is 1/sqrt(eps) rounded once, xhat = 0 and y = act(beta) bit for bit
        assert stats[cc, 0].item() == z[0, cc, 0].item(), what + " constant channel mean"
        want = torch.tensor(1.0 / float(torch.tensor(eps, dtype=torch.float32).double().sqrt()), dtype=torch.float32)
        assert stats[cc, 1].item() == want.item(), what + " constant channel invstd"
        assert torch.equal(y[:, cc], f(beta[cc].expand(B, P))), what + " constant channel y"
        close_fp32(dz[:, cc], gz64[:, cc], gz32[:, cc], what + " constant channel dz")


# ------------------------------------------------------------------ the modules over a process group
STACK_B, STACK_N, STACK_K, STACK_NA = 4, 256, 8, 100


def _stack_inputs(device):
    """The whole batch of the layer stack: x [4, 16, 256, 8], point features p [4, 24, 100, 1], the interpolation
    index [4, 2048, 1], the upstream gradient; frames 2 and 3 are offset from 0 and 1 (different statistics)."""
    g = torch.Generator(device=device).manual_seed(5)
    x = torch.randn(STACK_B, 16, STACK_N, STACK_K, generator=g, device=device)
    x[2:] = 0.7 * x[2:] + 0.4
    p = torch.randn(STACK_B, 24, STACK_NA, 1, generator=g, device=device)
    idx = torch.randint(0, STACK_NA, (STACK_B, STACK_N * STACK_K, 1), generator=g, device=device, dtype=torch.int32)
    go = torch.randn(STACK_B, 20, STACK_N * STACK_K, generator=g, device=device)
    return x, p, idx, go


def _stack_layers():
    torch.manual_seed(11)
    layers = nn.ModuleDict({"l1": M.RandLAConv2d(16, 32, bn=True), "l2": M.Conv2d(32, 48, bn=True),
                            "l3": M.Conv2d(48 + 24, 40, bn=True), "l4": M.Conv1d(40, 20, bn=True, activation=None)})
    g = torch.Generator().manual_seed(12)
    with torch.no_grad():
        for m in layers.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
    return layers


def _stack_forward(layers, x, p, idx):
    a = layers["l1"](x)
    b = layers["l2"](a).reshape(x.shape[0], 48, 64, 32)
    c = layers["l3"].forward_interp(b, p, idx)
    return layers["l4"](c.reshape(x.shape[0], 40, -1))


BN_OF = {"l1": ("bn", 1e-6, 0.99, "leaky"), "l2": ("normlayer", 1e-5, 0.1, "relu"), "l3": ("normlayer", 1e-5, 0.1, "relu"),
         "l4": ("normlayer", 1e-5, 0.1, None)}


def _twin_forward(sd, x, p, idx, bn):
    """The stack in torch ops; ``bn(name, t)`` is the layer's BatchNorm module (an nn.SyncBatchNorm)."""
    def layer(name, t):
        w = sd[name + ".conv.weight"]
        t = torch.einsum("oc,bc...->bo...", w.reshape(w.shape[0], -1), t)
        act = BN_OF[name][3]
        t = bn(name, t)
        return torch.relu(t) if act == "relu" else F_.leaky_relu(t, 0.2) if act == "leaky" else t

    B = x.shape[0]
    b = layer("l2", layer("l1", x)).reshape(B, 48, 64, 32)
    pi = torch.gather(p.squeeze(3), 2, idx.reshape(B, 1, -1).expand(-1, p.shape[1], -1).long()).reshape(B, -1, 64, 32)
    c = layer("l3", torch.cat((b, pi), 1))
    return layer("l4", c.reshape(B, 40, -1))


def _stack_results(layers, x, p, idx, go):
    x, p = x.clone().requires_grad_(True), p.clone().requires_grad_(True)
    out = _stack_forward(layers, x, p, idx)
    (out * go).sum().backward()
    res = {"out": out.detach(), "dx": x.grad, "dp": p.grad}
    for k, v in layers.named_parameters():
        res["grad." + k] = v.grad.clone()
    for k, v in layers.state_dict().items():
        if "running" in k:
            res[k] = v.clone()
    return res


def _twin_results(sd, x, p, idx, go, bn_mods, dtype):
    prm = {k: v.detach().to(dtype).requires_grad_("running" not in k) for k, v in sd.items() if v.dtype.is_floating_point}
    x, p = x.detach().to(dtype).requires_grad_(True), p.detach().to(dtype).requires_grad_(True)

    out = _twin_forward(prm, x, p, idx, lambda name, t: bn_mods[name](t))
    (out * go.to(dtype)).sum().backward()
    res = {"out": out.detach(), "dx": x.grad, "dp": p.grad}
    for name, m in bn_mods.items():
        pre = name + "." + BN_OF[name][0] + ".bn."
        res["grad." + pre + "weight"] = m.weight.grad
        res["grad." + pre + "bias"] = m.bias.grad
        res[pre + "running_mean"] = m.running_mean.detach().clone()
        res[pre + "running_var"] = m.running_var.detach().clone()
    for k, v in prm.items():
        if k.endswith("conv.weight"):
            res["grad." + k] = v.grad
    return res


def _twin_bns(sd, cls, dtype, device):
    mods = {}
    for name, (bn_name, eps, mom, _) in BN_OF.items():
        pre = name + "." + bn_name + ".bn."
        C = sd[pre + "weight"].shape[0]
        m = cls(C, eps=eps, momentum=mom).to(device=device, dtype=dtype).train()
        m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
        mods[name] = m
    return mods


def _fusion_setup(device, restructured):
    from ffb6d_b200.model import FFB6DFusionNet
    from ffb6d_b200.schedule import build_ffb6d_indices
    from ffb6d_b200.synthetic import make_batch
    h, w, n_pts, n_kps = 120, 160, 4096, 8
    torch.manual_seed(3)
    model = FFB6DFusionNet(n_classes=5, n_pts=n_pts, n_kps=n_kps, restructured=restructured).to(device)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
    batch = make_batch([3, 4], n_points=n_pts, h=h, w=w)
    cld = torch.from_numpy(batch["cld"]).to(device)
    xyz = torch.from_numpy(batch["dpt_xyz"]).to(device)
    inputs = build_ffb6d_indices(cld, xyz)
    inputs["choose"] = torch.from_numpy(batch["choose"]).to(device)
    inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(device)
    gg = torch.Generator(device=device).manual_seed(1)
    rgb = [torch.randn(s, generator=gg, device=device) for s in FFB6DFusionNet.rgb_feature_shapes(2, h, w)]
    return model, inputs, rgb, gg, n_kps


def _flat(d):
    return [d[k] for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")] + list(d["fused_rgb"])


def _fusion_results(model, inputs, rgb, go, frames):
    """One training step of ``model`` on ``frames`` (a slice of the two-frame batch)."""
    inp = {k: v[frames] for k, v in inputs.items()}
    feats = [t[frames].clone().requires_grad_(True) for t in rgb]
    out = _flat(model(inp, feats))
    sum((v * g_[frames]).sum() for v, g_ in zip(out, go)).backward()
    res = {"out%d" % i: v.detach() for i, v in enumerate(out)}
    res.update({"drgb%d" % i: t.grad for i, t in enumerate(feats)})
    res.update({"grad." + k: v.grad.clone() for k, v in model.named_parameters()})
    res.update({k: v.clone() for k, v in model.state_dict().items() if "running" in k})
    return res


def _worker(rank, world, backend, init_file, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    # the layers' weight gradients and gathers add with atomics otherwise: two runs must be bit-identical
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        dev = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(dev)
        kw = {"device_id": dev} if backend == "nccl" else {}
        dist.init_process_group(backend, init_method="file://" + init_file, rank=rank, world_size=world,
                                timeout=datetime.timedelta(seconds=120), **kw)
        half = slice(rank * STACK_B // world, (rank + 1) * STACK_B // world)
        res = {}
        if backend == "gloo":
            # the layer stack: ours converted, and torch's fp32 twin with nn.SyncBatchNorm over the same group
            x, p, idx, go = _stack_inputs(dev)
            layers = _stack_layers().to(dev)
            sd = {k: v.clone() for k, v in layers.state_dict().items()}
            layers = nn.SyncBatchNorm.convert_sync_batchnorm(layers).train()
            res["stack"] = _stack_results(layers, x[half], p[half], idx[half], go[half])
            res["stack_twin"] = _twin_results(sd, x[half], p[half], idx[half], go[half],
                                              _twin_bns(sd, nn.SyncBatchNorm, torch.float32, dev), torch.float32)
        for restructured in (False, True):
            model, inputs, rgb, gg, _ = _fusion_setup(dev, restructured)
            sd = {k: v.clone() for k, v in model.state_dict().items()}
            go = [torch.randn(s.shape, generator=gg, device=dev) for s in _flat_shapes(model, inputs, rgb)]
            model = nn.SyncBatchNorm.convert_sync_batchnorm(model).train()
            net = model
            if backend == "nccl":
                net = nn.parallel.DistributedDataParallel(model, device_ids=[dev.index])
            frames = slice(rank, rank + 1)
            runs = []
            for _ in range(2):        # two runs from the same state: bit-identical
                model.load_state_dict(sd)
                for q in model.parameters():
                    q.grad = None
                runs.append(_fusion_results(net, inputs, rgb, go, frames))
            res["fusion%d" % restructured] = runs
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()
        torch.save({k: _cpu(v) for k, v in res.items()}, os.path.join(out_dir, "rank%d.pt" % rank))
    except BaseException:
        with open(os.path.join(out_dir, "rank%d.err" % rank), "w") as fh:
            fh.write(traceback.format_exc())
        raise


def _flat_shapes(model, inputs, rgb):
    """The output shapes of the two-frame batch (an eval pass without autograd: statistics untouched)."""
    model.eval()
    with torch.no_grad():
        shapes = [v for v in _flat(model(inputs, rgb))]
    model.train()
    return shapes


def _cpu(v):
    if isinstance(v, torch.Tensor):
        return v.detach().cpu()
    if isinstance(v, dict):
        return {k: _cpu(t) for k, t in v.items()}
    if isinstance(v, list):
        return [_cpu(t) for t in v]
    return v


def _spawn(world, backend, tmp_path):
    ctx = mp.get_context("spawn")
    init_file = str(tmp_path / "pg_init")
    procs = [ctx.Process(target=_worker, args=(r, world, backend, init_file, str(tmp_path))) for r in range(world)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=900)
        errs = [open(tmp_path / ("rank%d.err" % r)).read() for r in range(world) if (tmp_path / ("rank%d.err" % r)).exists()]
        assert not errs, "\n".join(errs)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    return [torch.load(tmp_path / ("rank%d.pt" % r)) for r in range(world)]


def _check_fusion(res, cuda):
    """The whole network: rank-summed parameter gradients and per-rank input gradients against float64 TorchRef on
    the two-frame batch in one process, within test_gpu_model.py's bound (max(4x torch fp32, 2e-3)); two runs and both
    ranks' running statistics bit-identical."""
    from test_gpu_model import TorchRef
    for restructured in (False, True):
        runs = [r["fusion%d" % restructured] for r in res]
        what = "fusion restructured=%s" % restructured
        for rk in runs:
            a, b = rk
            for k in a:
                assert torch.equal(a[k], b[k]), "%s: run to run %s" % (what, k)
        for k in runs[0][0]:
            if "running" in k:
                assert torch.equal(runs[0][0][k], runs[1][0][k]), "%s: ranks differ in %s" % (what, k)
        model, inputs, rgb, gg, n_kps = _fusion_setup(cuda, restructured)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        go = [torch.randn(s.shape, generator=gg, device=cuda) for s in _flat_shapes(model, inputs, rgb)]
        got = [r[0] for r in runs]
        want_out = {}
        grads = {}
        for dtype in (torch.float64, torch.float32):
            ref = TorchRef(sd, True, n_kps, dtype=dtype)
            feats = [t.detach().to(dtype).requires_grad_(True) for t in rgb]
            out = _flat(ref.forward(inputs, feats))
            sum((v * g_.to(dtype)).sum() for v, g_ in zip(out, go)).backward()
            want_out[dtype] = [v.detach() for v in out]
            grads[dtype] = ({k: v.grad for k, v in ref.p.items() if v.grad is not None}, [t.grad for t in feats])
        for i, w in enumerate(want_out[torch.float64]):
            mine = torch.cat([g_["out%d" % i] for g_ in got]).to(cuda).double()
            err = (mine - w).abs().max().item()
            assert err <= 5e-5 * max(w.abs().max().item(), 1e-6), "%s out%d: %.3e" % (what, i, err)

        def unit(name):
            return name.rsplit(".conv.", 1)[0].rsplit(".normlayer.", 1)[0].rsplit(".bn.bn.", 1)[0].rsplit(".fc.", 1)[0]

        p64, p32 = grads[torch.float64][0], grads[torch.float32][0]
        scale_of = {}
        for name in p64:
            scale_of[unit(name)] = max(scale_of.get(unit(name), 1e-12), p64[name].norm().item())
        for name in p64:
            mine = sum(g_["grad." + name].double() for g_ in got).to(cuda)
            nrm = scale_of[unit(name)]
            e_ours = (mine - p64[name]).norm().item() / nrm
            e_t32 = (p32[name].double() - p64[name]).norm().item() / nrm
            assert e_ours <= max(4 * e_t32, 2e-3), "%s grad %s: %.3e (torch fp32 %.3e)" % (what, name, e_ours, e_t32)
        for i, (r64, r32) in enumerate(zip(grads[torch.float64][1], grads[torch.float32][1])):
            if r64 is None:
                continue
            mine = torch.cat([g_["drgb%d" % i] for g_ in got]).to(cuda).double()
            nrm = max(r64.norm().item(), 1e-12)
            e_ours = (mine - r64).norm().item() / nrm
            e_t32 = (r32.double() - r64).norm().item() / nrm
            assert e_ours <= max(4 * e_t32, 2e-3), "%s rgb grad %d: %.3e (torch fp32 %.3e)" % (what, i, e_ours, e_t32)


def test_two_ranks_gloo_one_gpu(cuda, tmp_path):
    res = _spawn(2, "gloo", tmp_path)
    # the layer stack against float64 on the whole batch; bound: 4x the error of torch's fp32 SyncBatchNorm twin
    x, p, idx, go = _stack_inputs(cuda)
    sd = {k: v.clone() for k, v in _stack_layers().to(cuda).state_dict().items()}
    # without a process group nn.SyncBatchNorm is plain training-mode BatchNorm (of any rank of input)
    want = _twin_results(sd, x, p, idx, go, _twin_bns(sd, nn.SyncBatchNorm, torch.float64, cuda), torch.float64)
    ours = [r["stack"] for r in res]
    twin = [r["stack_twin"] for r in res]
    for k in want:
        if k in ("out", "dx", "dp"):        # per rank: the halves of the batch
            got = torch.cat([o[k] for o in ours]).to(cuda)
            ref32 = torch.cat([t[k] for t in twin]).to(cuda)
        elif k.startswith("grad."):         # each rank's share of a parameter's gradient, added
            got = sum(o[k].double() for o in ours).to(cuda)
            ref32 = sum(t[k].double() for t in twin).to(cuda)
        else:                               # running statistics: every rank holds all of them, bit-identical
            assert torch.equal(ours[0][k], ours[1][k]), k
            got, ref32 = ours[0][k].to(cuda), twin[0][k].to(cuda)
        close_fp32(got.reshape(want[k].shape), want[k], ref32.reshape(want[k].shape), "stack " + k)
    _check_fusion(res, cuda)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_nccl_ddp(cuda, tmp_path):
    res = _spawn(2, "nccl", tmp_path)
    # DDP averages the gradients over the ranks: each rank holds the total / 2, and the two add up to the total
    _check_fusion(res, cuda)


def test_converted_model_without_group_is_bitwise_unconverted(cuda):
    algo = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)     # atomics would differ from run to run
    try:
        _converted_without_group(cuda)
    finally:
        torch.use_deterministic_algorithms(algo)


def _converted_without_group(cuda):
    model, inputs, rgb, gg, _ = _fusion_setup(cuda, False)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    go = [torch.randn(s.shape, generator=gg, device=cuda) for s in _flat_shapes(model, inputs, rgb)]
    model.train()
    a = _fusion_results(model, inputs, rgb, go, slice(0, 2))
    model.load_state_dict(sd)
    for q in model.parameters():
        q.grad = None
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(model).train()
    assert any(isinstance(m, nn.SyncBatchNorm) for m in conv.modules())
    b = _fusion_results(conv, inputs, rgb, go, slice(0, 2))
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k
