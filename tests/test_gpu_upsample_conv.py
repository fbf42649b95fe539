"""GPU: PSPUpsample at the input's resolution (``forward_restructured``, ``FFB6D(fused_upsample=True)``, DESIGN.md
§4.23) against float64 torch in the reference's order (``nn.Upsample -> nn.Conv2d -> nn.BatchNorm2d -> nn.PReLU``):
eval and training forwards at the three stages' shapes at B = 8 and at odd ones, the gradients of x, the weight, the
bias, gamma, beta and alpha, non-finite inputs, bitwise repeatability under ``torch.use_deterministic_algorithms(True)``
and through graph replays, a SyncBatchNorm-converted stage over two ranks, peak memory against the torch modules, and
the whole FFB6D with the flag on against it off and against its float64 restatement.

A result passes within 1e-5 of its scale of float64, or at most twice as far from it as the same composition on
torch's fp32 modules (cuDNN / cuBLAS TF32 off for this file), whichever is larger.  The second bound matters at up_3's
size: torch's float taps (scale = (float)(in - 1) / (out - 1)) are themselves about 2e-5 of scale from float64's
there, and the kernels read the same taps."""
import copy
import datetime
import os
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import ffb6d_b200 as F
from ffb6d_b200 import cnn, ops
from ffb6d_restatement import FullRef, close
from test_gpu_cnn import _network
from test_gpu_cnn_train import _item, _train_step, bound, deterministic
from test_gpu_graphed_step import assert_bitwise, eager_step, items, pair

pytestmark = pytest.mark.gpu
TOL = 1e-5
STAGES = [(8, 1024, 256, 60, 80), (8, 256, 64, 120, 160), (8, 64, 64, 240, 320)]          # up_1, up_2, up_3
ODD = [(1, 5, 3, 1, 1), (2, 7, 130, 3, 5), (1, 33, 200, 1, 6), (3, 40, 9, 7, 1), (1, 3, 2, 4, 3), (2, 1, 4, 2, 2)]
IDS = lambda s: "x".join(map(str, s))


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def make_up(Ci, Co, seed):
    torch.manual_seed(seed)
    m = cnn.PSPUpsample(Ci, Co).cuda()
    _, conv, bn, act = m.conv
    with torch.no_grad():
        conv.bias.normal_(0, 0.1)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.2)
        bn.running_mean.normal_(0, 0.1)
        bn.running_var.uniform_(0.5, 1.5)
        act.weight.fill_(0.1 + 0.05 * (seed % 5))
    return m


def rand(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda")


def params(m):
    _, conv, bn, act = m.conv
    return [("weight", conv.weight), ("bias", conv.bias), ("gamma", bn.weight), ("beta", bn.bias), ("alpha", act.weight)]


def within(got, want, what, tol=TOL):
    got, want = got.detach().double(), want.detach().double()
    scale = max(want.abs().max().item(), 1e-30)
    e = (got - want).abs().max().item()
    assert e <= tol * scale, "%s: %.2e of scale" % (what, e / scale)


# ------------------------------------------------------------------------------------------------ forwards
@pytest.mark.parametrize("shape", STAGES + ODD, ids=IDS)
def test_eval_forward(cuda, shape):
    B, Ci, Co, Hi, Wi = shape
    m = make_up(Ci, Co, 1).eval()
    x = rand((B, Ci, Hi, Wi), sum(shape))
    with torch.no_grad():
        got = m.forward_restructured(x)
        want = copy.deepcopy(m).double()(x.double())
        t32 = copy.deepcopy(m)(x)
    bound(got, want, t32, "eval forward %s" % (shape,))


@pytest.mark.parametrize("shape", STAGES + ODD, ids=IDS)
def test_train_forward_and_running_stats(cuda, shape):
    B, Ci, Co, Hi, Wi = shape
    m = make_up(Ci, Co, 2).train()
    m64, m32 = copy.deepcopy(m).double(), copy.deepcopy(m)
    x = rand((B, Ci, Hi, Wi), sum(shape) + 1)
    with torch.no_grad():
        got = m.forward_restructured(x)
        want = m64(x.double())
        t32 = m32(x)
    bound(got, want, t32, "training forward %s" % (shape,))
    bn, bn64 = m.conv[2], m64.conv[2]
    within(bn.running_mean, bn64.running_mean, "running_mean")
    within(bn.running_var, bn64.running_var, "running_var")
    assert bn.num_batches_tracked.item() == bn64.num_batches_tracked.item() == 1


@pytest.mark.parametrize("shape", STAGES + ODD, ids=IDS)
def test_train_backward(cuda, shape):
    B, Ci, Co, Hi, Wi = shape
    m = make_up(Ci, Co, 3).train()
    refs_m = [copy.deepcopy(m).double(), copy.deepcopy(m)]
    x0 = rand((B, Ci, Hi, Wi), sum(shape) + 2)
    x = x0.clone().requires_grad_(True)
    out = m.forward_restructured(x)
    grad = rand(out.shape, sum(shape) + 3)
    out.backward(grad)
    refs = []
    for r, dtype in zip(refs_m, (torch.float64, torch.float32)):
        xr = x0.to(dtype).requires_grad_(True)
        r(xr).backward(grad.to(dtype))
        refs.append([xr.grad] + [p.grad for _, p in params(r)])
    got = [x.grad] + [p.grad for _, p in params(m)]
    names = ["x"] + [n for n, _ in params(m)]
    for name, a, w64, w32 in zip(names, got, *refs):
        if name == "bias":
            # the conv bias feeds a training-mode BatchNorm: its exact gradient is 0, both paths give round-off,
            # bounded against the weight gradient's scale
            wscale = refs[0][1].abs().max().item()
            assert max(a.abs().max().item(), w64.abs().max().item()) <= 1e-3 * wscale, shape
        else:
            bound(a, w64, w32, "%s %s" % (shape, name))


@pytest.mark.parametrize("shape", [(2, 7, 130, 3, 5), (1, 3, 2, 4, 3)], ids=IDS)
def test_eval_backward(cuda, shape):
    """Eval mode under autograd: the conv's backward on the kernels, the module's BatchNorm and PReLU."""
    B, Ci, Co, Hi, Wi = shape
    m = make_up(Ci, Co, 4).eval()
    refs_m = [copy.deepcopy(m).double(), copy.deepcopy(m)]
    x0 = rand((B, Ci, Hi, Wi), 5)
    x = x0.clone().requires_grad_(True)
    out = m.forward_restructured(x)
    grad = rand(out.shape, 6)
    out.backward(grad)
    refs = []
    for r, dtype in zip(refs_m, (torch.float64, torch.float32)):
        xr = x0.to(dtype).requires_grad_(True)
        r(xr).backward(grad.to(dtype))
        refs.append([xr.grad] + [p.grad for _, p in params(r)])
    got = [x.grad] + [p.grad for _, p in params(m)]
    for name, a, w64, w32 in zip(["x"] + [n for n, _ in params(m)], got, *refs):
        bound(a, w64, w32, "eval %s %s" % (shape, name))


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
def test_nonfinite(cuda, train):
    m = make_up(6, 5, 5).train(train)
    x = rand((2, 6, 5, 7), 7)
    x[0, 1, 2, 3] = float("nan")
    x[1, 0, 0, 0] = float("inf")
    x[1, 5, 4, 6] = float("-inf")
    ref = copy.deepcopy(m)
    with torch.no_grad():
        got = m.forward_restructured(x)
        want = ref(x)
    bad = ~torch.isfinite(want)
    assert bad.any()
    assert (~torch.isfinite(got))[bad].all(), "%d outputs torch makes non-finite are finite here" % int(
        (torch.isfinite(got) & bad).sum())


# ------------------------------------------------------------------------------------------------ repeatability
def _stage_step(m, x, grad):
    for _, p in params(m):
        p.grad = None
    x.grad = None
    m.forward_restructured(x).backward(grad)
    return [x.grad.clone()] + [p.grad.clone() for _, p in params(m)]


def test_deterministic_mode_and_graph_replay(cuda):
    m = make_up(64, 64, 6).train()
    x = rand((2, 64, 30, 40), 8).requires_grad_(True)
    grad = rand((2, 64, 60, 80), 9)
    with deterministic():
        first, second = _stage_step(m, x, grad), _stage_step(m, x, grad)
        assert all(torch.equal(a, b) for a, b in zip(first, second))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                _stage_step(m, x, grad)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            m.forward_restructured(x).backward(grad)
        for _ in range(2):
            for _, p in params(m):
                p.grad.zero_()
            x.grad.zero_()
            graph.replay()
            torch.cuda.synchronize()
            got = [x.grad] + [p.grad for _, p in params(m)]
            assert all(torch.equal(a, b) for a, b in zip(first, got))


def test_graphed_train_step_bitwise_with_flag(cuda):
    seq = items(True)
    with deterministic():
        mg, og, me, oe = pair("ffb6d")
        mg.fused_upsample = me.fused_upsample = True
        step = F.GraphedTrainStep(mg, og, seq[0])
        assert_bitwise(mg, og, me, oe, "after warm-up and capture", with_adam=False)
        for i, item in enumerate(seq):
            loss, _ = step(item)
            want, _ = eager_step(me, oe, item)
            assert torch.equal(loss, want), "step %d" % i
            assert_bitwise(mg, og, me, oe, "step %d" % i)
        assert step.captures == 1
        mg.fused_upsample = me.fused_upsample = False          # a baked switch: the next call captures again
        step(seq[0])
        eager_step(me, oe, seq[0])
        assert step.captures == 2
        assert_bitwise(mg, og, me, oe, "after the switch")


def test_graphed_eval_step_bitwise_with_flag(cuda):
    seq = items(True)
    model = pair("ffb6d")[0].eval()
    model.fused_upsample = True
    step = F.GraphedEvalStep(model, seq[0])
    for item in seq:
        ep, loss, _ = step(item)
        with torch.no_grad():
            want = model(item)
        for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs"):
            assert torch.equal(ep[k], want[k]), k
    assert step.captures == 1


# ------------------------------------------------------------------------------------------------ SyncBatchNorm
SYNC = (4, 12, 10, 5, 7)        # B, Ci, Co, Hi, Wi


def _sync_worker(rank, world, init_file, out_dir):
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world,
                                timeout=datetime.timedelta(seconds=120))
        B, Ci, Co, Hi, Wi = SYNC
        m = nn.SyncBatchNorm.convert_sync_batchnorm(make_up(Ci, Co, 7)).train()
        assert isinstance(m.conv[2], nn.SyncBatchNorm)
        half = B // world
        x = rand((B, Ci, Hi, Wi), 10)[rank * half:(rank + 1) * half].clone().requires_grad_(True)
        grad = rand((B, Co, 2 * Hi, 2 * Wi), 11)[rank * half:(rank + 1) * half]
        out = m.forward_restructured(x)
        out.backward(grad)
        res = {"out": out.detach().cpu(), "x": x.grad.cpu(), "running_mean": m.conv[2].running_mean.cpu(),
               "running_var": m.conv[2].running_var.cpu()}
        res.update({n: p.grad.cpu() for n, p in params(m)})
        torch.save(res, os.path.join(out_dir, "rank%d.pt" % rank))
        dist.destroy_process_group()
    except Exception:
        with open(os.path.join(out_dir, "rank%d.err" % rank), "w") as f:
            f.write(traceback.format_exc())
        raise


def test_syncbn_two_ranks_gloo(cuda, tmp_path):
    world = 2
    mp.start_processes(_sync_worker, args=(world, str(tmp_path / "init"), str(tmp_path)), nprocs=world,
                       start_method="spawn", join=True)
    res = [torch.load(tmp_path / ("rank%d.pt" % r)) for r in range(world)]
    B, Ci, Co, Hi, Wi = SYNC
    m64 = make_up(Ci, Co, 7).double().train()
    x = rand((B, Ci, Hi, Wi), 10).double().requires_grad_(True)
    out = m64(x)
    out.backward(rand((B, Co, 2 * Hi, 2 * Wi), 11).double())
    within(torch.cat([r["out"] for r in res]), out.cpu(), "SyncBatchNorm forward")
    within(torch.cat([r["x"] for r in res]), x.grad.cpu(), "SyncBatchNorm grad x")
    for r in res:
        within(r["running_mean"], m64.conv[2].running_mean.cpu(), "running_mean")
        within(r["running_var"], m64.conv[2].running_var.cpu(), "running_var")
    for n, p in params(m64):
        if n != "bias":          # exactly 0 (training BatchNorm follows), round-off on both sides
            within(sum(r[n] for r in res), p.grad.cpu(), "SyncBatchNorm grad %s (sum over ranks)" % n, 1e-4)


# ------------------------------------------------------------------------------------------------ memory
@pytest.mark.parametrize("stage", [0, 1, 2], ids=["up_1", "up_2", "up_3"])
def test_peak_memory_at_or_below_torch(cuda, stage):
    B, Ci, Co, Hi, Wi = STAGES[stage]
    m = make_up(Ci, Co, 8).train()
    x = rand((B, Ci, Hi, Wi), 12).requires_grad_(True)
    grad = rand((B, Co, 2 * Hi, 2 * Wi), 13)

    def peak(fn):
        x.grad = None
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn(x).backward(grad)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    peak(m)
    peak(m.forward_restructured)                 # warm: cuDNN plans and the weight pack exist before measuring
    t, ours = peak(m), peak(m.forward_restructured)
    print("%s B=%d peak extra memory: torch %.1f MB, restructured %.1f MB" % (("up_1", "up_2", "up_3")[stage], B,
                                                                               t / 2 ** 20, ours / 2 ** 20))
    assert ours <= t


# ------------------------------------------------------------------------------------------------ whole network
def test_ffb6d_training_step_flag_on_matches_off(cuda):
    model, inputs, _ = _network(train=True)
    item = _item(inputs)
    want, want_stats = _train_step(copy.deepcopy(model), inputs, item)
    calls, real = [], ops.upsample_conv3x3

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)
    model.fused_upsample = True
    try:
        ops.upsample_conv3x3 = spy
        got, got_stats = _train_step(model, inputs, item)
    finally:
        ops.upsample_conv3x3 = real
    assert len(calls) == 3
    zero = [n for n in want if n.startswith("cnn_up_stages.") and n.endswith(".conv.1.bias")]
    assert len(zero) == 3
    for n in zero:
        wscale = want[n[:-len("bias")] + "weight"].abs().max().item()
        assert max(want[n].abs().max().item(), got[n].abs().max().item()) <= 1e-3 * wscale, n
    rel = sorted((((got[n] - w).abs().max().item() / max(w.abs().max().item(), 1e-30), n)
                  for n, w in want.items() if n not in zero), reverse=True)
    print("gradient differences, fused_upsample on against off: largest %s, median %.2e" % (rel[:5], rel[len(rel) // 2][0]))
    assert rel[0][0] <= 5e-2, rel[:5]
    assert rel[len(rel) // 2][0] <= 1e-2, rel[len(rel) // 2]
    for n, w in want_stats.items():
        if w.is_floating_point():
            close(got_stats[n], w, "buffer %s" % n, 1e-4)


def test_ffb6d_eval_flag_on_matches_float64_restatement(cuda):
    model, inputs, _ = _network()
    model.fused_upsample = True
    with torch.no_grad():
        out = model(inputs)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    with torch.no_grad():
        want = FullRef(model, sd, 8).forward(inputs, inputs["rgb"])
    model.fused_upsample = False
    with torch.enable_grad():
        out_t = model(inputs)            # the image branch on torch's modules, in fp32
    names = ["pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs"] + ["fused_rgb%d" % i for i in range(7)]

    def flat(d):
        return [d[k] for k in names[:3]] + list(d["fused_rgb"])
    for k, a, t32, b in zip(names, flat(out), flat(out_t), flat(want)):
        scale = b.abs().max().item()
        e_ours = (a.double() - b).abs().max().item() / scale
        e_t32 = (t32.detach().double() - b).abs().max().item() / scale
        assert e_ours <= max(5e-5, 2 * e_t32), "FFB6D eval %s: %.2e of scale (torch modules: %.2e)" % (k, e_ours, e_t32)
