"""GPU: FFB6D's training step captured in one CUDA graph (:class:`ffb6d_b200.GraphedTrainStep`, DESIGN.md §4.20).

Three graphed steps on three different items against three eager steps of a deep copy, bit for bit under
``torch.use_deterministic_algorithms(True)`` (losses, ``info``, every parameter, buffer and Adam state tensor) for
FFB6DFusionNet in its default, restructured and fused-LFA forms and for the whole FFB6D with the fused image head;
the same in default mode within the bounds of the atomic backwards; the fused head's packed weights under capture
(each replay packs the weights it is given); schedulers and re-capture; and the rejections.  Shapes are those of
test_gpu_model: B = 2, 120x160, 4096 points."""
import contextlib
import copy

import pytest
import torch
import torch.distributed as dist

import ffb6d_b200 as F
from ffb6d_b200 import _lib, cnn
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D, FFB6DFusionNet
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu

B, H, W, N, N_CLS, N_KPS = 2, 120, 160, 4096, 5, 8
LR = 1e-3
_items = {}


@contextlib.contextmanager
def deterministic(on=True):
    saved = torch.are_deterministic_algorithms_enabled(), torch.backends.cudnn.deterministic
    torch.use_deterministic_algorithms(on)
    torch.backends.cudnn.deterministic = on
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(saved[0])
        torch.backends.cudnn.deterministic = saved[1]


def make_item(seed, image, invalid=None):
    """A seeded batch: the indices of two synthetic frames, targets with 60 % background, and either the image
    (FFB6D) or the eight image-branch maps (FFB6DFusionNet).  ``invalid``: a frame flagged ``valid = False``."""
    key = (seed, image, invalid)
    if key not in _items:
        batch = make_batch([seed, seed + 1], n_points=N, h=H, w=W)
        item = build_ffb6d_indices(torch.from_numpy(batch["cld"]).cuda(), torch.from_numpy(batch["dpt_xyz"]).cuda())
        item["choose"] = torch.from_numpy(batch["choose"]).cuda()
        item["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).cuda()
        g = torch.Generator(device="cuda").manual_seed(seed)
        if image:
            item["rgb"] = torch.rand((B, 3, H, W), generator=g, device="cuda") * 2 - 1
        else:
            item["rgb_feats"] = [torch.randn(s, generator=g, device="cuda")
                                 for s in FFB6DFusionNet.rgb_feature_shapes(B, H, W)]
        labels = torch.randint(1, N_CLS, (B, N), generator=g, device="cuda", dtype=torch.int32)
        labels[torch.rand((B, N), generator=g, device="cuda") < 0.6] = 0
        item.update(labels=labels, kp_targ_ofst=torch.randn((B, N, N_KPS, 3), generator=g, device="cuda"),
                    ctr_targ_ofst=torch.randn((B, N, 3), generator=g, device="cuda"),
                    valid=torch.ones(B, dtype=torch.bool, device="cuda"))
        if invalid is not None:
            item["valid"][invalid] = False
        _items[key] = item
    return _items[key]


def items(image):
    return [make_item(3, image), make_item(11, image, invalid=1), make_item(21, image)]


def make_model(kind):
    torch.manual_seed(3)
    if kind == "ffb6d":
        model = FFB6D(n_classes=N_CLS, n_pts=N, n_kps=N_KPS, fused_image_head=True).cuda()
        for m in model.modules():
            if isinstance(m, torch.nn.modules.dropout._DropoutNd):
                m.p = 0.0                      # the runs are compared bit for bit
    else:
        model = FFB6DFusionNet(n_classes=N_CLS, n_pts=N, n_kps=N_KPS, restructured=kind == "restructured",
                               fused_lfa=kind == "fused_lfa").cuda()
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
    return model.train()


def adam(model, capturable=True):
    return torch.optim.Adam(model.parameters(), lr=torch.tensor(LR, device="cuda"), capturable=capturable)


def eager_step(model, opt, item):
    opt.zero_grad(set_to_none=True)
    out = model(item) if isinstance(model, FFB6D) else model(item, item["rgb_feats"])
    loss, info = ffb6d_loss(out, item, valid=item["valid"])
    loss.backward()
    opt.step()
    return loss.detach(), info


def pair(kind):
    """A model with its Adam, and a deep copy with its own, taken before any step."""
    model = make_model(kind)
    twin = copy.deepcopy(model)
    return model, adam(model), twin, adam(twin)


def state_pairs(mg, og, me, oe, with_adam=True):
    """``(what, graphed tensor, eager tensor)`` of every parameter, buffer and Adam state tensor."""
    out = [("param " + n, a, b) for (n, a), (_, b) in zip(mg.named_parameters(), me.named_parameters())]
    out += [("buffer " + n, a, b) for (n, a), (_, b) in zip(mg.named_buffers(), me.named_buffers())]
    for (n, pg), pe in zip(mg.named_parameters(), me.parameters()) if with_adam else ():
        sg, se = og.state.get(pg, {}), oe.state.get(pe, {})
        assert sorted(sg) == sorted(se), "Adam state keys of %s: %s vs %s" % (n, sorted(sg), sorted(se))
        out += [("Adam %s of %s" % (k, n), sg[k], se[k]) for k in sg]
    return out


def assert_bitwise(mg, og, me, oe, when, with_adam=True):
    diff = [w for w, a, b in state_pairs(mg, og, me, oe, with_adam) if not torch.equal(a, b)]
    assert diff == [], "%s: %d tensors differ, first %s" % (when, len(diff), diff[:5])


# ------------------------------------------------------------------------------------------ bitwise, deterministic
@pytest.mark.parametrize("kind", ["default", "restructured", "fused_lfa", "ffb6d"])
def test_graphed_steps_bitwise_equal_eager(cuda, kind):
    image = kind == "ffb6d"
    seq = items(image)
    with deterministic():
        mg, og, me, oe = pair(kind)
        step = F.GraphedTrainStep(mg, og, seq[0])
        assert step.captures == 1
        # the warm-up left no trace (its Adam state is zeroed; the eager twin has none before its first step)
        assert_bitwise(mg, og, me, oe, "after warm-up and capture", with_adam=False)
        assert all(not t.any() for st in og.state.values() for t in st.values())
        for i, item in enumerate(seq):
            loss, info = step(item)
            want, want_info = eager_step(me, oe, item)
            assert torch.equal(loss, want), "step %d: loss %r vs eager %r" % (i, loss.item(), want.item())
            for k in want_info:
                assert torch.equal(info[k], want_info[k]), "step %d: info %s" % (i, k)
            assert_bitwise(mg, og, me, oe, "step %d" % i)
        assert step.captures == 1


# ------------------------------------------------------------------------------------------ default mode
def sync_twin(mg, og, me, oe):
    """The eager twin takes the graphed model's parameters, buffers and Adam state, so each step starts equal."""
    with torch.no_grad():
        for a, b in zip(list(mg.parameters()) + list(mg.buffers()), list(me.parameters()) + list(me.buffers())):
            b.copy_(a)
        for pg, pe in zip(mg.parameters(), me.parameters()):
            for k, t in oe.state.get(pe, {}).items():
                t.copy_(og.state[pg][k])


def adam_restated(params, state, grads):
    """Adam's step on copies of ``params`` / ``state`` with the gradients ``grads``, eagerly."""
    copies = [p.detach().clone().requires_grad_(True) for p in params]
    opt = torch.optim.Adam(copies, lr=torch.tensor(LR, device="cuda"), capturable=True)
    for c, g, st in zip(copies, grads, state):
        c.grad = g
        if st:
            opt.state[c] = {k: t.clone() for k, t in st.items()}
    opt.step()
    return copies, opt


@pytest.mark.parametrize("kind", ["default", "restructured", "fused_lfa", "ffb6d"])
def test_graphed_steps_default_mode(cuda, kind):
    """Without the determinism switch the atomic backwards add in a run-dependent order.  Each of three steps starts the
    eager twin from the graphed model's state; then the loss and ``info`` agree within 1e-5, every gradient within
    test_gpu_deterministic's 2e-3 of its layer's scale, the running statistics within 1e-4, and the graphed Adam
    update is bit for bit Adam's update with the gradients the graph computed."""
    seq = items(kind == "ffb6d")
    mg, og, me, oe = pair(kind)
    with deterministic(False):
        step = F.GraphedTrainStep(mg, og, seq[0])
        for i, item in enumerate(seq):
            sync_twin(mg, og, me, oe)
            params = list(mg.parameters())
            before = [p.detach().clone() for p in params]
            state = [{k: t.clone() for k, t in og.state.get(p, {}).items()} for p in params]
            loss, info = step(item)
            grads = [p.grad.clone() if p.grad is not None else None for p in params]
            want, want_info = eager_step(me, oe, item)
            torch.testing.assert_close(loss, want, rtol=1e-5, atol=0, msg="step %d: loss" % i)
            for k in want_info:
                torch.testing.assert_close(info[k], want_info[k], rtol=1e-5, atol=1e-7, msg="step %d: %s" % (i, k))
            names = [n for n, _ in mg.named_parameters()]
            scale = {}
            for n, pe in zip(names, me.parameters()):
                if pe.grad is not None:
                    unit = n.rsplit(".", 1)[0]
                    scale[unit] = max(scale.get(unit, 1e-12), pe.grad.norm().item())
            for n, g, pe in zip(names, grads, me.parameters()):
                assert (g is None) == (pe.grad is None), "step %d: grad of %s" % (i, n)
                if g is not None:
                    err = (g - pe.grad).norm().item() / scale[n.rsplit(".", 1)[0]]
                    assert err <= 2e-3, "step %d: grad of %s differs by %.2e of its layer's scale" % (i, n, err)
            for (n, a), (_, b) in zip(mg.named_buffers(), me.named_buffers()):
                if a.is_floating_point():
                    torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-6, msg="step %d: buffer %s" % (i, n))
                else:
                    assert torch.equal(a, b), n
            # the parameters moved by exactly Adam's update of the gradients the graph computed
            copies, opt_c = adam_restated(before, state, grads)
            for n, p, c in zip(names, params, copies):
                assert torch.equal(p, c), "step %d: parameter %s is not Adam's update of its gradient" % (i, n)
                for k, t in opt_c.state.get(c, {}).items():
                    assert torch.equal(og.state[p][k], t), "step %d: Adam %s of %s" % (i, k, n)
        assert step.captures == 1


# ------------------------------------------------------------------------------------------ stale packs
def test_fused_head_repacks_every_replay(cuda):
    """PSPModule and Final reuse packed weights in eager mode.  Captured with the caches warm at the current weights,
    each replay must still pack the weights its captured Adam step left, as an eager step sees them."""
    torch.manual_seed(4)
    psp, up, final = cnn.PSPModule(64, 128).cuda(), cnn.PSPUpsample(128, 64).cuda().train(), cnn.Final(64).cuda()
    with torch.no_grad():
        psp.bottleneck.bias.normal_(0, 0.5)
    chain = torch.nn.ModuleList([psp, up, final])
    twin = copy.deepcopy(chain)
    x = torch.relu(torch.randn(B, 64, 30, 40, device="cuda"))
    w = torch.randn(B, 64, 60, 80, device="cuda")

    def step(c, opt):
        opt.zero_grad(set_to_none=True)
        loss = (c[2].forward_fused(c[1].forward_fused(c[0].forward_fused(x))) * w).sum()
        loss.backward()
        opt.step()
        return loss.detach()

    with deterministic():
        opt, opt_e = adam(chain), adam(twin)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step(chain, opt)                             # Adam's state, cuDNN plans
        torch.cuda.current_stream().wait_stream(side)
        step(twin, opt_e)
        with torch.no_grad():                            # both caches now hold the current weights' packs
            psp.forward_fused(x)
            final.forward_fused(w)
        assert psp._packed is not None and final._packed is not None
        opt.zero_grad(set_to_none=True)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss = step(chain, opt)
        for i in range(4):
            graph.replay()
            want = step(twin, opt_e)
            assert torch.equal(loss, want), "replay %d: loss %r vs eager %r" % (i, loss.item(), want.item())
            for (n, a), (_, b) in zip(chain.named_parameters(), twin.named_parameters()):
                assert torch.equal(a, b), "replay %d: %s" % (i, n)


# ------------------------------------------------------------------------------------------ schedulers, re-capture
def test_cyclic_lr_captures_once(cuda):
    seq = items(False)
    with deterministic():
        mg, og, me, oe = pair("default")
        scheds = [torch.optim.lr_scheduler.CyclicLR(o, base_lr=1e-5, max_lr=1e-3, step_size_up=2, cycle_momentum=False)
                  for o in (og, oe)]
        step = F.GraphedTrainStep(mg, og, seq[0])
        lrs = []
        for i in range(5):
            step(seq[i % 3])
            eager_step(me, oe, seq[i % 3])
            for s in scheds:
                s.step()
            lrs.append(og.param_groups[0]["lr"].item())
            assert_bitwise(mg, og, me, oe, "step %d" % i)
        assert len(set(lrs)) > 2, lrs                   # the learning rate did move
        assert step.captures == 1


def test_bn_momentum_change_recaptures(cuda):
    seq = items(False)
    with deterministic():
        mg, og, me, oe = pair("default")
        step = F.GraphedTrainStep(mg, og, seq[0])
        step(seq[0])
        eager_step(me, oe, seq[0])
        for m in (mg, me):                              # as BNMomentumScheduler sets it, on one layer
            m.rndla_pre_stages.bn.bn.momentum = 0.5
        step(seq[1])
        eager_step(me, oe, seq[1])
        assert step.captures == 2
        assert_bitwise(mg, og, me, oe, "after the new momentum")
        step(seq[2])
        eager_step(me, oe, seq[2])
        assert step.captures == 2
        assert_bitwise(mg, og, me, oe, "one step later")


def test_switches_recapture(cuda):
    seq = items(False)
    model = make_model("default")
    opt = adam(model)
    with deterministic():
        step = F.GraphedTrainStep(model, opt, seq[0], warmup=1)
        step(seq[0])
        assert step.captures == 1
        torch.use_deterministic_algorithms(False)
        step(seq[1])
        assert step.captures == 2
        model.fused_lfa = True
        step(seq[2])
        assert step.captures == 3
        step(seq[0])
        assert step.captures == 3
    loss, _ = step(seq[1])                              # the determinism switch restored by the context: again
    assert step.captures == 4 and torch.isfinite(loss).item()


def test_module_swap_recaptures(cuda):
    """A submodule swapped after construction (the optimizer left as it is) is what the next step runs, through a
    new capture: its loss is the eager forward's of the swapped model, bit for bit."""
    seq = items(False)
    model = make_model("default")
    with deterministic():
        step = F.GraphedTrainStep(model, adam(model), seq[0], warmup=1)
        step(seq[0])
        new_head = copy.deepcopy(model.rgbd_seg_layer[3])
        with torch.no_grad():
            new_head.conv.weight.mul_(0.5)
        model.rgbd_seg_layer[3] = new_head
        twin = copy.deepcopy(model)
        want, _ = ffb6d_loss(twin(seq[1], seq[1]["rgb_feats"]), seq[1], valid=seq[1]["valid"])
        loss, _ = step(seq[1])
        assert step.captures == 2
        assert torch.equal(loss, want.detach())


def test_eval_caches_see_graphed_updates(cuda):
    """After replays the eval path's packed weights follow the parameters the graph updated."""
    seq = items(True)
    model = make_model("ffb6d")
    step = F.GraphedTrainStep(model, adam(model), seq[0], warmup=1)
    model.eval()
    with torch.no_grad():
        model(seq[0])                                   # fills the eval caches
    model.train()
    step(seq[1])
    step(seq[2])
    model.eval()
    with torch.no_grad():
        got = model(seq[0])["pred_rgbd_segs"]
        fresh = copy.deepcopy(model)
        for m in fresh.modules():                       # every cached pack dropped: built from the weights as they are
            for attr in ("_packed", "_split", "_fc_pack"):
                if hasattr(m, attr):
                    setattr(m, attr, None)
        want = fresh(seq[0])["pred_rgbd_segs"]
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------ rejections
def test_rejects_mismatched_items(cuda):
    seq = items(False)
    model = make_model("default")
    step = F.GraphedTrainStep(model, adam(model), seq[0], warmup=1)
    bad_key = {k: v for k, v in seq[1].items() if k != "labels"}
    bad_shape = dict(seq[1], labels=seq[1]["labels"][:, :N // 2])
    bad_dtype = dict(seq[1], labels=seq[1]["labels"].long())
    bad_feat = dict(seq[1], rgb_feats=seq[1]["rgb_feats"][:7])
    for bad, what in ((bad_key, "missing"), (bad_shape, "captured for"), (bad_dtype, "captured for"),
                      (bad_feat, "missing")):
        with pytest.raises(ValueError, match=what):
            step(bad)
    assert step.captures == 1
    loss, _ = step(seq[1])
    torch.cuda.synchronize()                            # no CUDA error left behind
    assert torch.isfinite(loss).item()


def test_rejects_what_cannot_be_captured(cuda, monkeypatch):
    # the library reads FFB6D_CHECK_INDICES once, at its first use: let it read it unset before the test sets it
    assert not _lib.lib.ffb6d_check_indices_enabled()
    item = make_item(3, False)
    model = make_model("default")
    with pytest.raises(ValueError, match="capturable"):
        F.GraphedTrainStep(model, adam(model, capturable=False), item)
    model.rndla_pre_stages.bn.bn.momentum = None
    with pytest.raises(ValueError, match="momentum=None"):
        F.GraphedTrainStep(model, adam(model), item)
    model.rndla_pre_stages.bn.bn.momentum = 0.99
    model.eval()
    with pytest.raises(ValueError, match="eval mode"):
        F.GraphedTrainStep(model, adam(model), item)
    model.train()
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="FFB6D_CHECK_INDICES"):
        F.GraphedTrainStep(model, adam(model), item)
    monkeypatch.delenv("FFB6D_CHECK_INDICES")
    step = F.GraphedTrainStep(model, adam(model), item, warmup=1)
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="FFB6D_CHECK_INDICES"):
        step(item)
    monkeypatch.delenv("FFB6D_CHECK_INDICES")
    torch.cuda.synchronize()


def test_rejects_ddp(cuda, tmp_path):
    dist.init_process_group("gloo", init_method="file://%s" % (tmp_path / "store"), rank=0, world_size=1)
    try:
        model = make_model("default")
        ddp = torch.nn.parallel.DistributedDataParallel(model)
        with pytest.raises(ValueError, match="DataParallel"):
            F.GraphedTrainStep(ddp, adam(model), make_item(3, False))
    finally:
        dist.destroy_process_group()
    torch.cuda.synchronize()
