"""GPU: the training path of the PSP head, PSPUpsample's upsampling and ``final`` on the package's kernels
(DESIGN.md §4.18): each backward against float64 autograd at the training shapes and at odd ones, non-finite inputs,
determinism and graph replay, and the whole ``FFB6D(fused_image_head=True)`` training step against the torch-module
path, under ``torch.use_deterministic_algorithms(True)`` included.

A gradient passes within 1e-5 of its scale of float64 autograd, or at most twice as far from it as the same
composition on torch's fp32 modules (cuDNN / cuBLAS TF32 off for this file), whichever is larger."""
import contextlib
import copy

import pytest
import torch
import torch.nn.functional as Fn

from ffb6d_b200 import cnn, ops
from ffb6d_b200.loss import ffb6d_loss
from test_gpu_cnn import _network, same_nonfinite
from test_gpu_model import close

pytestmark = pytest.mark.gpu
TOL = 1e-5


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


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


def bound(got, want, t32, what):
    """``got`` within TOL of ``want``'s (float64) scale, or at most 2x as far from it as ``t32`` (torch fp32)."""
    got, want, t32 = got.detach().double(), want.detach().double(), t32.detach().double()
    scale = max(want.abs().max().item(), 1e-30)
    e, e32 = (got - want).abs().max().item(), (t32 - want).abs().max().item()
    assert e <= max(TOL * scale, 2 * e32), "%s: %.2e of scale (torch fp32: %.2e)" % (what, e / scale, e32 / scale)


# ----------------------------------------------------------------------------------------------- PSP head
def make_psp(C, Co, seed):
    torch.manual_seed(seed)
    m = cnn.PSPModule(C, Co).cuda()
    with torch.no_grad():
        m.bottleneck.bias.normal_(0, 0.5)
    return m


def psp_pre_relu(m, x):
    """The torch module's bottleneck sum before its ReLU (the reference's order of operations)."""
    h, w = x.shape[2], x.shape[3]
    priors = [Fn.interpolate(st(x), size=(h, w), mode="bilinear", align_corners=False) for st in m.stages] + [x]
    return m.bottleneck(torch.cat(priors, 1))


def psp_grads(m, x):
    return [x.grad] + [st[1].weight.grad for st in m.stages] + [m.bottleneck.weight.grad, m.bottleneck.bias.grad]


PSP_NAMES = ["x", "stage1", "stage2", "stage3", "stage6", "bottleneck", "bias"]
PSP_SHAPES = [(8, 512, 60, 80, 1024), (1, 512, 60, 80, 1024), (2, 5, 7, 11, 9), (3, 3, 5, 4, 7), (2, 3, 1, 1, 4),
              (1, 6, 2, 5, 3), (1, 2, 6, 1, 5), (1, 8, 4, 5, 130), (2, 16, 13, 17, 200)]


@pytest.mark.parametrize("shape", PSP_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_psp_backward(cuda, shape):
    B, C, H, W, Co = shape
    m = make_psp(C, Co, 1)
    g = torch.Generator(device="cuda").manual_seed(H * W + C)
    x0 = torch.relu(torch.randn((B, C, H, W), generator=g, device="cuda"))
    x = x0.clone().requires_grad_(True)
    out = m.forward_fused(x)
    with torch.no_grad():
        assert torch.equal(out, m.forward_fused(x0))        # the forward is the inference kernels', bitwise
    grad = torch.randn(out.shape, generator=g, device="cuda")
    out.backward(grad)
    got = psp_grads(m, x)
    # the references take the ReLU mask of the kernels' output, so that they differ from it only in the backward
    gz = torch.ops.aten.threshold_backward(grad, out.detach(), 0)
    refs = []
    for dtype in (torch.float64, torch.float32):
        mr = copy.deepcopy(m).to(dtype)
        xr = x0.to(dtype).requires_grad_(True)
        psp_pre_relu(mr, xr).backward(gz.to(dtype))
        refs.append(psp_grads(mr, xr))
    for name, a, w64, w32 in zip(PSP_NAMES, got, *refs):
        if name == "bottleneck":
            for i in range(5):
                sl = slice(i * C, (i + 1) * C)
                bound(a.reshape(Co, -1)[:, sl], w64.reshape(Co, -1)[:, sl], w32.reshape(Co, -1)[:, sl],
                      "psp %s block %d" % (shape, i))
        else:
            bound(a, w64, w32, "psp %s %s" % (shape, name))


def table_reference(gz, H, W, dtype=torch.float64):
    """d/dT_s of sum(gz * up_s(T_s)) for the four prior tables, by autograd of F.interpolate (align_corners=False),
    each [B, Co, s, s]."""
    B, Co = gz.shape[:2]
    out = []
    for s in ops.PSP_SIZES:
        t = torch.zeros((B, Co, s, s), dtype=dtype, device=gz.device, requires_grad=True)
        up = Fn.interpolate(t, size=(H, W), mode="bilinear", align_corners=False)
        (up * gz.to(dtype)).sum().backward()
        out.append(t.grad)
    return out


def table_blocks(table, B, Co):
    blocks, row = [], 0
    for s in ops.PSP_SIZES:
        blocks.append(table[row:row + B * s * s].view(B, s, s, Co).permute(0, 3, 1, 2))
        row += B * s * s
    return blocks


@pytest.mark.parametrize("shape", [(8, 1024, 60, 80), (2, 9, 7, 11), (1, 3, 1, 1), (2, 5, 2, 5), (1, 4, 6, 1)],
                         ids=lambda s: "x".join(map(str, s)))
def test_psp_bottleneck_bwd_kernel(cuda, shape):
    B, Co, H, W = shape
    g = torch.Generator(device="cuda").manual_seed(H + W)
    out = torch.relu(torch.randn(shape, generator=g, device="cuda"))
    grad = torch.randn(shape, generator=g, device="cuda")
    gz, table, gsum = ops.psp_bottleneck_bwd(grad, out)
    assert torch.equal(gz, torch.ops.aten.threshold_backward(grad, out, 0))
    for s, a, w64, w32 in zip(ops.PSP_SIZES, table_blocks(table, B, Co), table_reference(gz, H, W),
                              table_reference(gz, H, W, torch.float32)):
        bound(a, w64, w32, "table s=%d %s" % (s, shape))
    close(gsum, gz.double().sum((2, 3)), "plane sums", TOL)


def test_psp_bottleneck_bwd_nonfinite(cuda):
    B, Co, H, W = 2, 6, 7, 11
    g = torch.Generator(device="cuda").manual_seed(5)
    out = torch.relu(torch.randn((B, Co, H, W), generator=g, device="cuda"))
    grad = torch.randn((B, Co, H, W), generator=g, device="cuda")
    out[0, 0, 0, :4] = torch.tensor([0.0, -0.0, float("nan"), 1.0])   # the ReLU mask at 0, -0 and NaN
    grad[0, 0, 0, :4] = 3.0
    grad[0, 1, 3, 5] = float("nan")
    grad[1, 2, 6, 10] = float("inf")
    grad[1, 3, 0, 0] = float("-inf")
    out[0, 1, 3, 5] = out[1, 2, 6, 10] = out[1, 3, 0, 0] = 1.0
    gz, table, gsum = ops.psp_bottleneck_bwd(grad, out)
    want = torch.ops.aten.threshold_backward(grad, out, 0)
    assert torch.equal(torch.isnan(gz), torch.isnan(want))
    fin = ~torch.isnan(want)
    assert torch.equal(gz[fin], want[fin])
    assert gz[0, 0, 0, :4].tolist() == [0.0, 0.0, 3.0, 3.0]              # NaN out passes the gradient, as in torch
    for s, a, w in zip(ops.PSP_SIZES, table_blocks(table, B, Co), table_reference(gz, H, W)):
        same_nonfinite(a, w, "table s=%d" % s)
    same_nonfinite(gsum, gz.double().sum((2, 3)), "plane sums")


@pytest.mark.parametrize("shape", [(8, 512, 60, 80), (2, 5, 7, 11), (1, 3, 1, 1), (2, 4, 5, 4), (1, 2, 1024, 7)],
                         ids=lambda s: "x".join(map(str, s)))
def test_psp_pool_bwd_kernel(cuda, shape):
    B, C, H, W = shape
    g = torch.Generator(device="cuda").manual_seed(H * W)
    gp = [torch.randn((B, C, s, s), generator=g, device="cuda") for s in ops.PSP_SIZES]
    base = torch.randn(shape, generator=g, device="cuda")
    got = ops.psp_pool_bwd(gp, base.clone())
    ref = []
    for dtype in (torch.float64, torch.float32):
        x = torch.zeros(shape, dtype=dtype, device="cuda", requires_grad=True)
        sum((Fn.adaptive_avg_pool2d(x, s) * p.to(dtype)).sum() for s, p in zip(ops.PSP_SIZES, gp)).backward()
        ref.append(x.grad + base.to(dtype))
    bound(got, *ref, "pool adjoint %s" % (shape,))
    gp[1][0, 0, 1, 0] = float("nan")
    gp[3][1 % B, C - 1, 5, 5] = float("inf")
    got = ops.psp_pool_bwd(gp, base.clone())
    x = torch.zeros(shape, dtype=torch.float64, device="cuda", requires_grad=True)
    sum((Fn.adaptive_avg_pool2d(x, s) * p.double()).sum() for s, p in zip(ops.PSP_SIZES, gp)).backward()
    same_nonfinite(got, x.grad + base.double(), "pool adjoint non-finite %s" % (shape,))


# ----------------------------------------------------------------------------------------------- final
FINAL_SHAPES = [(8, 64, 240, 320, 64), (8, 64, 480, 640, 64), (1, 64, 13, 17, 22), (2, 64, 7, 5, 128),
                (1, 3, 2, 3, 1), (3, 64, 1, 1, 64)]


def final_grads(f, x):
    return [x.grad, f[0].weight.grad, f[0].bias.grad]


@pytest.mark.parametrize("shape", FINAL_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_final_backward(cuda, shape, large=False):
    B, Ci, H, W, Co = shape
    torch.manual_seed(Co)
    f = cnn.Final(Ci)
    f[0] = torch.nn.Conv2d(Ci, Co, 1)
    f = f.cuda()
    g = torch.Generator(device="cuda").manual_seed(H)
    x0 = torch.randn((B, Ci, H, W), generator=g, device="cuda") * 2
    if large:
        with torch.no_grad():
            f[0].weight.copy_(torch.eye(Co, Ci, device="cuda").reshape(Co, Ci, 1, 1))
        x0 = 80.0 * torch.sign(x0)
        x0[0, :, 0, 0] = -80.0
    x = x0.clone().requires_grad_(True)
    out = f.forward_fused(x)
    with torch.no_grad():
        assert torch.equal(out, f.forward_fused(x0))
    grad = torch.randn(out.shape, generator=g, device="cuda")
    out.backward(grad)
    refs = []
    for dtype in (torch.float64, torch.float32):
        fr = copy.deepcopy(f).to(dtype)
        xr = x0.to(dtype).requires_grad_(True)
        fr(xr).backward(grad.to(dtype))
        refs.append(final_grads(fr, xr))
    for name, a, w64, w32 in zip(["x", "weight", "bias"], final_grads(f, x), *refs):
        bound(a, w64, w32, "final %s %s" % (shape, name))


def test_final_backward_large_logits(cuda):
    test_final_backward(cuda, (2, 64, 33, 41, 64), large=True)


def test_log_softmax_bwd_nonfinite(cuda):
    g = torch.Generator(device="cuda").manual_seed(7)
    z = torch.randn((2, 64, 9, 13), generator=g, device="cuda") * 30
    z[0, :, 1, 1] = -80.0
    z[1, 5, 2, 2] = 80.0
    out = torch.log_softmax(z, 1)
    grad = torch.randn(out.shape, generator=g, device="cuda")
    grad[0, 3, 4, 4] = float("nan")
    grad[1, 0, 0, 0] = float("inf")
    grad[1, 1, 8, 12] = float("-inf")
    out[0, 0, 7, 7] = float("nan")
    want = torch.ops.aten._log_softmax_backward_data(grad, out, 1, torch.float32)
    same_nonfinite(ops.log_softmax_bwd(grad, out), want, "log_softmax backward")


# ----------------------------------------------------------------------------------------------- PSPUpsample
UP_SHAPES = [(8, 1024, 60, 80), (8, 256, 120, 160), (8, 64, 240, 320), (2, 3, 5, 7), (1, 2, 1, 4), (1, 1, 1, 1),
             (2, 2, 3, 1), (1, 3, 1, 1)]


@pytest.mark.parametrize("shape", UP_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_upsample_backward(cuda, shape):
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x0 = torch.randn(shape, generator=g, device="cuda")
    x = x0.clone().requires_grad_(True)
    y = ops.upsample_bilinear2d(x)
    assert torch.equal(y, Fn.interpolate(x0, scale_factor=2, mode="bilinear", align_corners=True))
    grad = torch.randn(y.shape, generator=g, device="cuda")
    y.backward(grad)
    refs = []
    for dtype in (torch.float64, torch.float32):
        xr = x0.to(dtype).requires_grad_(True)
        Fn.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=True).backward(grad.to(dtype))
        refs.append(xr.grad)
    bound(x.grad, *refs, "upsample %s" % (shape,))


@pytest.mark.parametrize("sizes", [((2, 3, 5, 7), (10, 14)), ((1, 2, 1, 4), (2, 8)), ((1, 2, 9, 4), (1, 1)),
                                   ((1, 1, 3, 3), (17, 2))], ids=str)
def test_upsample_bwd_nonfinite(cuda, sizes):
    shape, out_hw = sizes
    g = torch.Generator(device="cuda").manual_seed(3)
    grad = torch.randn(shape[:2] + out_hw, generator=g, device="cuda")
    grad[0, 0, 0, 0] = float("nan")
    grad[0, -1, -1, -1] = float("inf")
    grad[-1, 0, out_hw[0] // 2, out_hw[1] // 2] = float("-inf")
    x = torch.zeros(shape, device="cuda", requires_grad=True)
    Fn.interpolate(x, size=out_hw, mode="bilinear", align_corners=True).backward(grad)   # torch's float taps
    same_nonfinite(ops.upsample_bilinear2d_bwd(grad, shape[2:]), x.grad, "upsample backward non-finite %s" % (sizes,))


def test_pspupsample_forward_fused(cuda):
    torch.manual_seed(0)
    up = cnn.PSPUpsample(16, 8).cuda().train()
    x = torch.randn(2, 16, 7, 9, device="cuda")
    state = copy.deepcopy(up.state_dict())
    a = up.forward_fused(x.clone().requires_grad_(True))
    up.load_state_dict(state)
    assert torch.equal(a, up(x))


# ----------------------------------------------------------------------------------------------- determinism
def head_chain(B=2):
    torch.manual_seed(4)
    psp, up, final = make_psp(64, 128, 3), cnn.PSPUpsample(128, 64).cuda().train(), cnn.Final(64).cuda()
    params = list(psp.parameters()) + list(up.parameters()) + list(final.parameters())
    x = torch.relu(torch.randn(B, 64, 30, 40, device="cuda")).requires_grad_(True)
    grad = torch.randn(B, 64, 60, 80, device="cuda")

    def step():
        for p in params + [x]:
            p.grad = None
        final.forward_fused(up.forward_fused(psp.forward_fused(x))).backward(grad)
        return [p.grad.clone() for p in params + [x]]
    return step, params, x


def test_backward_is_deterministic_and_replays(cuda):
    with deterministic():
        step, params, x = head_chain()
        first, second = step(), step()
        assert all(torch.equal(a, b) for a, b in zip(first, second))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                step()
        torch.cuda.current_stream().wait_stream(s)
        for p in params + [x]:
            p.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            assert all(torch.equal(a, p.grad) for a, p in zip(first, params + [x]))


# ----------------------------------------------------------------------------------------------- whole network
def _item(inputs, seed=2):
    B, N = inputs["choose"].shape[0], inputs["choose"].shape[-1]
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"labels": torch.randint(0, 22, (B, N), generator=g, device="cuda", dtype=torch.int32),
            "kp_targ_ofst": torch.randn((B, N, 8, 3), generator=g, device="cuda"),
            "ctr_targ_ofst": torch.randn((B, N, 3), generator=g, device="cuda")}


def _train_step(model, inputs, item, seed=11):
    torch.manual_seed(seed)                       # the dropouts' draws
    model.zero_grad(set_to_none=True)
    loss, _ = ffb6d_loss(model(inputs), item)
    loss.backward()
    grads = {n: p.grad.clone() for n, p in model.named_parameters()}
    stats = {n: b.clone() for n, b in model.named_buffers()}
    return grads, stats


def test_ffb6d_fused_head_training_matches_torch_path(cuda, monkeypatch):
    model, inputs, _ = _network(train=True)
    item = _item(inputs)
    m_torch = copy.deepcopy(model)
    want, want_stats = _train_step(m_torch, inputs, item)
    model.fused_image_head = True
    final = model.cnn_up_stages[2][0]
    uses, real = [], cnn.Final.forward_fused

    def spy(self, x):
        out = real(self, x)
        out.retain_grad()
        uses.append((x, out))
        return out
    monkeypatch.setattr(cnn.Final, "forward_fused", spy)
    got, got_stats = _train_step(model, inputs, item)
    assert len(uses) == 2
    assert not [n for n in want if got.get(n) is None]
    # conv biases feeding a training-mode BatchNorm (PSPUpsample's conv) have an exact gradient of 0: both paths give
    # round-off there, bounded against the conv's weight gradient; every other gradient is compared with its scale
    zero = [n for n in want if n.startswith("cnn_up_stages.") and n.endswith(".conv.1.bias")]
    assert len(zero) == 3
    for n in zero:
        wscale = want[n[:-len("bias")] + "weight"].abs().max().item()
        assert max(want[n].abs().max().item(), got[n].abs().max().item()) <= 1e-3 * wscale, n
    rel = sorted((((got[n] - w).abs().max().item() / max(w.abs().max().item(), 1e-30), n)
                  for n, w in want.items() if n not in zero), reverse=True)
    print("gradient differences, fused head against torch modules: largest %s, median %.2e"
          % (rel[:5], rel[len(rel) // 2][0]))
    # both paths are fp32 with the same dropout draws; they differ by round-off in the head's forward, which can flip
    # a ReLU mask here and there downstream, and the backward through ~60 layers carries that to every gradient
    # (measured on an H100: at most 1.1e-2 of scale, in the fusion layers; the median over the parameters 3.3e-3)
    assert rel[0][0] <= 5e-2, rel[:5]
    assert rel[len(rel) // 2][0] <= 1e-2, rel[len(rel) // 2]
    for n, w in want_stats.items():
        if w.is_floating_point():
            close(got_stats[n], w, "buffer %s" % n, 1e-4)
    # the shared `final`: its gradients are the sums of its two uses'
    dz = [(o.grad - torch.exp(o) * o.grad.sum(1, keepdim=True)).double() for _, o in uses]
    want_w = sum(torch.einsum("bohw,bihw->oi", d, x.double()) for d, (x, _) in zip(dz, uses))
    close(final[0].weight.grad.reshape(64, 64), want_w, "final weight grad = sum of both uses", 1e-4)
    close(final[0].bias.grad, sum(d.sum((0, 2, 3)) for d in dz), "final bias grad", 1e-4)


def test_ffb6d_torch_path_raises_under_deterministic_mode(cuda):
    model, inputs, _ = _network(train=True)
    item = _item(inputs)
    with deterministic():
        loss, _ = ffb6d_loss(model(inputs), item)
        with pytest.raises(RuntimeError, match="deterministic"):
            loss.backward()


def test_ffb6d_fused_head_trains_deterministically(cuda):
    model, inputs, _ = _network(train=True)
    model.fused_image_head = True
    item = _item(inputs)
    with deterministic():
        runs = [_train_step(copy.deepcopy(model), inputs, item) for _ in range(2)]
    (g1, s1), (g2, s2) = runs
    assert [n for n in g1 if not torch.equal(g1[n], g2[n])] == []
    assert [n for n in s1 if not torch.equal(s1[n], s2[n])] == []
    assert all(torch.isfinite(g).all() for g in g1.values())
