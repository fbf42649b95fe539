"""GPU: the PSP-head kernels (pyramid pooling, the restructured bottleneck, 1x1 conv + log-softmax) against float64
torch in the reference's order of operations, and the whole ``FFB6D`` (image branch included) against a float64
restatement built from the same state dict; a training step through the image branch.

cuDNN's and cuBLAS's TF32 are switched off for this file (fixture ``no_tf32``), so that the torch parts of the
network are fp32 and the float64 comparisons measure the kernels."""
import copy

import pytest
import torch
import torch.nn.functional as Fn

from ffb6d_b200 import cnn, ops
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_b200.synthetic import make_batch
from test_gpu_model import TorchRef, close

pytestmark = pytest.mark.gpu
TOL = 1e-5


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def same_nonfinite(got, want, what):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    for f in (torch.isnan, torch.isposinf, torch.isneginf):
        a, b = f(got), f(want)
        assert torch.equal(a, b), "%s: %s at %d positions, torch at %d" % (what, f.__name__, int(a.sum()), int(b.sum()))
    fin = torch.isfinite(want)
    if fin.any():
        close(got[fin], want[fin], what + " (finite part)", TOL)


# ----------------------------------------------------------------------------------------------- (a) pooling
POOL_SHAPES = [(8, 512, 60, 80), (2, 7, 13, 17), (1, 5, 4, 5), (3, 2, 1, 1), (1, 3, 6, 1), (1, 4, 11, 23),
               (1, 2, 1024, 7)]


@pytest.mark.parametrize("shape", POOL_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_psp_pool(cuda, shape):
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x = torch.randn(shape, generator=g, device="cuda") + 0.3
    got = ops.psp_pool(x)
    for s, p in zip(ops.PSP_SIZES, got):
        close(p, Fn.adaptive_avg_pool2d(x.double(), s), "pool %s s=%d" % (shape, s), TOL)


def test_psp_pool_nonfinite(cuda):
    x = torch.randn(2, 3, 13, 17, device="cuda")
    x[0, 0, 5, 5] = float("nan")
    x[0, 1, 12, 16] = float("inf")
    x[1, 2, 0, 0] = float("-inf")
    x[1, 0, 3, 3], x[1, 0, 3, 4] = float("inf"), float("-inf")
    for s, p in zip(ops.PSP_SIZES, ops.psp_pool(x)):
        same_nonfinite(p, Fn.adaptive_avg_pool2d(x.double(), s), "pool s=%d" % s)


# ----------------------------------------------------------------------------------------------- (b) bottleneck
def make_psp(C, Co, seed):
    torch.manual_seed(seed)
    m = cnn.PSPModule(C, Co).cuda().eval()
    with torch.no_grad():
        m.bottleneck.bias.normal_(0, 0.5)
    return m


def psp_kernels(m, x):
    w = ops.psp_pack([st[1].weight for st in m.stages], m.bottleneck.weight, m.bottleneck.bias)
    return ops.psp_bottleneck(x, ops.psp_pool(x), w)


BOTTLE_SHAPES = [(8, 512, 60, 80, 1024), (1, 512, 60, 80, 1024), (2, 16, 13, 17, 40), (1, 8, 4, 5, 130),
                 (2, 33, 7, 9, 64), (1, 4, 1, 1, 3), (1, 12, 5, 2, 200), (3, 64, 15, 20, 256)]


@pytest.mark.parametrize("shape", BOTTLE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_psp_bottleneck(cuda, shape):
    B, C, H, W, Co = shape
    m = make_psp(C, Co, 1)
    g = torch.Generator(device="cuda").manual_seed(H * W)
    x = torch.relu(torch.randn((B, C, H, W), generator=g, device="cuda"))     # post-ReLU, as layer4's output
    with torch.no_grad():
        got = psp_kernels(m, x)
        want = copy.deepcopy(m).double()(x.double())
        via_module = m.forward_fused(x)
    close(got, want, "bottleneck %s" % (shape,), TOL)
    assert torch.equal(got, via_module)


def test_psp_bottleneck_nonfinite(cuda):
    m = make_psp(16, 40, 2)
    x = torch.relu(torch.randn(3, 16, 13, 17, device="cuda"))
    x[0, 3, 4, 4] = float("nan")
    x[1, 0, 12, 16] = float("inf")
    with torch.no_grad():
        got = psp_kernels(m, x)
        want = copy.deepcopy(m).double()(x.double())
    same_nonfinite(got, want, "bottleneck")
    assert torch.isfinite(got[2]).all()


# ----------------------------------------------------------------------------------------------- (c) final
def make_final(Ci, Co, seed):
    torch.manual_seed(seed)
    conv = torch.nn.Conv2d(Ci, Co, 1).cuda()
    return conv.weight.detach(), conv.bias.detach()


def want_final(x, w, b):
    return torch.log_softmax(Fn.conv2d(x.double(), w.double(), b.double()), dim=1)


LSM_SHAPES = [(8, 64, 240, 320, 64), (2, 64, 480, 640, 64), (1, 64, 13, 17, 22), (2, 64, 7, 5, 128),
              (1, 3, 2, 3, 1), (1, 100, 9, 11, 2), (3, 64, 1, 1, 64)]


@pytest.mark.parametrize("shape", LSM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_conv1x1_log_softmax(cuda, shape):
    B, Ci, H, W, Co = shape
    w, b = make_final(Ci, Co, Co)
    x = torch.randn((B, Ci, H, W), generator=torch.Generator(device="cuda").manual_seed(H), device="cuda") * 2
    close(ops.conv1x1_log_softmax(x, w, b), want_final(x, w, b), "final %s" % (shape,), TOL)


def test_conv1x1_log_softmax_large_logits(cuda):
    g = torch.Generator(device="cuda").manual_seed(4)
    w = torch.eye(64, device="cuda").reshape(64, 64, 1, 1)
    b = torch.randn(64, generator=g, device="cuda") * 0.1
    x = 80.0 * torch.sign(torch.randn((2, 64, 33, 41), generator=g, device="cuda"))
    x[0, :, 0, 0] = -80.0                                            # every channel at the floor
    x[1, 5, 1, 1], x[1, :5, 1, 1], x[1, 6:, 1, 1] = 80.0, -80.0, -80.0  # one channel alone at the top
    close(ops.conv1x1_log_softmax(x, w, b), want_final(x, w, b), "final +-80", TOL)
    w2, b2 = make_final(64, 64, 9)
    x2 = torch.randn((1, 64, 20, 30), generator=g, device="cuda") * 40
    close(ops.conv1x1_log_softmax(x2, w2, b2), want_final(x2, w2, b2), "final large random logits", TOL)


def test_conv1x1_log_softmax_nonfinite(cuda):
    w, b = make_final(64, 64, 3)
    x = torch.randn(2, 64, 13, 17, device="cuda")
    x[0, 7, 2, 3] = float("nan")
    x[0, 0, 5, 5] = float("inf")
    x[1, 63, 12, 16] = float("-inf")
    got = ops.conv1x1_log_softmax(x, w, b)
    same_nonfinite(got, want_final(x, w, b), "final")
    assert int(torch.isnan(got).any(dim=1).sum()) == 3


def test_final_module_fused_matches(cuda):
    f = cnn.Final(64).cuda()
    x = torch.randn(2, 64, 30, 40, device="cuda")
    with torch.no_grad():
        close(f.forward_fused(x), copy.deepcopy(f).double()(x.double()), "Final.forward_fused", TOL)


# ----------------------------------------------------------------------------------------------- whole network
class FullRef(TorchRef):
    """TorchRef with the image branch: float64 copies of the model's own ``cnn_*`` torch modules, run where
    models/ffb6d.py runs them (the reference's order of operations)."""

    def __init__(self, model, sd, n_kps):
        super().__init__(sd, False, n_kps)
        m64 = copy.deepcopy(model).double().eval()
        self.pre, self.ds, self.up = m64.cnn_pre_stages, m64.cnn_ds_stages, m64.cnn_up_stages

    def forward(self, inp, rgb):
        with torch.no_grad():
            p_emb = self.rconv("rndla_pre_stages", inp["cld_rgb_nrm"].to(self.dtype)).unsqueeze(3)
            rgb_emb = self.pre(rgb.double())
            ds_emb, fused = [], []
            for i in range(4):
                rgb0 = self.ds[i](rgb_emb)
                f_enc = self.block("rndla_ds_stages.%d" % i, p_emb, inp["cld_xyz%d" % i].to(self.dtype),
                                   inp["cld_nei_idx%d" % i])
                p0 = self.random_sample(f_enc, inp["cld_sub_idx%d" % i])
                if i == 0:
                    ds_emb.append(f_enc)
                rgb_emb, p_emb = self.fuse("ds", i, rgb0, p0, inp["p2r_ds_nei_idx%d" % i], inp["r2p_ds_nei_idx%d" % i])
                ds_emb.append(p_emb)
                fused.append(rgb_emb)
            for i in range(3):
                rgb0 = self.up[i](rgb_emb)
                f_interp = self.nearest(p_emb, inp["cld_interp_idx%d" % (3 - i)])
                p0 = self.rconv("rndla_up_stages.%d" % i, torch.cat([ds_emb[-i - 2], f_interp], 1))
                rgb_emb, p_emb = self.fuse("up", i, rgb0, p0, inp["p2r_up_nei_idx%d" % i], inp["r2p_up_nei_idx%d" % i])
                fused.append(rgb_emb)
            f_interp = self.nearest(p_emb, inp["cld_interp_idx0"])
            p_emb = self.rconv("rndla_up_stages.3", torch.cat([ds_emb[0], f_interp], 1)).squeeze(-1)
            rgb = self.up[3](rgb_emb)
            bs, di = rgb.shape[0], rgb.shape[1]
            rgb_c = torch.gather(rgb.view(bs, di, -1), 2, inp["choose"].expand(-1, di, -1).long())
            x0 = torch.cat([rgb_c, p_emb], 1)
            outs = []
            for head in ("rgbd_seg_layer", "kp_ofst_layer", "ctr_ofst_layer"):
                x = x0
                for j in range(3):
                    x = self.conv("%s.%d" % (head, j), x, "normlayer", 1e-5, "relu")
                outs.append(self.conv("%s.3" % head, x, "normlayer", 1e-5, None))
        segs, kp, ctr = outs
        kp = kp.view(bs, self.n_kps, 3, -1).permute(0, 1, 3, 2).contiguous()
        ctr = ctr.view(bs, 1, 3, -1).permute(0, 1, 3, 2).contiguous()
        return {"pred_rgbd_segs": segs, "pred_kp_ofs": kp, "pred_ctr_ofs": ctr, "fused_rgb": fused}


def _network(B=2, h=120, w=160, n_pts=4096, seed=3, train=False):
    torch.manual_seed(seed)
    model = FFB6D(n_classes=22, n_pts=n_pts, n_kps=8).cuda()
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
        model.cnn_ds_stages[3][0].bottleneck.bias.normal_(0, 0.1)
    batch = make_batch(list(range(3, 3 + B)), n_points=n_pts, h=h, w=w)
    inputs = build_ffb6d_indices(torch.from_numpy(batch["cld"]).cuda(), torch.from_numpy(batch["dpt_xyz"]).cuda())
    inputs["choose"] = torch.from_numpy(batch["choose"]).cuda()
    inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).cuda()
    gg = torch.Generator(device="cuda").manual_seed(1)
    inputs["rgb"] = torch.rand((B, 3, h, w), generator=gg, device="cuda") * 2 - 1
    if not train:
        # running statistics of this batch (as a trained network has them for its data): without them the 40-layer
        # trunk and the fusion stages grow activations to 1e4 and fp32 round-off with them, in torch as here
        bns = [m for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]
        saved = [m.momentum for m in bns]
        for m in bns:
            m.momentum = 1.0
        model.train()
        with torch.no_grad():
            model(inputs)
        for m, mo in zip(bns, saved):
            m.momentum = mo
    model.train(train)
    return model, inputs, batch


def test_ffb6d_eval_matches_float64_restatement(cuda, monkeypatch):
    model, inputs, _ = _network()
    calls = {"psp": 0, "final": 0}
    real_psp, real_final = ops.psp_bottleneck, ops.conv1x1_log_softmax

    def spy_psp(*a, **k):
        calls["psp"] += 1
        return real_psp(*a, **k)

    def spy_final(*a, **k):
        calls["final"] += 1
        return real_final(*a, **k)
    monkeypatch.setattr(ops, "psp_bottleneck", spy_psp)
    monkeypatch.setattr(ops, "conv1x1_log_softmax", spy_final)
    with torch.no_grad():
        out = model(inputs)
    assert calls == {"psp": 1, "final": 2}, calls
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    ref = FullRef(model, sd, 8)
    want = ref.forward(inputs, inputs["rgb"])
    # the eval path without the kernels (autograd on): the image branch on its torch modules, in fp32
    with torch.enable_grad():
        out_t = model(inputs)
    assert calls == {"psp": 1, "final": 2}
    names = ["pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs"] + ["fused_rgb%d" % i for i in range(7)]

    def flat(d):
        return [d[k] for k in names[:3]] + list(d["fused_rgb"])
    for k, a, t32, b in zip(names, flat(out), flat(out_t), flat(want)):
        # within 5e-5 of the output's scale, or at most twice as far from fp64 as the same network on torch's modules
        scale = b.abs().max().item()
        e_ours = (a.double() - b).abs().max().item() / scale
        e_t32 = (t32.detach().double() - b).abs().max().item() / scale
        assert e_ours <= max(5e-5, 2 * e_t32), "FFB6D eval %s: %.2e of scale (torch modules in fp32: %.2e)" % (
            k, e_ours, e_t32)


def test_ffb6d_training_step(cuda):
    model, inputs, batch = _network(train=True)
    final_conv = model.cnn_up_stages[2][0][0]
    uses = []

    def hook(mod, inp, out):
        out.retain_grad()
        uses.append((inp[0], out))
    hd = final_conv.register_forward_hook(hook)
    out = model(inputs)
    hd.remove()
    assert len(uses) == 2
    B, N = inputs["choose"].shape[0], inputs["choose"].shape[-1]
    g = torch.Generator(device="cuda").manual_seed(2)
    item = {"labels": torch.randint(0, 22, (B, N), generator=g, device="cuda", dtype=torch.int32),
            "kp_targ_ofst": torch.randn((B, N, 8, 3), generator=g, device="cuda"),
            "ctr_targ_ofst": torch.randn((B, N, 3), generator=g, device="cuda")}
    loss, _ = ffb6d_loss(out, item)
    loss.backward()
    missing = [n for n, p in model.named_parameters() if p.grad is None]
    assert not missing, missing[:10]
    bad = [n for n, p in model.named_parameters() if not torch.isfinite(p.grad).all()]
    assert not bad, bad[:10]
    assert all(p.grad.abs().sum() > 0 for n, p in model.named_parameters() if n.startswith("cnn_") and "bias" not in n)
    # the shared `final` conv: its weight gradient is the sum of the gradients of its two uses
    want = sum(torch.einsum("bohw,bihw->oi", o.grad.double(), x.double()) for x, o in uses)
    close(final_conv.weight.grad.reshape(64, 64), want, "final weight grad = sum of both uses", 1e-4)
    close(final_conv.bias.grad, sum(o.grad.double().sum((0, 2, 3)) for _, o in uses), "final bias grad", 1e-4)
