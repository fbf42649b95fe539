"""GPU: FFB6DFusionNet (the RandLA branch + the 28 fusion layers + the heads of FFB6D.forward, models/ffb6d.py:
203-337, on this package's kernels) against a plain-torch float64 restatement of the same lines built from the
same state dict: forward values and, in training mode, the gradients of every parameter and of the image-branch
inputs.  Index tensors come from build_ffb6d_indices (itself pinned to the reference elsewhere)."""
import pytest
import torch

from ffb6d_b200.model import FFB6DFusionNet
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_b200.synthetic import make_batch
from ffb6d_restatement import TorchRef, close, unit

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
def test_fusion_net_matches_torch_restatement(cuda, train):
    B, h, w, n_pts, n_kps = 2, 120, 160, 4096, 8
    torch.manual_seed(3)
    model = FFB6DFusionNet(n_classes=5, n_pts=n_pts, n_kps=n_kps).cuda()
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():   # non-trivial BatchNorm parameters and statistics
        for m in model.modules():
            if isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
    model.train(train)
    batch = make_batch([3, 4], n_points=n_pts, h=h, w=w)
    cld = torch.from_numpy(batch["cld"]).cuda()
    xyz = torch.from_numpy(batch["dpt_xyz"]).cuda()
    inputs = build_ffb6d_indices(cld, xyz)
    inputs["choose"] = torch.from_numpy(batch["choose"]).cuda()
    inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).cuda()
    gg = torch.Generator(device="cuda").manual_seed(1)
    rgb_feats = [torch.randn(s, generator=gg, device="cuda").requires_grad_(train)
                 for s in FFB6DFusionNet.rgb_feature_shapes(B, h, w)]
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    ref = TorchRef(sd, train, n_kps)
    rgb64 = [t.detach().double().requires_grad_(train) for t in rgb_feats]
    if train:
        out = model(inputs, rgb_feats)
        want = ref.forward(inputs, rgb64)
    else:
        with torch.no_grad():
            out = model(inputs, rgb_feats)
            want = ref.forward(inputs, rgb64)
    def flat(d):
        return [(k, d[k]) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")] + \
               [("fused_rgb%d" % i, t) for i, t in enumerate(d["fused_rgb"])]

    for (k, a), (_, b) in zip(flat(out), flat(want)):
        close(a, b, "%s %s" % ("train" if train else "eval", k), 5e-5)
    if not train:
        return
    go = [torch.randn(v.shape, generator=gg, device="cuda") for _, v in flat(out)]
    sum((v * g_).sum() for (_, v), g_ in zip(flat(out), go)).backward()
    sum((v * g_.double()).sum() for (_, v), g_ in zip(flat(want), go)).backward()
    # the same composition through torch in fp32: how far plain fp32 autograd lands from the fp64 gradients.
    # (A 60-layer network with batch-statistics BatchNorm over as few as 32 positions, max-pools and ReLU kinks
    # amplifies fp32 round-off; gradient parity per LAYER is pinned at 1e-5 against the reference's own modules
    # in tests/test_gpu_train.py -- here the whole-network gradients must be as close to fp64 as torch's own.)
    ref32 = TorchRef(sd, train, n_kps, dtype=torch.float32)
    rgb32 = [t.detach().clone().requires_grad_(True) for t in rgb_feats]
    want32 = ref32.forward(inputs, rgb32)
    sum((v * g_).sum() for (_, v), g_ in zip(flat(want32), go)).backward()
    # errors are measured against the gradient scale of the parameter's LAYER (largest gradient norm among the
    # parameters of the same conv + BatchNorm unit, `unit`)
    scale_of = {}
    for name, _ in model.named_parameters():
        scale_of[unit(name)] = max(scale_of.get(unit(name), 1e-12), ref.p[name].grad.norm().item())
    report = []
    for name, prm in model.named_parameters():
        r, r32 = ref.p[name].grad, ref32.p[name].grad
        assert prm.grad is not None and r is not None, name
        nrm = scale_of[unit(name)]
        e_ours = (prm.grad.double() - r).norm().item() / nrm
        e_t32 = (r32.double() - r).norm().item() / nrm
        report.append((e_ours, e_t32, name))
    report.sort(reverse=True)
    import json
    import os
    from conftest import ROOT
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "model_grad_errors.json"), "w") as fh:
        json.dump({"worst": report[:10], "median_ours": sorted(x[0] for x in report)[len(report) // 2],
                   "median_torch_fp32": sorted(x[1] for x in report)[len(report) // 2]}, fh, indent=1)
    for e_ours, e_t32, name in report:
        assert e_ours <= max(4 * e_t32, 2e-3), "grad %s: error %.3e of its layer's gradient scale (torch fp32: %.3e); worst: %s" % (
            name, e_ours, e_t32, report[:5])
    for t, r, r32 in zip(rgb_feats, rgb64, rgb32):
        if r.grad is not None:
            nrm = max(r.grad.norm().item(), 1e-12)
            e_ours = (t.grad.double() - r.grad).norm().item() / nrm
            e_t32 = (r32.grad.double() - r.grad).norm().item() / nrm
            assert e_ours <= max(4 * e_t32, 2e-3), (e_ours, e_t32)
