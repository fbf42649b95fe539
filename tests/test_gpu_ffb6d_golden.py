"""GPU: the whole ``FFB6D`` on this package's kernels against the reference's own ``models.ffb6d.FFB6D``, forward
and one training step, through ``ffb6d_net_cases.npz`` (tests/golden/make_ffb6d_golden.py; the reference's float64
run and, as the yardstick of what float32 can reach, its float32 run).  Weights and inputs are regenerated from
seeds (oracle/net_oracle.py) and loaded through ``load_reference_checkpoint``; the network runs on the fixture's
index tensors, which ``build_ffb6d_indices`` must reproduce.

cuDNN's and cuBLAS's TF32 are switched off for this file, so that the torch parts of the network are fp32."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from ffb6d_b200 import ops
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D, load_reference_checkpoint
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_restatement import first_divergence, unit
from oracle import cpu_oracle as O, net_oracle as N
from test_gpu_cnn_train import deterministic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "ffb6d_net_cases.npz")))


@pytest.fixture(scope="module")
def data(golden):
    d = N.make_inputs()
    N.check_inputs(d, golden)
    return d


@pytest.fixture(scope="module")
def stored_idx(golden, data):
    """The reference's index tensors: the exact CPU oracle's, held to the fixture's digests."""
    idx = N.oracle_indices(data)
    N.check_indices(idx, golden)
    return idx


def network(state, **kw):
    model = FFB6D(n_classes=N.N_CLASSES, n_pts=N.N_POINTS, n_kps=N.N_KPS, **kw)
    load_reference_checkpoint(model, {"model_state": {"module." + k: v for k, v in state(model.state_dict()).items()}})
    return model.cuda()


def report(name, value):
    """Print the measured errors of this run (``pytest -rP`` shows them)."""
    print("%s: %s" % (name, json.dumps(value)))


def test_index_build_reproduces_reference_indices(cuda, data, stored_idx):
    got = build_ffb6d_indices(torch.from_numpy(data["cld"]).cuda(), torch.from_numpy(data["dpt_xyz"]).cuda())
    n = N.N_POINTS
    for i in range(4):
        assert np.array_equal(got["cld_xyz%d" % i].cpu().numpy(), data["cld"][:, :n])
        n //= 4
        assert torch.equal(got["cld_sub_idx%d" % i], got["cld_nei_idx%d" % i][:, :n])
    from conftest import frame_point_sets
    from ffb6d_b200.tables import knn_schedule
    for key, s, q, k in knn_schedule(N.N_POINTS, N.H, N.W):
        g = got[key].cpu().numpy()
        assert g.dtype == np.int32 and g.shape == stored_idx[key].shape, key
        if np.array_equal(g, stored_idx[key]):
            continue
        for b in range(len(N.SEEDS)):       # a row with exact-distance ties may differ as the tie contract allows
            ps = frame_point_sets({"cld": data["cld"][b], "dpt_xyz": data["dpt_xyz"][b]}, N.N_POINTS)
            ok, _, _, msg = O.knn_matches(ps[s][None], ps[q][None], g[b][None], stored_idx[key][b][None])
            assert ok, "%s frame %d: %s" % (key, b, msg)


def stage_bound(e32):
    """A stage's largest error (root mean square over the sampled positions, as a fraction of the stage's scale):
    5e-5, or four times the reference's own float32 error.  Round-off grows along the 60 layers, and the reference's
    float32 run is torch on the CPU.  Measured on an H100 80GB HBM3 (700 W): every stage is 1.4 to 2.1 times as far
    from float64 as that run, with the PSP head and ``final`` on the kernels or on torch's modules, in reference
    order or ``restructured`` alike (at most 2.1 times, 3.3e-5 against 1.6e-5 at ``rndla_up_stages.3``; the
    ``end_points`` 8.5e-5 against 5.2e-5).  Twice that leaves room for another cuDNN or summation order; a wiring
    edit moves a stage by its whole scale (tests/test_ffb6d_golden.py)."""
    return max(5e-5, 4 * e32)


def hooked(model, names, outputs):
    mods = dict(model.named_modules())
    return [mods[n].register_forward_hook(lambda m, i, o, n=n: outputs.__setitem__(n, o.detach()))
            for n in names if n not in N.END_POINTS]


def stages_of(outputs, out):
    """The hooked modules' outputs, the ``end_points`` and ``fused_rgb`` (the outputs of the seven ``p2r_fuse``
    layers, whichever path computed them) under the fixture's names."""
    got = dict(outputs, **{k: out[k] for k in N.END_POINTS})
    for i, t in enumerate(out["fused_rgb"]):
        got["%s_fuse_p2r_fuse_layers.%d" % (("ds", i) if i < 4 else ("up", i - 4))] = t
    return got


@pytest.mark.parametrize("restructured", [False, True], ids=["reference_order", "restructured"])
def test_eval_matches_reference(cuda, golden, data, stored_idx, monkeypatch, restructured):
    stored = N.unpack(golden, "eval", N.STAGE_SAMPLES)
    model = network(lambda sd: N.eval_tensors(sd, golden), restructured=restructured).eval()
    inputs = N.network_inputs(data, stored_idx, device="cuda")
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
    worst = {}
    for path, grad in (("kernels", False), ("torch_image_modules", True)):
        outputs = {}
        hooks = hooked(model, stored, outputs)
        with torch.set_grad_enabled(grad):
            out = model(inputs)
        for h in hooks:
            h.remove()
        assert calls == {"psp": 1, "final": 2}, (path, calls)      # the kernels ran without autograd, and only then
        got = stages_of(outputs, out)
        # psp + drop_1, final and up_3 + final are not called as stage modules when the kernels run them
        assert len(got) == (46 if grad else 43) + 3, sorted(set(stored) - set(got))
        first, w = first_divergence(got, stored, N.STAGE_SEED, N.STAGE_SAMPLES, stage_bound)
        worst[path] = w
        report("eval_restructured" if restructured else "eval", worst)
        assert first is None, "%s, restructured=%s: %s" % (path, restructured, first)


CONFIGS = {"reference_order": {}, "restructured": {"restructured": True},
           "fused_image_head": {"fused_image_head": True}}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_training_step_matches_reference(cuda, golden, data, stored_idx, config):
    model = network(N.seeded_tensors, **CONFIGS[config]).train()
    for m in model.modules():
        if isinstance(m, (torch.nn.Dropout, torch.nn.Dropout2d)):
            m.eval()                                  # the fixture's step has them off: the draws cannot be shared
    inputs = N.network_inputs(data, stored_idx, device="cuda")
    with deterministic(config == "fused_image_head"):
        out = model(inputs)
        loss, info = ffb6d_loss(out, N.targets(data, device="cuda"))
        loss.backward()
    worst = {}
    for k, want, want32 in zip(N.LOSSES, golden["train/loss"], golden["train/loss32"]):
        err = abs(info[k].item() - want)
        assert err <= max(1e-5 * abs(want), 2 * abs(float(want32) - want)), (k, info[k].item(), want, float(want32))
        worst[k] = (err / abs(want), abs(float(want32) - want) / abs(want))
    first, worst["end_points"] = first_divergence(out, N.unpack(golden, "train/out", N.STAGE_SAMPLES), N.STAGE_SEED,
                                                  N.STAGE_SAMPLES, stage_bound)
    assert first is None, first
    # gradients at the sampled positions and by norm, measured against the layer's gradient scale: at most 4x as far
    # from float64 as the reference's own float32 (a ReLU or max-pool that flips is fp32 behaviour), or 2e-3
    stored = N.unpack(golden, "train/grad", N.PARAM_SAMPLES)
    params = dict(model.named_parameters())
    assert sorted(params) == sorted(stored)
    missing = [n for n, p in params.items() if p.grad is None]
    assert not missing, missing[:10]
    scale = {}
    for name, e in stored.items():
        scale[unit(name)] = max(scale.get(unit(name), 1e-12), e["norm"])
    rows = []
    for name, e in stored.items():
        g, s = params[name].grad, scale[unit(name)]
        assert tuple(g.shape) == e["shape"], name
        err = np.linalg.norm(N.sample(g, N.GRAD_SEED + e["k"], N.PARAM_SAMPLES) - e["f64"]) / s
        e32 = e["e32norm"] / s
        nerr = abs(g.double().norm().item() - e["norm"]) / s
        rows.append((float(err), float(e32), float(nerr), e["err32"] / s, name))
    rows.sort(reverse=True)
    worst["grad"] = rows[:5]
    worst["grad_median"] = (sorted(r[0] for r in rows)[len(rows) // 2], sorted(r[1] for r in rows)[len(rows) // 2])
    report("train_" + config, worst)
    for err, e32, nerr, n32, name in rows:
        assert err <= max(2e-3, 4 * e32), "grad %s: %.3e of its layer's gradient scale at the sampled positions " \
            "(the reference's own float32: %.3e); worst: %s" % (name, err, e32, rows[:5])
        assert nerr <= max(2e-3, 4 * n32), "grad %s: its norm is %.3e of its layer's gradient scale off (the " \
            "reference's own float32 differs by %.3e over the whole tensor)" % (name, nerr, n32)
    # running statistics and the batch counters after the step
    sd = model.state_dict()
    stored = N.unpack(golden, "train/stat", N.PARAM_SAMPLES)
    assert sorted(stored) == N.running_keys(sd)
    for name, e in stored.items():
        s = max(np.abs(e["f64"]).max(), 1e-3)
        err = np.abs(N.sample(sd[name], N.STAT_SEED + e["k"], N.PARAM_SAMPLES) - e["f64"]).max() / s
        e32 = e["e32max"] / s
        # 1e-4: the bound the running statistics of the whole network are held to in tests/test_gpu_cnn_train.py
        # (measured on an H100 80GB HBM3 (700 W): 5.0e-5 at worst, the running variance of rndla_up_stages.0, taken
        # over 128 positions behind 30 fp32 layers; the reference's own float32 is 2.3e-5 off there)
        assert err <= max(1e-4, 2 * e32), "%s after the step: %.3e of scale (the reference's float32: %.3e)" % (
            name, err, e32)
    counts = [int(v) for k, v in sd.items() if k.endswith("num_batches_tracked")]
    assert counts == [1] * len(golden["train/num_batches_tracked"])
