"""GPU: the whole ``FFB6D`` at the size it trains at -- two 480x640 frames with 12288 points, hole pixels included
(``make_batch``) -- against its float64 restatement ``FullRef`` (tests/ffb6d_restatement.py, held to the reference's
own float64 to 1e-9 stage by stage on the CPU), run on the GPU.  The yardstick of what float32 can reach is the same
restatement in float32 on the GPU; cuDNN's and cuBLAS's TF32 are off for this file.

At this size the network runs kernels the 120x160 tests never reach: the K-lane max-pool gathers of the four sparse
r2p maps, the long-row ``choose`` gather, segment sums over runs of hundreds of hole pixels, BatchNorm reductions and
split-K weight gradients over many chunks, the PSP pooling of 60x80 maps and the upsampling adjoint at 240x320.
``test_full_size_gathers_take_the_long_row_kernels`` pins which gather kernels those are.

Full tensors are compared, not samples.  Every stage is held to two bounds, as fractions of the float64 stage's
largest magnitude: the root mean square error to max(5e-5, 4x the float32 restatement's), as
tests/test_gpu_ffb6d_golden.py holds it, and the largest element error to ``MAX_FACTOR`` times the float32
restatement's largest (measured values beside ``MAX_FACTOR``).  One neighbour set or one ``choose`` entry pointing at
the wrong pixel is reported at the stage that reads it (``test_one_wrong_index_is_reported_at_its_stage``).

On an H100 80GB HBM3 (700 W) the file takes 38 s (the first test 15 s of it: cuDNN's first launches and a profiled
training step), and torch's allocator peaks at 11.8 GB, during the training steps."""
import copy
import json
import math

import numpy as np
import pytest
import torch

from ffb6d_b200 import tables as T
from ffb6d_b200._lib import lib, LAYOUT_NCS
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_restatement import FullRef, unit
from oracle import loss_oracle
from test_gpu_cnn import _network
from test_gpu_cnn_train import deterministic
from test_gpu_deterministic import kernel_names
from test_gpu_ffb6d_golden import hooked, stages_of

pytestmark = pytest.mark.gpu

B, H, W, N_PTS, N_CLASSES, N_KPS = 2, 480, 640, 12288, 22, 8
END_POINTS = ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")
LOSSES = ("loss_rgbd_seg", "loss_kp_of", "loss_ctr_of", "loss_all")
# A stage's largest element error may be at most this many times the float32 restatement's largest error.  Measured
# on an H100 80GB HBM3 (700 W), over the whole tensors of every stage of both eval paths, reference order and
# `restructured`, and the training steps' end_points: at most 2.7 times (rndla_ds_stages.0 on the torch-modules path,
# 1.26e-6 against 4.7e-7 of its scale), the kernel path at most 1.5 times.  One wrong index moves the stage that reads
# it by 1.8e-1 (a `choose` entry) to 7.1e-1 (an r2p neighbour set) of its scale, over 1000 times the float32 error.
MAX_FACTOR = 5.0


@pytest.fixture(scope="module", autouse=True)
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def report(name, value):
    """Print the measured errors of this run (``pytest -rP`` shows them)."""
    print("%s: %s" % (name, json.dumps(value)))


# ----------------------------------------------------------------------------------------------- comparisons
def errors(got, want):
    """(root mean square, largest) of ``got - want`` over the whole tensor, as fractions of ``want``'s largest
    magnitude."""
    d = got.detach().to(want.device, torch.float64) - want
    scale = max(want.abs().max().item(), 1e-30)
    return d.norm().item() / math.sqrt(max(d.numel(), 1)) / scale, d.abs().max().item() / scale


def stage_bounds(y_rms, y_max):
    return max(5e-5, 4 * y_rms), MAX_FACTOR * y_max


def first_divergence(got, want, want32, order):
    """Walk the stages ``order`` (the order in which the reference computes them) present in ``got``; returns
    ``(message naming the first stage beyond a bound or None, rows)``, a row ``(name, rms, max, rms32, max32)``."""
    first, rows = None, []
    for name in order:
        if name not in got:
            continue
        if tuple(got[name].shape) != tuple(want[name].shape):
            return "%s: shape %s, the restatement's is %s" % (name, tuple(got[name].shape), tuple(want[name].shape)), rows
        (e_rms, e_max), (y_rms, y_max) = errors(got[name], want[name]), errors(want32[name], want[name])
        rows.append((name, e_rms, e_max, y_rms, y_max))
        b_rms, b_max = stage_bounds(y_rms, y_max)
        if first is None and not (e_rms <= b_rms and e_max <= b_max):
            first = "%s is the first stage that differs from float64: rms %.3e, largest %.3e of its scale (the float32 " \
                    "restatement's: %.3e, %.3e)" % (name, e_rms, e_max, y_rms, y_max)
    return first, rows


def summary(rows):
    """The worst stages by root mean square and by largest error, each against the float32 restatement."""
    by_rms = sorted(rows, key=lambda r: -r[1] / max(r[3], 1e-30))[:3]
    by_max = sorted(rows, key=lambda r: -r[2] / max(r[4], 1e-30))[:5]
    return {"worst_rms_ratio": [(n, "%.3e" % a, "%.3e" % c, round(a / max(c, 1e-30), 2)) for n, a, _, c, _ in by_rms],
            "worst_max_ratio": [(n, "%.3e" % b, "%.3e" % d, round(b / max(d, 1e-30), 2)) for n, _, b, _, d in by_max]}


def peak_gb():
    return round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)


# ----------------------------------------------------------------------------------------------- eval
def ref_stages(model, sd, inputs, dtype):
    """``(stages {name: output}, order)`` of FullRef's eval forward in ``dtype``."""
    ref = FullRef(model, sd, N_KPS, dtype=dtype)
    ref.trace = []
    with torch.no_grad():
        out = ref.forward(inputs, inputs["rgb"])
    got = dict(ref.trace, **{k: out[k] for k in END_POINTS})
    return got, [n for n, _ in ref.trace] + list(END_POINTS)


@pytest.fixture(scope="module")
def eval_case(cuda):
    """The eval network (running statistics of this batch), its inputs, and FullRef's stages in float64 and float32."""
    model, inputs, _ = _network(B=B, h=H, w=W, n_pts=N_PTS)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    want, order = ref_stages(model, sd, inputs, torch.float64)
    want32, _ = ref_stages(model, sd, inputs, torch.float32)
    return dict(model=model, inputs=inputs, want=want, want32=want32, order=order)


def model_stages(model, inputs, names, grad):
    outputs = {}
    hooks = hooked(model, names, outputs)
    try:
        with torch.set_grad_enabled(grad):
            out = model(inputs)
    finally:
        for h in hooks:
            h.remove()
    return stages_of(outputs, out)


def test_full_size_gathers_take_the_long_row_kernels(cuda, eval_case):
    """The dispatch of ``launch_ncs`` (csrc/gather.cu) at 480x640 with 12288 points: the four sparse r2p max-pools
    take the K-lane kernel and ``choose`` the long-row K = 1 kernel; every other gather stages its rows in shared
    memory.  If the dispatch changes, this says so before the comparisons below silently cover less."""
    long_rows = {"r2p_ds_nei_idx3": "gather_max_ncs_klane_kernel", "r2p_up_nei_idx0": "gather_max_ncs_klane_kernel",
                 "r2p_up_nei_idx1": "gather_max_ncs_klane_kernel", "r2p_up_nei_idx2": "gather_max_ncs_klane_kernel",
                 "choose": "gather1_ncs_direct_kernel"}
    staged = {"gather_max_ncs_staged_kernel", "gather1_ncs_staged_v4_kernel"}
    for op, key, C, S, Q, K in T.gather_schedule(N_PTS, H, W):
        name = lib.ffb6d_gather_kernel_name(B, C, S, Q, K, LAYOUT_NCS).decode()
        if key in long_rows:
            assert name == long_rows[key], (key, C, S, Q, K, name)
        else:
            assert name in staged, (key, C, S, Q, K, name)
    # ... and they run inside the forward and the default backward compared below
    model, inputs = eval_case["model"], eval_case["inputs"]
    with torch.no_grad():
        names = kernel_names(lambda: model(inputs))
    assert set(long_rows.values()) | staged <= names, names
    train = copy.deepcopy(model).train()
    names = kernel_names(lambda: ffb6d_loss(train(inputs), targets(inputs))[0].backward())
    assert {"gather_max_ncs_klane_kernel", "gather1_ncs_direct_kernel", "gather_max_bwd_kernel",
            "gather1_bwd_runs_kernel"} <= names, names


@pytest.mark.parametrize("restructured", [False, True], ids=["reference_order", "restructured"])
def test_eval_matches_float64(cuda, eval_case, restructured):
    """The kernel path (no autograd: PSP head and ``final`` on this package's kernels) and the torch-modules path
    (autograd on), every stage against FullRef in float64."""
    model = eval_case["model"]
    model.restructured = restructured
    measured, firsts = {}, {}
    try:
        for path, grad in (("kernels", False), ("torch_image_modules", True)):
            got = model_stages(model, eval_case["inputs"], eval_case["order"], grad)
            firsts[path], rows = first_divergence(got, eval_case["want"], eval_case["want32"], eval_case["order"])
            assert len(rows) >= 40, [r[0] for r in rows]
            measured[path] = summary(rows)
            del got
    finally:
        model.restructured = False
    report("eval_restructured" if restructured else "eval", dict(measured, peak_gb=peak_gb()))
    for path, first in firsts.items():
        assert first is None, "%s, restructured=%s: %s" % (path, restructured, first)


def far_pixel(p, S):
    """A pixel half an image away from pixel ``p`` of a map with ``S`` pixels."""
    return (int(p) + S // 2) % S


@pytest.mark.parametrize("edit,stage", [("r2p_up_nei_idx2", "up_fuse_r2p_pre_layers.2"), ("choose", "pred_rgbd_segs")])
def test_one_wrong_index_is_reported_at_its_stage(cuda, eval_case, edit, stage):
    """The kernel side reads one wrong index map; the restatement keeps the true one.  ``r2p_up_nei_idx2``: the 16
    neighbours of one query all point at one pixel half an image away; ``choose``: one point picks such a pixel.
    The first stage beyond its bound must be the one that reads the edited map."""
    inputs = dict(eval_case["inputs"])
    idx = inputs[edit].clone()
    S = T.set_size(("img", 2 if edit != "choose" else 1), N_PTS, H, W)
    if edit == "choose":
        q = idx.shape[-1] // 3
        idx[1, 0, q] = far_pixel(idx[1, 0, q], S)
    else:
        q = idx.shape[1] // 2
        idx[0, q, :] = far_pixel(idx[0, q, 0], S)
    inputs[edit] = idx
    got = model_stages(eval_case["model"], inputs, eval_case["order"], False)
    first, rows = first_divergence(got, eval_case["want"], eval_case["want32"], eval_case["order"])
    at = {r[0]: r for r in rows}[stage]
    report("edit_" + edit, {"first": first, stage: at})
    assert first is not None and first.startswith(stage + " is the first stage"), first


# ----------------------------------------------------------------------------------------------- training step
def targets(inputs, dtype=torch.float32):
    """Seeded targets: half of the points background, as a frame with objects has them."""
    rs = np.random.RandomState(7)
    labels = rs.randint(1, N_CLASSES, (B, N_PTS)).astype(np.int32)
    labels[rs.rand(B, N_PTS) < 0.5] = 0
    dev = inputs["rgb"].device
    return {"labels": torch.from_numpy(labels).to(dev),
            "kp_targ_ofst": torch.from_numpy(rs.randn(B, N_PTS, N_KPS, 3)).to(dev, dtype),
            "ctr_targ_ofst": torch.from_numpy(rs.randn(B, N_PTS, 3)).to(dev, dtype)}


def ref_train(model, sd, inputs, dtype):
    """One training step of FullRef in ``dtype``: (losses, end_points, gradients, running statistics after it)."""
    ref = FullRef(model, sd, N_KPS, train=True, dtype=dtype)
    out = ref.forward(inputs, inputs["rgb"])
    loss, info = loss_oracle.ffb6d_loss_torch(out, targets(inputs, dtype))
    loss.backward()
    grads = {k: v.grad for k, v in ref.p.items() if v.requires_grad}
    grads.update({k: v.grad for k, v in ref.cnn.named_parameters() if k.startswith("cnn_")})
    stats = dict(ref.after, **{k: v for k, v in ref.cnn.state_dict().items()
                              if k.startswith("cnn_") and k.endswith(("running_mean", "running_var"))})
    return ({k: info[k].item() for k in LOSSES}, {k: out[k].detach() for k in END_POINTS},
            {k: g.detach() for k, g in grads.items()}, {k: v.detach() for k, v in stats.items()})


@pytest.fixture(scope="module")
def train_case(cuda):
    model, inputs, _ = _network(B=B, h=H, w=W, n_pts=N_PTS, train=True)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    return dict(model=model, inputs=inputs, want=ref_train(model, sd, inputs, torch.float64),
                want32=ref_train(model, sd, inputs, torch.float32))


CONFIGS = {"reference_order": {}, "restructured": {"restructured": True},
           "fused_image_head": {"fused_image_head": True}}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_training_step_matches_float64(cuda, train_case, config):
    """One training step with the dropouts off: the loss terms, the ``end_points``, every parameter's gradient
    (against its layer's gradient scale, ``unit``) and every BatchNorm's running statistics after the step.
    ``fused_image_head`` runs under ``torch.use_deterministic_algorithms(True)``."""
    model = copy.deepcopy(train_case["model"]).train()
    for k, v in CONFIGS[config].items():
        setattr(model, k, v)
    for m in model.modules():
        if isinstance(m, (torch.nn.Dropout, torch.nn.Dropout2d)):
            m.eval()
    inputs = train_case["inputs"]
    with deterministic(config == "fused_image_head"):
        out = model(inputs)
        loss, info = ffb6d_loss(out, targets(inputs))
        loss.backward()
    (l64, ep64, g64, s64), (l32, ep32, g32, s32) = train_case["want"], train_case["want32"]
    measured = {}
    for k in LOSSES:
        err, e32 = abs(info[k].item() - l64[k]), abs(l32[k] - l64[k])
        measured[k] = ("%.3e" % (err / abs(l64[k])), "%.3e" % (e32 / abs(l64[k])))
        assert err <= max(1e-5 * abs(l64[k]), 2 * e32), (k, info[k].item(), l64[k], l32[k])
    first, rows = first_divergence(out, ep64, ep32, END_POINTS)
    measured["end_points"] = [(n, "%.3e" % a, "%.3e" % b, "%.3e" % c, "%.3e" % d) for n, a, b, c, d in rows]
    assert first is None, first
    # gradients by norm, against the layer's gradient scale: at most 4x as far from float64 as the float32
    # restatement (a ReLU or max-pool that flips is float32 behaviour), or 2e-3
    params = dict(model.named_parameters())
    assert sorted(params) == sorted(g64)
    missing = [n for n, p in params.items() if p.grad is None]
    assert not missing, missing[:10]
    scale = {}
    for name, g in g64.items():
        scale[unit(name)] = max(scale.get(unit(name), 1e-12), g.norm().item())
    rows = []
    for name, g in g64.items():
        s = scale[unit(name)]
        err = (params[name].grad.double() - g).norm().item() / s
        e32 = (g32[name].double() - g).norm().item() / s
        rows.append((err, e32, name))
    rows.sort(reverse=True)
    measured["grad"] = [("%.3e" % a, "%.3e" % b, n) for a, b, n in rows[:5]]
    measured["grad_median"] = ("%.3e" % sorted(r[0] for r in rows)[len(rows) // 2],
                               "%.3e" % sorted(r[1] for r in rows)[len(rows) // 2])
    # running statistics after the step: largest error over the whole tensor against its scale
    sd = model.state_dict()
    assert sorted(k for k in sd if k.endswith(("running_mean", "running_var"))) == sorted(s64)
    srows = []
    for name, want in s64.items():
        s = max(want.abs().max().item(), 1e-3)
        err = (sd[name].double() - want).abs().max().item() / s
        e32 = (s32[name].double() - want).abs().max().item() / s
        srows.append((err, e32, name))
    srows.sort(reverse=True)
    measured["stat"] = [("%.3e" % a, "%.3e" % b, n) for a, b, n in srows[:3]]
    report("train_" + config, dict(measured, peak_gb=peak_gb()))
    for err, e32, name in rows:
        assert err <= max(2e-3, 4 * e32), "grad %s: %.3e of its layer's gradient scale (the float32 restatement: " \
            "%.3e); worst: %s" % (name, err, e32, rows[:5])
    for err, e32, name in srows:
        assert err <= max(1e-4, 2 * e32), "%s after the step: %.3e of scale (the float32 restatement: %.3e)" % (
            name, err, e32)
    assert all(int(v) == 1 for k, v in sd.items() if k.endswith("num_batches_tracked"))
