#!/usr/bin/env python
"""Generate tests/golden/ffb6d_net_cases.npz by running the reference's own ``models.ffb6d.FFB6D`` on the CPU: the
whole network, forward and one training step.

Source of truth: the reference's ``FFB6D`` (constructed as ``make_cnn_golden.reference_ffb6d`` constructs it), its
compiled KNN (``oracle/_ref/libknn_ref.so``) for the 22 index tensors of each frame, and its models/loss.py combined
as train_ycb.py:237-250 combines it.  Nothing of the reference is copied: the weights, the image, the clouds and
the targets are regenerated from seeds (``oracle/net_oracle.py``), and only the reference's index tensors and
outputs are stored.

Stored (``n_classes=22, n_kps=8``, two 120x160 frames with 4096 points):

* ``digest/<input>``: sha256 of every regenerated input; ``idx_sha256/<key>``: sha256 of each of
  the 22 index tensors ``[2,Q,K]`` int32 (the tests recompute them with the exact CPU oracle).
* ``eval/*``: eval mode, with the running statistics of this batch (``eval/running``, float32: one training-mode
  forward of the reference in float64 with every momentum at 1).  The outputs of ``cnn_pre_stages``, every
  ``cnn_ds_stages[j]`` / ``cnn_up_stages[j]`` (the stage containers are hooked, so the shared ``final`` is seen
  once at stage 2 and once, behind ``up_3``, at stage 3), ``rndla_pre_stages``, every
  ``rndla_ds_stages[i]`` / ``rndla_up_stages[i]`` and all 28 fusion layers, in the order the reference computes
  them, then the three ``end_points``; up to 512 sampled values of each.
* ``train/*``: one training step with every ``Dropout`` / ``Dropout2d`` left in eval mode (two implementations
  cannot share dropout draws).  ``train/loss``: the three loss terms and their weighted sum; ``train/out``: the
  ``end_points``; ``train/grad``: the gradient of every parameter (norm and up to 48 sampled values);
  ``train/stat``: every BatchNorm's ``running_mean`` / ``running_var`` after the step; ``train/num_batches_tracked``.

Every group holds the reference's float64 run (``f64``) and how far its float32 run is from it (``err32``: the norm
of their difference over the whole tensor; ``e32max`` / ``e32norm``: the largest difference and the norm of the
differences at the sampled positions): how close to float64 the reference's own arithmetic gets.

Run:  python tests/golden/make_ffb6d_golden.py      (needs the reference's sources; rewrites ffb6d_net_cases.npz)
"""
import io
import os
import sys
import warnings
import zipfile

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, HERE]
from oracle import net_oracle as N, ref_loader as R                 # noqa: E402
from ffb6d_b200.schedule import knn_schedule                        # noqa: E402
from make_golden import point_sets                                  # noqa: E402
from make_cnn_golden import reference_ffb6d                         # noqa: E402
from make_loss_golden import reference_loss_module                  # noqa: E402

OUT = os.path.join(HERE, "ffb6d_net_cases.npz")
STAGES = (["cnn_pre_stages", "rndla_pre_stages"]
          + ["%s_stages.%d" % (b, j) for b in ("cnn_ds", "cnn_up", "rndla_ds", "rndla_up") for j in range(4)]
          + ["%s_fuse_%s_%s_layers.%d" % (t, d, k, i) for t, n in (("ds", 4), ("up", 3)) for i in range(n)
             for d in ("p2r", "r2p") for k in ("pre", "fuse")])


def reference_indices(data):
    idx = {}
    for b in range(len(N.SEEDS)):
        ps = point_sets({"cld": data["cld"][b], "dpt_xyz": data["dpt_xyz"][b]}, N.N_POINTS)
        for key, s, q, k in knn_schedule(N.N_POINTS, N.H, N.W):
            idx.setdefault(key, []).append(R.knn_search(ps[s][None], ps[q][None], k, omp=False)[0])
    return {k: np.stack(v).astype(np.int32) for k, v in idx.items()}


def prepare(net, state, data, idx, dtype, train):
    net = net.to(dtype)
    net.load_state_dict({k: v.to(dtype) if v.dtype.is_floating_point else v for k, v in state.items()}, strict=True)
    net.train(train)
    for m in net.modules():
        if isinstance(m, (nn.Dropout, nn.Dropout2d)):
            m.eval()
    return net, N.network_inputs(data, idx, dtype=dtype, index_dtype=torch.int64)


def batch_statistics(data, idx):
    """Every BatchNorm's statistics of this batch, float32, end to end in the order of their sorted keys: one
    training-mode forward of the reference (float64) with every momentum at 1."""
    net = reference_ffb6d()
    net, inp = prepare(net, N.seeded_tensors(net.state_dict()), data, idx, torch.float64, True)
    for m in net.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            m.momentum = 1.0
    with torch.no_grad():
        net(inp)
    sd = net.state_dict()
    return np.concatenate([sd[k].numpy().reshape(-1) for k in N.running_keys(sd)]).astype(np.float32)


def run(net, state, data, idx, dtype, train):
    """One run of the reference: ``(stages [(name, array)], end_points, losses, grads, stats)``."""
    net, inp = prepare(net, state(net.state_dict()), data, idx, dtype, train)
    mods = dict(net.named_modules())
    stages = []
    hooks = [mods[name].register_forward_hook(
        lambda m, i, o, name=name: stages.append((name, o.detach().clone().numpy()))) for name in STAGES]
    with torch.set_grad_enabled(train):
        ep = net(inp)
    for h in hooks:
        h.remove()
    assert sorted(n for n, _ in stages) == sorted(STAGES)
    out = {k: ep[k].detach().numpy() for k in N.END_POINTS}
    if not train:
        return stages, out, None, None, None
    ns = reference_loss_module()
    item = N.targets(data, dtype=dtype)
    labels = item["labels"].long()
    loss_rgbd_seg = ns["FocalLoss"](gamma=2)(ep["pred_rgbd_segs"], labels.view(-1)).sum()
    loss_kp_of = ns["OFLoss"]()(ep["pred_kp_ofs"], item["kp_targ_ofst"], labels).sum()
    loss_ctr_of = ns["OFLoss"]()(ep["pred_ctr_ofs"], item["ctr_targ_ofst"], labels).sum()
    loss = sum([ls * w for ls, w in [(loss_rgbd_seg, 2.0), (loss_kp_of, 1.0), (loss_ctr_of, 1.0)]])
    loss.backward()
    losses = np.array([t.item() for t in (loss_rgbd_seg, loss_kp_of, loss_ctr_of, loss)], np.float64)
    missing = [n for n, p in net.named_parameters() if p.grad is None]
    assert not missing, missing
    grads = [(n, p.grad.numpy()) for n, p in net.named_parameters()]
    sd = net.state_dict()
    stats = [(k, v.numpy()) for k, v in sd.items() if k.endswith(("running_mean", "running_var"))]
    nbt = np.array([int(v) for k, v in sd.items() if k.endswith("num_batches_tracked")], np.int64)
    return stages, out, losses, grads, (stats, nbt)


def both(state, data, idx, train):
    torch.manual_seed(0)
    a = run(reference_ffb6d(), state, data, idx, torch.float64, train)
    b = run(reference_ffb6d(), state, data, idx, torch.float32, train)
    return a, b


def triples(a, b):
    assert [n for n, _ in a] == [n for n, _ in b]
    return [(n, x, y) for (n, x), (_, y) in zip(a, b)]


def show(group, items):
    for name, a, _ in items:
        print("%s %s: %s, %d values, scale %.3g" % (group, name, a.shape, a.size, np.abs(a).max()))


def main():
    if not R.reference_sources_present():
        raise SystemExit("needs the reference's sources (FFB6D_REFERENCE)")
    R.build_ref()
    warnings.simplefilter("ignore")                # F.upsample, the implicit LogSoftmax dim, _Loss(size_average)
    data = N.make_inputs()
    idx = reference_indices(data)
    out = {"digest/" + k: np.array(N.sha(data[k])) for k in N.INPUT_KEYS}
    out.update({"idx_sha256/" + k: np.array(N.sha(v)) for k, v in idx.items()})

    out["eval/running"] = batch_statistics(data, idx)
    (st64, ep64, _, _, _), (st32, ep32, _, _, _) = both(lambda sd: N.eval_tensors(sd, out), data, idx, False)
    items = triples(st64 + [(k, ep64[k]) for k in N.END_POINTS], st32 + [(k, ep32[k]) for k in N.END_POINTS])
    show("eval", items)
    out.update(N.pack("eval", items, N.STAGE_SEED, N.STAGE_SAMPLES))

    (_, ep64, l64, g64, (s64, nbt)), (_, ep32, l32, g32, (s32, nbt32)) = both(N.seeded_tensors, data, idx, True)
    assert np.array_equal(nbt, nbt32)
    out["train/loss"], out["train/loss32"] = l64, l32.astype(np.float32)
    out["train/num_batches_tracked"] = nbt
    print("train losses", dict(zip(N.LOSSES, l64)), "float32 run", l32)
    items = triples([(k, ep64[k]) for k in N.END_POINTS], [(k, ep32[k]) for k in N.END_POINTS])
    show("train", items)
    out.update(N.pack("train/out", items, N.STAGE_SEED, N.STAGE_SAMPLES))
    items = triples(g64, g32)
    show("grad", items)
    out.update(N.pack("train/grad", items, N.GRAD_SEED, N.PARAM_SAMPLES))
    out.update(N.pack("train/stat", triples(s64, s32), N.STAT_SEED, N.PARAM_SAMPLES))

    # fixed member order and timestamps, so the file is reproducible byte for byte
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(out[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
