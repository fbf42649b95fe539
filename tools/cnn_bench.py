#!/usr/bin/env python
"""Time FFB6D's image branch on one GPU at 480x640 (B = 1 and B = 8), CUDA-graph replays timed with events:

* ``psp`` / ``final240`` / ``final480``: the PSP block (PSPModule + drop_1 in eval) and the two uses of ``final``,
  torch's modules (cuDNN at torch's defaults) against this package's kernels, with each kernel's fraction of the HBM
  roofline from its algorithmic bytes (inputs read once, outputs written once; 3.35 TB/s);
* ``ffb6d_eval``: the whole ``FFB6D`` eval forward (kernels on the PSP head);
* ``train_step``: forward + ``ffb6d_loss`` + backward in training mode at BASELINE config 3's shape (LineMOD:
  2 classes, B = 8, 12288 points; the image branch runs its torch modules in training).

Prints one JSON line per measurement.  Usage: python tools/cnn_bench.py [--iters 20] [--batches 1,8] [--no-train]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ffb6d_b200 import cnn, ops                                        # noqa: E402
from ffb6d_b200.loss import ffb6d_loss                                 # noqa: E402
from ffb6d_b200.model import FFB6D                                     # noqa: E402
from ffb6d_b200.schedule import build_ffb6d_indices                    # noqa: E402
from ffb6d_b200.synthetic import make_batch                            # noqa: E402

HBM = 3.35e12


def graph_time(fn, iters, warmup=3):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    return times[len(times) // 2], times[0]


def eager_time(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    return times[len(times) // 2], times[0]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def head_blocks(B, iters):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    pre, ds, up = cnn.image_branch()
    psp, final = ds[3].to(dev).eval(), up[2][0].to(dev).eval()
    x = torch.relu(torch.randn(B, 512, 60, 80, device=dev))
    y240 = torch.randn(B, 64, 240, 320, device=dev)
    y480 = torch.randn(B, 64, 480, 640, device=dev)
    with torch.no_grad():
        cases = [("psp", lambda: psp(x), lambda: psp[0].forward_fused(x),
                  4 * B * (512 * 4800 + 1024 * 4800 + 50 * 1024)),     # read f, write out (+ the prior table)
                 ("final240", lambda: final(y240), lambda: final.forward_fused(y240), 4 * B * 2 * 64 * 240 * 320),
                 ("final480", lambda: final(y480), lambda: final.forward_fused(y480), 4 * B * 2 * 64 * 480 * 640)]
        for name, ref, ker, nbytes in cases:
            t_ref, t_ref_min = graph_time(ref, iters)
            t_ker, t_ker_min = graph_time(ker, iters)
            emit(what=name, B=B, torch_ms=round(t_ref, 4), kernels_ms=round(t_ker, 4),
                 kernels_min_ms=round(t_ker_min, 4), speedup=round(t_ref / t_ker, 3),
                 algorithmic_MB=round(nbytes / 1e6, 2), hbm_roofline_fraction=round(nbytes / HBM / (t_ker * 1e-3), 3))
        # the pooling alone, against its HBM floor (one read of f)
        t, _ = graph_time(lambda: ops.psp_pool(x), iters)
        nb = 4 * B * 512 * (4800 + 50)
        emit(what="psp_pool", B=B, kernels_ms=round(t, 4), hbm_roofline_fraction=round(nb / HBM / (t * 1e-3), 3))


def network(B, n_pts, train, n_classes=22):
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = FFB6D(n_classes=n_classes, n_pts=n_pts, n_kps=8).to(dev).train(train)
    batch = make_batch(list(range(B)), n_points=n_pts)
    inputs = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(dev), torch.from_numpy(batch["dpt_xyz"]).to(dev))
    inputs["choose"] = torch.from_numpy(batch["choose"]).to(dev)
    inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(dev)
    inputs["rgb"] = torch.rand(B, 3, 480, 640, device=dev) * 2 - 1
    return model, inputs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--no-train", action="store_true")
    a = ap.parse_args()
    emit(gpu=torch.cuda.get_device_name(0), cudnn_allow_tf32=torch.backends.cudnn.allow_tf32)
    for B in [int(b) for b in a.batches.split(",")]:
        head_blocks(B, a.iters)
        model, inputs = network(B, 12288, False)
        with torch.no_grad():
            t, tmin = eager_time(lambda: model(inputs), max(3, a.iters // 4))
        emit(what="ffb6d_eval", B=B, ms=round(t, 3), min_ms=round(tmin, 3))
        del model, inputs
        torch.cuda.empty_cache()
    if not a.no_train:
        B = 8
        model, inputs = network(B, 12288, True, n_classes=2)       # config 3: LineMOD-shaped, 8 frames
        N = inputs["choose"].shape[-1]
        item = {"labels": torch.randint(0, 2, (B, N), device="cuda", dtype=torch.int32),
                "kp_targ_ofst": torch.randn(B, N, 8, 3, device="cuda"),
                "ctr_targ_ofst": torch.randn(B, N, 3, device="cuda")}

        def step():
            model.zero_grad(set_to_none=True)
            loss, _ = ffb6d_loss(model(inputs), item)
            loss.backward()
        t, tmin = eager_time(step, max(3, a.iters // 4))
        emit(what="train_step", B=B, n_pts=12288, ms=round(t, 3), min_ms=round(tmin, 3))


if __name__ == "__main__":
    main()
