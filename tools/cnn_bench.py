#!/usr/bin/env python
"""Time FFB6D's image branch on one GPU at 480x640 (B = 1 and B = 8), CUDA-graph replays timed with events:

* ``psp`` / ``final240`` / ``final480``: the PSP block (PSPModule + drop_1 in eval) and the two uses of ``final``,
  torch's modules (cuDNN at torch's defaults) against this package's kernels, with each kernel's fraction of the HBM
  roofline from its algorithmic bytes (inputs read once, outputs written once; 3.35 TB/s);
* ``ffb6d_eval``: the whole ``FFB6D`` eval forward (kernels on the PSP head);
* ``train_step``: forward + ``ffb6d_loss`` + backward in training mode at BASELINE config 3's shape (LineMOD:
  2 classes, B = 8, 12288 points; the image branch runs its torch modules in training).

With ``--train-arms`` it measures the training path instead (DESIGN.md §4.18), every arm alternated within each of
``--reps`` repetitions, and prints the card's name and power limit first:

* ``psp_train`` (B = 1, 8) and ``final240_train`` / ``final480_train`` (B = 8): forward + backward of the PSP block
  and of both uses of ``final``, torch's modules against ``forward_fused`` (median of ``--iters`` graph replays), and
  the peak memory one eager call of each allocates above what was allocated before it;
* ``train_step_arm``: the config-3 step with ``fused_image_head`` off, on, and on under
  ``torch.use_deterministic_algorithms(True)`` (median of max(3, ``--iters`` // 4) eager steps), each with
  ``torch.cuda.max_memory_allocated``;
* with ``--profile``, the CUDA time per kernel name of one step of each setting (``torch.profiler``).

Prints one JSON line per measurement.  Usage: python tools/cnn_bench.py [--iters 20] [--batches 1,8] [--no-train]
[--train-arms [--reps 3] [--profile]]
"""
import argparse
import contextlib
import json
import os
import subprocess
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


def card():
    """The card's name and its power limit (read-only query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "unavailable (%s)" % e
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def head_train_cases(B):
    """(name, torch-module step, kernel step) of the PSP block and both uses of ``final``, forward + backward."""
    dev = torch.device("cuda")
    torch.manual_seed(0)
    pre, ds, up = cnn.image_branch()
    psp, final = ds[3][0].to(dev).train(), up[2][0].to(dev).train()
    x = torch.relu(torch.randn(B, 512, 60, 80, device=dev)).requires_grad_(True)
    g = torch.randn(B, 1024, 60, 80, device=dev)
    y240 = torch.randn(B, 64, 240, 320, device=dev).requires_grad_(True)
    y480 = torch.randn(B, 64, 480, 640, device=dev).requires_grad_(True)
    g240, g480 = torch.randn_like(y240), torch.randn_like(y480)
    params = list(psp.parameters()) + list(final.parameters())

    def run(f):
        def step():
            for p in params + [x, y240, y480]:
                p.grad = None
            f()
        return step
    cases = [("psp_train", run(lambda: psp(x).backward(g)), run(lambda: psp.forward_fused(x).backward(g)))]
    if B > 1:
        cases += [("final240_train", run(lambda: final(y240).backward(g240)),
                   run(lambda: final.forward_fused(y240).backward(g240))),
                  ("final480_train", run(lambda: final(y480).backward(g480)),
                   run(lambda: final.forward_fused(y480).backward(g480)))]
    return cases


def peak_extra_mb(fn):
    """Peak memory one eager call allocates above what is allocated before it (MB)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 1e6, 1)


@contextlib.contextmanager
def deterministic(on):
    saved = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(saved)


def train_arms(iters, reps, profile):
    emit(**card(), cudnn_allow_tf32=torch.backends.cudnn.allow_tf32)
    heads = {B: head_train_cases(B) for B in (1, 8)}
    B = 8
    model, inputs = network(B, 12288, True, n_classes=2)        # config 3: LineMOD-shaped, 8 frames
    N = inputs["choose"].shape[-1]
    item = {"labels": torch.randint(0, 2, (B, N), device="cuda", dtype=torch.int32),
            "kp_targ_ofst": torch.randn(B, N, 8, 3, device="cuda"),
            "ctr_targ_ofst": torch.randn(B, N, 3, device="cuda")}

    def step():
        model.zero_grad(set_to_none=True)
        loss, _ = ffb6d_loss(model(inputs), item)
        loss.backward()
    settings = [("off", False, False), ("on", True, False), ("on_deterministic", True, True)]
    for rep in range(reps):
        for hb, cases in heads.items():
            for name, ref, ker in cases:
                t_ref, _ = graph_time(ref, iters)
                t_ker, t_ker_min = graph_time(ker, iters)
                emit(what=name, B=hb, rep=rep, torch_ms=round(t_ref, 4), kernels_ms=round(t_ker, 4),
                     kernels_min_ms=round(t_ker_min, 4), speedup=round(t_ref / t_ker, 3),
                     torch_peak_extra_MB=peak_extra_mb(ref), kernels_peak_extra_MB=peak_extra_mb(ker))
        for label, flag, det in settings:
            model.fused_image_head = flag
            with deterministic(det):
                step()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t, tmin = eager_time(step, max(3, iters // 4))
            emit(what="train_step_arm", fused_image_head=label, B=B, n_pts=12288, rep=rep, ms=round(t, 3),
                 min_ms=round(tmin, 3), max_memory_allocated_GB=round(torch.cuda.max_memory_allocated() / 1e9, 3))
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        for label, flag, det in settings:
            model.fused_image_head = flag
            with deterministic(det):
                step()
                torch.cuda.synchronize()
                with prof(activities=[ProfilerActivity.CUDA]) as p:
                    step()
                    torch.cuda.synchronize()
            rows = {}
            for e in p.key_averages():
                if e.device_type == torch.autograd.DeviceType.CUDA or getattr(e, "self_device_time_total", 0) > 0:
                    rows[e.key] = rows.get(e.key, 0.0) + getattr(e, "self_device_time_total", 0.0) / 1e3
            top = sorted(rows.items(), key=lambda kv: -kv[1])[:25]
            emit(what="train_step_profile", fused_image_head=label, total_cuda_ms=round(sum(rows.values()), 3),
                 top_ms=[(k[:90], round(v, 3)) for k, v in top])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--no-train", action="store_true")
    ap.add_argument("--train-arms", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if a.train_arms:
        train_arms(a.iters, a.reps, a.profile)
        return
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
