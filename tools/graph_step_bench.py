#!/usr/bin/env python
"""Eager against CUDA-graphed training steps (:class:`ffb6d_b200.GraphedTrainStep`), alternated in one process:

* ``fusion_c3``: FFB6DFusionNet, BASELINE config 3 (B = 8, 2 classes, 12288 points, 480x640);
* ``fusion_c4``: FFB6DFusionNet, config 4 (B = 4, 22 classes);
* ``ffb6d_c3``: the whole FFB6D at config 3 with ``fused_image_head=True``.

The graphed step's ``max_memory_allocated`` leaves out its graph's private pool, whose blocks are free between
replays; ``reserved_gb`` is the reserved memory that building the step added (pool, gradients, Adam state, inputs).

Each case with and without ``torch.use_deterministic_algorithms(True)``; both arms train with Adam
(``capturable=True``, tensor lr) through ``ffb6d_loss``.  Per arm: ms per step of every repeat (CUDA events and the
host clock around ``--iters`` steps ending in a synchronise, the larger), ``max_memory_allocated`` over the timed
steps, the package's kernel launches per step issued from the host (``_lib.launch_count()``), and, in a separate
profiled step, the number of GPU kernels ``torch.profiler`` records for one step.

    python tools/graph_step_bench.py [--repeats 5] [--iters 10] [--cases fusion_c3,fusion_c4,ffb6d_c3] [--out f.json]

Prints one line per case and mode, then one JSON object with the card, its power limit and every figure.
"""
import argparse
import copy
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {"fusion_c3": ("fusion", 8, 2), "fusion_c4": ("fusion", 4, 22), "ffb6d_c3": ("ffb6d", 8, 2)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_item(kind, B, n_classes, dev, N=12288, n_kps=8):
    import torch
    from ffb6d_b200.model import FFB6DFusionNet
    from ffb6d_b200.schedule import build_ffb6d_indices
    from ffb6d_b200.synthetic import make_batch
    batch = make_batch(list(range(B)), n_points=N)
    item = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(dev), torch.from_numpy(batch["dpt_xyz"]).to(dev))
    item["choose"] = torch.from_numpy(batch["choose"]).to(dev)
    item["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    if kind == "ffb6d":
        item["rgb"] = torch.rand((B, 3, 480, 640), generator=g, device=dev) * 2 - 1
    else:
        item["rgb_feats"] = [torch.randn(s, generator=g, device=dev) for s in FFB6DFusionNet.rgb_feature_shapes(B)]
    labels = torch.randint(1, n_classes, (B, N), generator=g, device=dev, dtype=torch.int32)
    labels[torch.rand((B, N), generator=g, device=dev) < 0.6] = 0            # background, as in a real frame
    item.update(labels=labels, kp_targ_ofst=torch.randn((B, N, n_kps, 3), generator=g, device=dev),
                ctr_targ_ofst=torch.randn((B, N, 3), generator=g, device=dev),
                valid=torch.arange(B, device=dev) % 4 != 1)
    return item


def run_case(name, det, repeats, iters):
    import torch
    from ffb6d_b200 import GraphedTrainStep, _lib
    from ffb6d_b200.loss import ffb6d_loss
    from ffb6d_b200.model import FFB6D, FFB6DFusionNet

    kind, B, n_classes = CASES[name]
    dev = torch.device("cuda")
    torch.use_deterministic_algorithms(det)
    torch.manual_seed(0)
    if kind == "ffb6d":
        model = FFB6D(n_classes=n_classes, fused_image_head=True).to(dev).train()
    else:
        model = FFB6DFusionNet(n_classes=n_classes).to(dev).train()
    twin = copy.deepcopy(model)
    item = make_item(kind, B, n_classes, dev)

    def adam(m):
        return torch.optim.Adam(m.parameters(), lr=torch.tensor(1e-4, device=dev), capturable=True)
    opt_e, opt_g = adam(model), adam(twin)

    def eager():
        opt_e.zero_grad(set_to_none=True)
        out = model(item) if kind == "ffb6d" else model(item, item["rgb_feats"])
        loss, _ = ffb6d_loss(out, item, valid=item["valid"])
        loss.backward()
        opt_e.step()
        return loss

    gc.collect()
    torch.cuda.empty_cache()
    reserved0 = torch.cuda.memory_reserved(dev)
    graphed = GraphedTrainStep(twin, opt_g, item)
    gc.collect()
    torch.cuda.empty_cache()
    # max_memory_allocated does not see the graph's private pool (its blocks are free between replays): what the
    # graphed step holds is the reserved memory it added (pool, gradients, Adam state, input buffers)
    graph_reserved_gb = (torch.cuda.memory_reserved(dev) - reserved0) / 1e9
    arms = {"eager": eager, "graphed": lambda: graphed(item)[0]}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    res = {a: {"ms": [], "peak_gb": [], "launches_per_step": None, "profiled_kernels_per_step": None} for a in arms}
    for _ in range(repeats):
        for a, fn in arms.items():
            torch.cuda.reset_peak_memory_stats(dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            res[a]["ms"].append(max(e0.elapsed_time(e1), wall) / iters)
            res[a]["peak_gb"].append(torch.cuda.max_memory_allocated(dev) / 1e9)
    for a, fn in arms.items():
        n0 = _lib.launch_count()
        fn()
        torch.cuda.synchronize()
        res[a]["launches_per_step"] = _lib.launch_count() - n0
    from torch.profiler import ProfilerActivity, profile
    for a, fn in arms.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        res[a]["profiled_kernels_per_step"] = sum(
            1 for ev in prof.events() if ev.device_type is not None and "cuda" in str(ev.device_type).lower()
            and "memcpy" not in ev.name.lower() and "memset" not in ev.name.lower())
    res["graphed"]["captures"] = graphed.captures
    res["graphed"]["reserved_gb"] = graph_reserved_gb
    for a in arms:
        r = res[a]
        r["ms_min"], r["ms_max"] = min(r["ms"]), max(r["ms"])
        r["peak_gb_max"] = max(r["peak_gb"])
    del graphed, model, twin, opt_e, opt_g, item
    gc.collect()
    torch.cuda.empty_cache()
    torch.use_deterministic_algorithms(False)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("graph_step_bench: needs a CUDA device")
    out = {"card": card(), "device": torch.cuda.get_device_name(0), "repeats": args.repeats, "iters": args.iters,
           "cases": {}}
    print("card: %s" % out["card"], flush=True)
    for name in args.cases.split(","):
        for det in (False, True):
            key = "%s_%s" % (name, "deterministic" if det else "default")
            r = run_case(name, det, args.repeats, args.iters)
            out["cases"][key] = r
            print("%-28s eager %6.2f-%6.2f ms %5.2f GB %4d launches %5d kernels | graphed %6.2f-%6.2f ms %5.2f GB "
                  "(%.2f GB reserved) %4d launches %5d kernels (%d capture)"
                  % (key, r["eager"]["ms_min"], r["eager"]["ms_max"], r["eager"]["peak_gb_max"],
                     r["eager"]["launches_per_step"], r["eager"]["profiled_kernels_per_step"],
                     r["graphed"]["ms_min"], r["graphed"]["ms_max"], r["graphed"]["peak_gb_max"],
                     r["graphed"]["reserved_gb"],
                     r["graphed"]["launches_per_step"], r["graphed"]["profiled_kernels_per_step"],
                     r["graphed"]["captures"]), flush=True)
    text = json.dumps(out)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
