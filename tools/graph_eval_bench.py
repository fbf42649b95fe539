#!/usr/bin/env python
"""Eager against CUDA-graphed eval steps (:class:`ffb6d_b200.GraphedEvalStep`), alternated in one process:

* ``ffb6d_b1``, ``ffb6d_b8``: the whole FFB6D (22 classes, 480x640, 12288 points) at B = 1 and B = 8, the eval
  forward alone (validation's and ``demo.py``'s network call);
* ``fusion_c3``, ``fusion_c4``: FFB6DFusionNet at BASELINE configs 3 (B = 8, 2 classes) and 4 (B = 4, 22 classes),
  forward and ``ffb6d_loss``, as ``model_fn`` computes them with ``is_eval=True``.

Per case: ms per step of every repeat (CUDA events and the host clock around ``--iters`` steps ending in a
synchronise, the larger), the package's kernel launches per step issued from the host (``_lib.launch_count()``), and
the reserved memory that building the graphed step added.  A separate profiled run records, with ``torch.profiler``,
the GPU kernels of one step per arm and the kernel time of one replay, and, in the same run, the kernel time of the
weight and BatchNorm packs that the replay makes (every ``modules.weight_cache`` pack made while the step was
captured, captured again on their own into a second graph): ``pack_share`` is their share of the replay's kernel
time.  Before timing, eager and graphed outputs are compared bit for bit.

    python tools/graph_eval_bench.py [--repeats 5] [--iters 10] [--cases ffb6d_b1,ffb6d_b8,fusion_c3,fusion_c4]

Prints the card and its power limit, one line per case, then one JSON object with every figure.
"""
import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from graph_step_bench import card, make_item  # noqa: E402

CASES = {"ffb6d_b1": ("ffb6d", 1, 22), "ffb6d_b8": ("ffb6d", 8, 22),
         "fusion_c3": ("fusion", 8, 2), "fusion_c4": ("fusion", 4, 22)}
LOSS_KEYS = ("labels", "kp_targ_ofst", "ctr_targ_ofst")


def _flat(res):
    out, loss, info = res
    ts = [out[k] for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")] + list(out["fused_rgb"])
    if loss is not None:
        ts += [loss] + [info[k] for k in sorted(info)]
    return ts


def _kernels(prof):
    """(count, µs) of the GPU kernels a profile recorded (copies and memsets left out)."""
    evs = [ev for ev in prof.events() if ev.device_type is not None and "cuda" in str(ev.device_type).lower()
           and "memcpy" not in ev.name.lower() and "memset" not in ev.name.lower()]
    return len(evs), sum(ev.time_range.elapsed_us() for ev in evs)


def run_case(name, repeats, iters):
    import torch
    from ffb6d_b200 import GraphedEvalStep, _lib, modules
    from ffb6d_b200.loss import ffb6d_loss
    from ffb6d_b200.model import FFB6D, FFB6DFusionNet
    from torch.profiler import ProfilerActivity, profile

    kind, B, n_classes = CASES[name]
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = (FFB6D(n_classes=n_classes) if kind == "ffb6d" else FFB6DFusionNet(n_classes=n_classes)).to(dev).eval()
    item = make_item(kind, B, n_classes, dev)
    if kind == "ffb6d":
        item = {k: v for k, v in item.items() if k not in LOSS_KEYS}
    with_loss = kind != "ffb6d"

    def eager():
        with torch.no_grad():
            out = model(item) if kind == "ffb6d" else model(item, item["rgb_feats"])
            loss, info = ffb6d_loss(out, item, valid=item["valid"]) if with_loss else (None, None)
        return out, loss, info

    # every pack the capture makes, kept to be captured again on its own for the pack share
    packs, weight_cache = [], modules.weight_cache

    def recording(owner, attr, key, make):
        if torch.cuda.is_current_stream_capturing():
            packs.append(make)
        return weight_cache(owner, attr, key, make)

    gc.collect()
    torch.cuda.empty_cache()
    reserved0 = torch.cuda.memory_reserved(dev)
    modules.weight_cache = recording
    try:
        graphed = GraphedEvalStep(model, item)
    finally:
        modules.weight_cache = weight_cache
    gc.collect()
    torch.cuda.empty_cache()
    reserved_gb = (torch.cuda.memory_reserved(dev) - reserved0) / 1e9

    want = [t.clone() for t in _flat(eager())]
    got = _flat(graphed(item))
    bitwise = len(got) == len(want) and all(torch.equal(a, b) for a, b in zip(got, want))
    del want, got

    arms = {"eager": eager, "graphed": lambda: graphed(item)}
    res = {a: {"ms": []} for a in arms}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    for _ in range(repeats):
        for a, fn in arms.items():
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
    for a, fn in arms.items():
        n0 = _lib.launch_count()
        fn()
        torch.cuda.synchronize()
        res[a]["launches_per_step"] = _lib.launch_count() - n0

    # the profiled run: one step per arm, then the packs alone, from a graph of their own
    pack_graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(pack_graph):
        for make in packs:
            make()
    for a, fn in arms.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        res[a]["profiled_kernels_per_step"], res[a]["kernel_us"] = _kernels(prof)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pack_graph.replay()
        torch.cuda.synchronize()
    pack_kernels, pack_us = _kernels(prof)
    g = res["graphed"]
    g.update(captures=graphed.captures, reserved_gb=reserved_gb, packs=len(packs), pack_kernels=pack_kernels,
             pack_us=pack_us, pack_share=pack_us / g["kernel_us"] if g["kernel_us"] else None)
    for a in arms:
        res[a]["ms_min"], res[a]["ms_max"] = min(res[a]["ms"]), max(res[a]["ms"])
    res["bitwise_equal"] = bitwise
    del graphed, pack_graph, packs, model, item, arms
    gc.collect()
    torch.cuda.empty_cache()
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
        sys.exit("graph_eval_bench: needs a CUDA device")
    out = {"card": card(), "device": torch.cuda.get_device_name(0), "repeats": args.repeats, "iters": args.iters,
           "cases": {}}
    print("card: %s" % out["card"], flush=True)
    for name in args.cases.split(","):
        r = run_case(name, args.repeats, args.iters)
        out["cases"][name] = r
        e, g = r["eager"], r["graphed"]
        print("%-10s eager %6.2f-%6.2f ms %4d launches %5d kernels | graphed %6.2f-%6.2f ms %4d launches %5d kernels "
              "%.2f GB reserved, packs %d (%d kernels) %.1f %% of replay kernel time | bitwise %s (%d capture)"
              % (name, e["ms_min"], e["ms_max"], e["launches_per_step"], e["profiled_kernels_per_step"],
                 g["ms_min"], g["ms_max"], g["launches_per_step"], g["profiled_kernels_per_step"], g["reserved_gb"],
                 g["packs"], g["pack_kernels"], 100 * (g["pack_share"] or 0), r["bitwise_equal"], g["captures"]),
              flush=True)
    text = json.dumps(out)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
