#!/usr/bin/env python
"""PSPUpsample on torch's modules against ``forward_restructured`` (DESIGN.md §4.23), arms alternated and repeated in
one process, cuDNN / cuBLAS at torch's defaults:

* ``stage``: each of ``up_1`` / ``up_2`` / ``up_3`` at B = 1 and 8 -- the eval forward (no autograd) and the
  training forward + backward -- ms per call, and the peak memory one training forward + backward adds;
* ``step``: the whole FFB6D training step at config 3 (B = 8, 2 classes, 12288 points, 480x640, Adam,
  ``fused_image_head=True``), eager and through :class:`ffb6d_b200.GraphedTrainStep`, ``fused_upsample`` off and on,
  with ``max_memory_allocated`` over the timed steps;
* ``eval``: the FFB6D eval forward at B = 1 and 8, ``fused_upsample`` off and on.

Times: CUDA events around ``--iters`` calls ending in a synchronise.  Every repeat is printed, so the spread is in
the output.

    python tools/upsample_bench.py [--repeats 5] [--iters 10] [--parts stage,step,eval] [--out f.json]

Prints one line per figure, then one JSON object with the card, its power limit and every figure.
"""
import argparse
import copy
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from graph_step_bench import card, make_item    # noqa: E402

STAGES = {"up_1": (1024, 256, 60, 80), "up_2": (256, 64, 120, 160), "up_3": (64, 64, 240, 320)}
rows = []


def emit(**kw):
    rows.append(kw)
    print(json.dumps(kw), flush=True)


def timed(fn, iters):
    import torch
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def stages(repeats, iters):
    import torch
    from ffb6d_b200 import cnn
    for name, (Ci, Co, Hi, Wi) in STAGES.items():
        for B in (1, 8):
            torch.manual_seed(0)
            m = cnn.PSPUpsample(Ci, Co).cuda()
            x = torch.randn(B, Ci, Hi, Wi, device="cuda")
            xg = x.clone().requires_grad_(True)
            grad = torch.randn(B, Co, 2 * Hi, 2 * Wi, device="cuda")
            arms = {"torch": m.forward, "kernels": m.forward_restructured}

            def ev(f):
                with torch.no_grad():
                    f(x)

            def tr(f):
                f(xg).backward(grad)
            m.train()
            for f in arms.values():          # warm-up: cuDNN plans, the weight pack
                tr(f)
                tr(f)
            for arm, f in arms.items():
                xg.grad = None
                m.zero_grad(set_to_none=True)
                tr(f)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                xg.grad = None
                m.zero_grad(set_to_none=True)
                tr(f)
                torch.cuda.synchronize()
                emit(what="stage_peak_extra_mb", stage=name, B=B, arm=arm,
                     mb=round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1))
            for rep in range(repeats):
                for arm, f in arms.items():
                    m.train()
                    t_tr = timed(lambda: tr(f), iters)
                    m.eval()
                    ev(f)
                    t_ev = timed(lambda: ev(f), iters)
                    emit(what="stage", stage=name, B=B, arm=arm, rep=rep, train_fwd_bwd_ms=round(t_tr, 3),
                         eval_fwd_ms=round(t_ev, 3))
            del m, x, xg, grad
            gc.collect()
            torch.cuda.empty_cache()


def step(repeats, iters):
    import torch
    from ffb6d_b200 import GraphedTrainStep
    from ffb6d_b200.loss import ffb6d_loss
    from ffb6d_b200.model import FFB6D
    dev = torch.device("cuda")
    item = make_item("ffb6d", 8, 2, dev)
    torch.manual_seed(0)
    base = FFB6D(n_classes=2, fused_image_head=True).to(dev).train()
    arms = {}
    for flag in (False, True):
        model = copy.deepcopy(base)
        model.fused_upsample = flag
        opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device=dev), capturable=True)

        def eager(model=model, opt=opt):
            opt.zero_grad(set_to_none=True)
            loss, _ = ffb6d_loss(model(item), item, valid=item["valid"])
            loss.backward()
            opt.step()
        eager()
        eager()
        arms[("eager", flag)] = eager
        gm = copy.deepcopy(base)
        gm.fused_upsample = flag
        gopt = torch.optim.Adam(gm.parameters(), lr=torch.tensor(1e-4, device=dev), capturable=True)
        gstep = GraphedTrainStep(gm, gopt, item)
        arms[("graphed", flag)] = lambda s=gstep: s(item)
    for rep in range(repeats):
        for (mode, flag), f in arms.items():
            f()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t = timed(f, iters)
            emit(what="step", mode=mode, fused_upsample=flag, B=8, rep=rep, ms=round(t, 3),
                 max_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 3))
    del arms
    gc.collect()
    torch.cuda.empty_cache()


def evals(repeats, iters):
    import torch
    from ffb6d_b200.model import FFB6D
    dev = torch.device("cuda")
    for B in (1, 8):
        item = make_item("ffb6d", B, 2, dev)
        torch.manual_seed(0)
        model = FFB6D(n_classes=2).to(dev).eval()
        outs = {}
        for flag in (False, True):
            model.fused_upsample = flag
            with torch.no_grad():
                outs[flag] = model(item)["pred_rgbd_segs"]
        d = (outs[True] - outs[False]).abs().max().item() / max(outs[False].abs().max().item(), 1e-30)
        emit(what="eval_output_difference", B=B, rel=d)
        for rep in range(repeats):
            for flag in (False, True):
                model.fused_upsample = flag

                def f():
                    with torch.no_grad():
                        model(item)
                f()
                emit(what="eval", B=B, fused_upsample=flag, rep=rep, ms=round(timed(f, iters), 3))
        del model, item
        gc.collect()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--parts", default="stage,step,eval")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("upsample_bench needs a CUDA device")
    info = card()
    print("card, power limit:", info, flush=True)
    parts = a.parts.split(",")
    if "stage" in parts:
        stages(a.repeats, a.iters)
    if "step" in parts:
        step(a.repeats, a.iters)
    if "eval" in parts:
        evals(a.repeats, a.iters)
    res = {"card": info, "rows": rows}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
