#!/usr/bin/env python
"""``fused_lfa`` off and on at BASELINE config 3 (FFB6DFusionNet, 2 classes, 8 keypoints, batch 8, 12288 points), one
GPU, alternated and repeated:

* ``encoder_ms``: forward + backward of the encoder (``rndla_pre_stages`` and the four ``Dilated_res_block`` s with
  their ``random_sample`` s), CUDA-event time per iteration;
* ``saved_mb``: the bytes autograd keeps for the backward of that encoder forward (every tensor handed to
  ``save_for_backward`` or saved by a torch op, each storage counted once);
* ``step_ms`` / ``step_peak_gb``: one training step of the whole FusionNet (forward, FFB6D's loss, backward) and its
  ``torch.cuda.max_memory_allocated``.

    python tools/lfa_train_bench.py [--repeats 5] [--iters 10] [--out lfa_train_bench.json]

Prints one JSON object: the card, its power limit, and per mode every repeat plus the lowest and highest value.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from ffb6d_b200 import ops
    from ffb6d_b200.loss import ffb6d_loss
    from ffb6d_b200.model import FFB6DFusionNet
    from ffb6d_b200.schedule import build_ffb6d_indices
    from ffb6d_b200.synthetic import make_batch

    assert torch.cuda.is_available(), "lfa_train_bench measures on a GPU"
    dev = torch.device("cuda", 0)
    B, N0, n_cls, n_kps = args.batch, 12288, 2, 8
    torch.manual_seed(0)
    model = FFB6DFusionNet(n_classes=n_cls, n_pts=N0, n_kps=n_kps).to(dev).train()
    batch = make_batch(list(range(B)), n_points=N0)
    with torch.no_grad():
        inputs = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(dev), torch.from_numpy(batch["dpt_xyz"]).to(dev))
    inputs["choose"] = torch.from_numpy(batch["choose"]).to(dev)
    inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    rgb = [torch.randn(s, generator=g, device=dev).requires_grad_(True) for s in FFB6DFusionNet.rgb_feature_shapes(B)]
    item = {"labels": torch.randint(0, n_cls, (B, N0), generator=g, device=dev, dtype=torch.int32),
            "kp_targ_ofst": torch.randn((B, N0, n_kps, 3), generator=g, device=dev),
            "ctr_targ_ofst": torch.randn((B, N0, 3), generator=g, device=dev)}

    def encoder(fused):
        p = model.rndla_pre_stages(inputs["cld_rgb_nrm"]).unsqueeze(3)
        outs = []
        for i in range(4):
            f = model.rndla_ds_stages[i](p, inputs["cld_xyz%d" % i], inputs["cld_nei_idx%d" % i], fused_lfa=fused)
            p = ops.random_sample(f, inputs["cld_sub_idx%d" % i])
            outs.append(p)
        return outs

    def encoder_step(fused):
        outs = encoder(fused)
        sum(o.sum() for o in outs).backward()

    def saved_bytes(fused):
        seen = {}

        def pack(t):     # keeps a detached alias: handing back `t` itself would tie a saved output to its node
            if t.device.type == "cuda":
                st = t.untyped_storage()
                seen[st.data_ptr()] = st.nbytes()
            return t.detach()

        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            outs = encoder(fused)
        del outs
        gc.collect()
        return sum(seen.values())

    def full_step(fused):
        model.fused_lfa = fused
        for t in rgb:
            t.grad = None
        model.zero_grad(set_to_none=True)
        out = model(inputs, rgb)
        loss = ffb6d_loss(out, item)[0] + sum(r.mean() for r in out["fused_rgb"]) * 1e-3
        loss.backward()

    def timed(fn, fused, iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            model.zero_grad(set_to_none=True)
            fn(fused)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    modes = {"off": False, "on": True}
    for fused in modes.values():       # warm-up of every shape the windows use
        for _ in range(3):
            encoder_step(fused)
            full_step(fused)
    res = {m: {"encoder_ms": [], "step_ms": [], "step_peak_gb": [], "saved_mb": []} for m in modes}
    for _ in range(args.repeats):
        for m, fused in modes.items():
            res[m]["encoder_ms"].append(timed(encoder_step, fused, args.iters))
            res[m]["step_ms"].append(timed(full_step, fused, args.iters))
            model.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            full_step(fused)
            torch.cuda.synchronize()
            res[m]["step_peak_gb"].append(torch.cuda.max_memory_allocated(dev) / 1e9)
            res[m]["saved_mb"].append(saved_bytes(fused) / 1e6)
    model.fused_lfa = False
    summary = {"card": card(), "config": 3, "batch": B, "points": N0, "repeats": args.repeats, "iters": args.iters}
    for m in modes:
        summary[m] = {k: {"runs": [round(x, 3) for x in v], "min": round(min(v), 3), "max": round(max(v), 3)}
                      for k, v in res[m].items()}
    line = json.dumps(summary)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
