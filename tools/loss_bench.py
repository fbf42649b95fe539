#!/usr/bin/env python
"""Time FFB6D's training loss, forward + backward, as CUDA-graph replays: the fused kernels (ffb6d_b200.loss.ffb6d_loss)
against the reference's float32 torch ops (oracle/loss_oracle.ffb6d_loss_torch) on the same GPU and inputs.

    python tools/loss_bench.py [--iters 200] [--rounds 5]

Config 3: LineMOD-shaped, B = 8, C = 2; config 4: YCB-shaped, B = 4, C = 22; N = 12288, n_kps = 8, every frame valid
(the reference's boolean indexing of a masked batch synchronises the host and cannot be captured).  The two sides
alternate, ``--rounds`` times, each timing ``--iters`` replays with CUDA events.  The outputs of both are compared
first.  ``bytes`` is the least traffic of the fused pass: the forward reads logits, labels, offsets and targets once,
the backward reads them again and writes the gradients.  One JSON line per config.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KEYS = ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_inputs(dev, B, C, K, N, seed=0):
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    ep = {"pred_rgbd_segs": torch.randn(B, C, N, generator=g, device=dev) * 3,
          "pred_kp_ofs": torch.randn(B, K, N, 3, generator=g, device=dev),
          "pred_ctr_ofs": torch.randn(B, 1, N, 3, generator=g, device=dev)}
    labels = torch.randint(0, C, (B, N), generator=g, device=dev, dtype=torch.int32)
    labels[torch.rand(B, N, generator=g, device=dev) < 0.6] = 0
    item = {"labels": labels, "kp_targ_ofst": torch.randn(B, N, K, 3, generator=g, device=dev),
            "ctr_targ_ofst": torch.randn(B, N, 3, generator=g, device=dev)}
    return {k: v.requires_grad_(True) for k, v in ep.items()}, item


def captured(fn, ep, item):
    """A CUDA graph of fn(ep, item) -> loss; loss.backward(); returns (graph, [loss, grads...])."""
    import torch

    def step():
        for t in ep.values():
            t.grad = None
        loss = fn(ep, item)[0]
        loss.backward()
        return [loss.detach()] + [ep[k].grad for k in KEYS]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    return graph, outs


def time_replays(graph, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters          # us per replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    from ffb6d_b200.loss import ffb6d_loss
    from oracle.loss_oracle import ffb6d_loss_torch
    if not torch.cuda.is_available():
        raise SystemExit("loss_bench needs a GPU")
    dev = torch.device("cuda:0")
    limit = power_limit()
    for config, B, C in ((3, 8, 2), (4, 4, 22)):
        K, N = 8, 12288
        ep_f, item = make_inputs(dev, B, C, K, N)
        ep_r = {k: v.detach().clone().requires_grad_(True) for k, v in ep_f.items()}
        g_f, out_f = captured(ffb6d_loss, ep_f, item)
        g_r, out_r = captured(ffb6d_loss_torch, ep_r, item)
        g_f.replay()
        g_r.replay()
        torch.cuda.synchronize()
        loss_rel = abs(out_f[0].item() - out_r[0].item()) / abs(out_r[0].item())
        of_equal = all(torch.equal(a, b) for a, b in zip(out_f[2:], out_r[2:]))
        seg_diff = (out_f[1] - out_r[1]).abs().max().item()
        for _ in range(3):
            time_replays(g_f, 20)
            time_replays(g_r, 20)
        fused, ref = [], []
        for _ in range(args.rounds):
            fused.append(time_replays(g_f, args.iters))
            ref.append(time_replays(g_r, args.iters))
        nbytes = 4 * (B * C * N + B * N + 2 * (B * K * N * 3 + B * N * 3))          # logits, labels, offsets, targets
        nbytes = 2 * nbytes + 4 * (B * C * N + B * (K + 1) * N * 3) + 4 * B * N      # read twice, grads, lse
        fmin = min(fused)
        print(json.dumps({
            "metric": "FFB6D training loss, forward + backward, CUDA-graph replay", "config": config, "B": B, "C": C,
            "n_kps": K, "N": N, "fused_us": sorted(fused), "reference_torch_us": sorted(ref),
            "speedup_min": min(ref) / fmin, "bytes": nbytes, "fused_GBps": nbytes / fmin / 1e3,
            "hbm_floor_us_at_3.35TBps": nbytes / 3.35e6, "loss_rel_diff": loss_rel, "offset_grads_equal": of_equal,
            "seg_grad_max_abs_diff": seg_diff, "gpu": torch.cuda.get_device_name(dev), "power_limit": limit}))


if __name__ == "__main__":
    main()
