#!/usr/bin/env python
"""Backward time of every gather and 1x1-layer weight gradient of one FFB6DFusionNet training step, with the atomic
kernels (default) and with the deterministic paths taken under torch.use_deterministic_algorithms(True).

    python tools/det_bench.py [--batch 2] [--reps 20]

Gathers: the 23 of tables.gather_schedule plus the two K = 1 neighbour gathers of every Building_block, on the real
indices of synthetic 480x640 frames (NCS layout, as the model calls them).  Weight gradients: the layer shapes one
training step of the model calls modules._wgrad with, recorded during that step.  The deterministic time includes
everything its backward does per call (CSR plan, arg-max map, workspace).  CUDA events over --reps calls after a
warm-up; one JSON line per op on stdout, then a summary line.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    from ffb6d_b200 import modules, ops
    from ffb6d_b200 import tables as T
    from ffb6d_b200._lib import LAYOUT_NCS
    from ffb6d_b200.model import FFB6DFusionNet
    from ffb6d_b200.schedule import build_ffb6d_indices
    from ffb6d_b200.synthetic import make_batch

    dev = torch.device("cuda")
    B = args.batch
    batch = make_batch(list(range(B)))
    ind = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(dev), torch.from_numpy(batch["dpt_xyz"]).to(dev))
    ind["choose"] = torch.from_numpy(batch["choose"]).to(dev)
    ind["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(dev)

    def timed(fn, det):
        torch.use_deterministic_algorithms(det)
        try:
            for _ in range(3):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3 / args.reps
        finally:
            torch.use_deterministic_algorithms(False)

    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    n_lvl = [T.set_size(("cld", i)) for i in range(5)]
    gathers = [(op, key, C, S, Q, K) for op, key, C, S, Q, K in T.gather_schedule()]
    gathers += [("neighbour", "cld_nei_idx%d" % i, d // 2, n_lvl[i], n_lvl[i] * 16, 1) for i, d in enumerate((32, 64, 128, 256))]
    for op, key, C, S, Q, K in gathers:
        idx = ind[key].reshape(B, Q, K).contiguous()
        f3 = torch.randn((B, C, S), generator=g, device=dev)
        gout = torch.randn((B, C, Q), generator=g, device=dev)
        fn = lambda: ops._gather_max_bwd(f3, idx, gout, LAYOUT_NCS)
        t_atomic, t_det = timed(fn, False), timed(fn, True)
        rows.append({"op": op, "index": key, "C": C, "S": S, "Q": Q, "K": K, "atomic_us": t_atomic, "det_us": t_det})
        print(json.dumps(rows[-1]))

    shapes = []
    wgrad = modules._wgrad

    def record(dz, x1, x2, Bw, Co, P):
        shapes.append((Bw, x1.shape[1], x2.shape[1] if x2 is not None else 0, Co, P))
        return wgrad(dz, x1, x2, Bw, Co, P)

    model = FFB6DFusionNet().to(dev).train()
    rgb = [torch.randn(s, generator=g, device=dev).requires_grad_(True) for s in FFB6DFusionNet.rgb_feature_shapes(B)]
    modules._wgrad = record
    try:
        out = model(ind, rgb)
        (sum(v.float().mean() for k, v in out.items() if k != "fused_rgb") + sum(r.mean() for r in out["fused_rgb"])).backward()
    finally:
        modules._wgrad = wgrad
    for shp in sorted(set(shapes), key=shapes.index):
        Bw, C1, C2, Co, P = shp
        dz = torch.randn((Bw, Co, P), generator=g, device=dev)
        x1 = torch.randn((Bw, C1, P), generator=g, device=dev)
        x2 = torch.randn((Bw, C2, P), generator=g, device=dev) if C2 else None
        fn = lambda: wgrad(dz, x1, x2, Bw, Co, P)
        t_atomic, t_det = timed(fn, False), timed(fn, True)
        rows.append({"op": "wgrad", "B": Bw, "C1": C1, "C2": C2, "Co": Co, "P": P, "calls": shapes.count(shp),
                     "atomic_us": t_atomic, "det_us": t_det})
        print(json.dumps(rows[-1]))
    tot = lambda kind, col: sum(r[col] * r.get("calls", 1) for r in rows if (r["op"] == "wgrad") == (kind == "wgrad"))
    print(json.dumps({"summary": True, "gpu": torch.cuda.get_device_name(dev), "batch": B, "reps": args.reps,
                      "gathers_atomic_us": tot("gather", "atomic_us"), "gathers_det_us": tot("gather", "det_us"),
                      "wgrad_atomic_us": tot("wgrad", "atomic_us"), "wgrad_det_us": tot("wgrad", "det_us")}))


if __name__ == "__main__":
    main()
