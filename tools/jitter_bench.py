#!/usr/bin/env python
"""Time the colour jitter (``ffb6d_color_jitter``) on 32 frames of 480x640.

Device time from CUDA events around replays of a CUDA graph of the C ABI call (plans already on the device, so no
copy and no host-side validation in the window), after warm-up, for two sets of plans:
  random    ColorJitter(0.2, 0.2, 0.2, 0.05) draws (draw_color_jitter), so the op orders are uniform
  hue_pre   the same factors with the hue op before contrast in every frame, so both launches convert to HSV and
            back (the slowest order)
Also the time of one ``ops.color_jitter`` call (plan copy and validation included), the card's name and power limit
read in the same run, and the HBM floor: 2 reads + 1 write of the batch's bytes at 3.35 TB/s.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffb6d_b200 import augment as A                      # noqa: E402
from ffb6d_b200.synthetic import make_aug_frame         # noqa: E402

H, W = 480, 640
HBM_BYTES_PER_S = 3.35e12


def event_ms(torch, fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import ffb6d_b200 as F
    from ffb6d_b200 import _lib
    if not torch.cuda.is_available():
        raise SystemExit("jitter_bench.py needs a GPU")
    dev = torch.device("cuda:0")
    B = args.batch
    rgb = torch.from_numpy(np.stack([make_aug_frame(b, H, W)["rgb"] for b in range(B)])).to(dev)
    torch.manual_seed(0)
    random = A.draw_color_jitter(B)
    hue_pre = random.copy()
    hue_pre[:, :4] = (3, 1, 0, 2)
    act = torch.ones(B, dtype=torch.uint8, device=dev)
    out, work = torch.empty_like(rgb), torch.empty(B, dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    res = {}
    for name, plans in (("random", random), ("hue_pre", hue_pre)):
        plan_d = torch.from_numpy(plans).to(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                _lib.check(_lib.lib.ffb6d_color_jitter(rgb.data_ptr(), B, H, W, plans.ctypes.data, plan_d.data_ptr(),
                                                       act.data_ptr(), out.data_ptr(), work.data_ptr(), s.cuda_stream))
        res[name + "_device_us_per_batch"] = round(1e3 * event_ms(torch, g.replay, args.iters, args.warmup), 2)
        torch.cuda.synchronize()
        assert torch.equal(out, F.color_jitter(rgb, plans))
    res["ops_color_jitter_us_per_batch"] = round(
        1e3 * event_ms(torch, lambda: F.color_jitter(rgb, random), args.iters, args.warmup), 2)
    nbytes = B * H * W * 3
    floor_us = 3 * nbytes / HBM_BYTES_PER_S * 1e6
    res["hbm_floor_us"] = round(floor_us, 2)
    res["random_share_of_hbm_floor"] = round(floor_us / res["random_device_us_per_batch"], 3)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res.update(batch=B, h=H, w=W, gpu=q[0] if q else torch.cuda.get_device_name(0),
               note="device_us: graph replays of the C ABI call (memset + 2 launches), plans on the device; "
                    "hbm_floor: 2 reads + 1 write of %d bytes at 3.35 TB/s" % nbytes)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
