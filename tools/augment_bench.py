#!/usr/bin/env python
"""Time the synthetic-frame augmentation on one plan with every stage on.

Both arms use the same scalars (``make_aug_golden.script``): HSV, sharpen, a 137-degree length-7 motion blur, a 5x5
Gaussian blur, gaussian_noise with sigma 12 and YCB's final normal(0, 7), on 480x640 frames.

Default (GPU): device time of ``ffb6d_rgb_add_noise`` and ``ffb6d_add_real_back`` on 32 frames, from CUDA events
around replays of a CUDA graph of the C ABI call (records already on the device, so no copy and no host-side
validation in the window), after warm-up; also the time of one ``ops.rgb_add_noise`` call, which adds the copy of
the records to the device and their validation.  The card's name and power limit are read in the same run.
``--cpu-reference DIR``: the reference's own ``rgb_add_noise`` (OpenCV + numpy, including numpy's per-pixel normal
draws) per frame on one CPU core, run from the reference's source tree DIR; this is a CPU number."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_aug_golden as M                             # noqa: E402
from ffb6d_b200 import augment as A                      # noqa: E402
from ffb6d_b200.synthetic import make_aug_frame         # noqa: E402

SCRIPT = M.script("ycb", hsv=(0.5, 0.5), sharpen=0.5, motion=(137, 7), gauss=(5, 0.6), noise=(0.9, 12), final=True)
H, W = 480, 640


class ForcedRNG:
    """The scripted scalars; per-pixel normals drawn by numpy, as the reference draws them."""

    def __init__(self, seed):
        self.script, self.rs = list(SCRIPT), np.random.RandomState(seed)

    def rand(self):
        return float(self.script.pop(0))

    def randint(self, *a):
        return int(self.script.pop(0))

    def randn(self, *shape):
        return self.rs.randn(*shape)

    def normal(self, loc=0.0, scale=1.0, size=None):
        return self.rs.normal(loc, scale, size)


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


def gpu(args):
    import torch
    import ffb6d_b200 as F
    from ffb6d_b200 import _lib
    dev = torch.device("cuda:0")
    B = args.batch
    fr = make_aug_frame(1, H, W)
    t = lambda k: torch.from_numpy(np.stack([fr[k]] * B)).to(dev)       # noqa: E731
    rgb, lab, dpt, brgb, blab, bdpt = (t(k) for k in ("rgb", "labels", "raw", "back_rgb", "back_labels", "back_dpt"))
    plans = np.stack([A.draw_rgb_noise(M.ScriptRNG(SCRIPT), "ycb")] * B)
    plan_d = torch.from_numpy(plans).to(dev)
    mode = torch.full((B,), 3, dtype=torch.uint8, device=dev)
    out, work = torch.empty_like(rgb), torch.empty_like(rgb)
    rgb2, dpt2 = torch.empty_like(rgb), torch.empty_like(dpt)
    s = torch.cuda.Stream()
    graphs = {}
    with torch.cuda.stream(s):
        for name in ("rgb_add_noise", "add_real_back"):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                if name == "rgb_add_noise":
                    _lib.check(_lib.lib.ffb6d_rgb_add_noise(rgb.data_ptr(), B, H, W, plans.ctypes.data,
                                                            plan_d.data_ptr(), 1, None, out.data_ptr(),
                                                            work.data_ptr(), s.cuda_stream))
                else:
                    _lib.check(_lib.lib.ffb6d_add_real_back(rgb.data_ptr(), lab.data_ptr(), dpt.data_ptr(),
                                                            brgb.data_ptr(), blab.data_ptr(), 1, bdpt.data_ptr(),
                                                            mode.data_ptr(), 0, B, H, W, rgb2.data_ptr(),
                                                            dpt2.data_ptr(), s.cuda_stream))
            graphs[name] = g
    res = {name + "_device_ms_per_batch": round(event_ms(torch, g.replay, args.iters, args.warmup), 4)
           for name, g in graphs.items()}
    assert torch.equal(out, F.rgb_add_noise(rgb, plans, 1))
    res["ops_rgb_add_noise_ms_per_batch"] = round(
        event_ms(torch, lambda: F.rgb_add_noise(rgb, plans, 1), args.iters, args.warmup), 4)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res.update(batch=B, h=H, w=W, gpu=q[0] if q else torch.cuda.get_device_name(0),
               stages="hsv, sharpen, motion 137/7, gaussian 5x5, noise sigma 12, final normal(0, 7)",
               note="device_ms: graph replays of the C ABI call, records on the device; ops_ms: ops.rgb_add_noise, "
                    "which also copies the records to the device and validates them")
    return res


def cpu_reference(args):
    os.environ["FFB6D_REFERENCE"] = args.cpu_reference
    M.R.REF_ROOT = args.cpu_reference
    import cv2
    cv2.setNumThreads(1)
    fr = make_aug_frame(1, H, W)
    times = []
    for i in range(args.iters):
        me = M.reference_self("ycb", ForcedRNG(i), fr)
        t0 = time.perf_counter()
        me.rgb_add_noise(fr["rgb"])
        times.append(time.perf_counter() - t0)
    return dict(cpu_reference_rgb_add_noise_ms_per_frame=round(1e3 * float(np.median(times)), 3), threads=1,
                stages="hsv, sharpen, motion 137/7, gaussian 5x5, noise sigma 12, final normal(0, 7)",
                note="CPU number: the reference's rgb_add_noise, one core, median of %d frames" % args.iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-reference", default=None)
    args = ap.parse_args()
    print(json.dumps(cpu_reference(args) if args.cpu_reference else gpu(args)))


if __name__ == "__main__":
    main()
