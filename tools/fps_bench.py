#!/usr/bin/env python
"""Time farthest point sampling: the device kernel (ffb6d_farthest_point_sampling) against the reference's compiled
farthest_point_sampling.cpp on the host cores (oracle/_ref/libfps_ref.so, built by ``make -C oracle -f fps_ref.mk REF=...``).

The reference runs one cloud at a time on one core; the device runs a batch of G clouds in one launch.  Device
times are CUDA events over ``--repeats`` launches after a warm-up; host times are wall clock over the same clouds.
Both arms get the same clouds and init_center, and their indices are compared before anything is timed.
Prints the GPU's name and power limit and the host's core count with the table.

    python tools/fps_bench.py [--repeats 20] [--out fps_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, G, P, S): the tool's own case (one mesh, 8 keypoints), YCB's 21 objects in one batch, LineMOD-sized meshes,
# more keypoints, and the largest cloud one cluster holds
CASES = [("ycb_1x2621_s8", 1, 2621, 8), ("ycb_21x2621_s8", 21, 2621, 8), ("lm_1x40000_s8", 1, 40000, 8),
         ("lm_15x40000_s8", 15, 40000, 8), ("ycb_21x2621_s64", 21, 2621, 64), ("max_1x114688_s64", 1, 114688, 64)]


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from ffb6d_b200 import ops
    from oracle import fps_oracle
    if not torch.cuda.is_available():
        raise SystemExit("fps_bench needs a CUDA device")
    if not fps_oracle.available():
        raise SystemExit("oracle/_ref/libfps_ref.so is missing: build it with oracle/fps_ref.mk where the reference's sources are present")
    dev = torch.device("cuda:0")
    rows = []
    print("GPU: %s | host cores: %d" % (gpu_info(), os.cpu_count()))
    print("%-18s %10s %12s %12s %8s" % ("case", "points", "device ms", "host ms", "ratio"))
    for name, G, P, S in CASES:
        clouds = np.random.RandomState(P + G).rand(G, P, 3).astype(np.float32)
        x = torch.from_numpy(clouds).to(dev)
        idx = ops.farthest_point_sampling(x, S, init_center=True, return_index=True)[1]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        want = np.stack([fps_oracle.fps(c, S, init_center=True) for c in clouds])
        host_ms = (time.perf_counter() - t0) * 1e3
        assert np.array_equal(idx.cpu().numpy(), want), name
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(a.repeats):
            ops.farthest_point_sampling(x, S, init_center=True)
        ev[1].record()
        torch.cuda.synchronize()
        dev_ms = ev[0].elapsed_time(ev[1]) / a.repeats
        rows.append(dict(case=name, G=G, P=P, S=S, device_ms=dev_ms, host_ms=host_ms))
        print("%-18s %10d %12.3f %12.3f %8.1f" % (name, G * P, dev_ms, host_ms, host_ms / dev_ms))
    res = dict(gpu=gpu_info(), host_cores=os.cpu_count(), repeats=a.repeats, rows=rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
