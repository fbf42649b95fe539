"""Developer tool: GPU time of the YCB depth completion (``ffb6d_fill_depth``) for a batch of raw 480x640 frames,
and of the captured index build from raw depth (completion -> msk_dp sampling -> back-projection -> 22 searches)
against the same build from depth already in metres.  CUDA events, after warm-up, each timed window >= --min-s
of work.  Prints one JSON line with the card's name and power limit read in the same run.

usage: python tools/fill_bench.py [--batch 32] [--min-s 1.0]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

CAM_SCALE = 10000.0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in q[torch.cuda.current_device()].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown", "max_sm_clock": "unknown"}


def time_ms(fn, min_s):
    """Mean ms per call of ``fn`` over a window of at least ``min_s`` seconds (CUDA events)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    n = max(10, int(min_s * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, n


def capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--points", type=int, default=12288)
    ap.add_argument("--min-s", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fill_bench.py needs a GPU")
    import ffb6d_b200 as F
    from ffb6d_b200 import _lib
    from ffb6d_b200.ops import intrinsics_to_device, _stream
    from ffb6d_b200.synthetic import INTRINSICS, make_raw_depth

    dev = torch.device("cuda:0")
    B, H, W = args.batch, 480, 640
    raw = torch.from_numpy(np.stack([make_raw_depth(s) for s in range(B)])).to(dev)
    filled = torch.empty((B, H, W), dtype=torch.float32, device=dev)
    depth_m = torch.empty_like(filled)
    nbytes = int(_lib.lib.ffb6d_fill_depth_workspace_bytes(B, H, W))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    st = _stream(dev)

    def fill():
        _lib.check(_lib.lib.ffb6d_fill_depth(raw.data_ptr(), B, H, W, C.c_float(CAM_SCALE), filled.data_ptr(),
                                             depth_m.data_ptr(), ws.data_ptr(), nbytes, st))

    fill_ms, fill_n = time_ms(fill, args.min_s)

    intr = intrinsics_to_device(INTRINSICS["ycb_K1"], dev)
    fill()
    torch.cuda.synchronize()
    dpt_m = depth_m.clone()
    from_raw = capture(lambda: F.build_ffb6d_indices_from_raw_depth(raw, CAM_SCALE, intr, args.points, seed=1))
    from_m = capture(lambda: F.build_ffb6d_indices_from_depth(
        dpt_m, intr, F.sample_valid_pixels(dpt_m, args.points, seed=1)))
    raw_ms, raw_n = time_ms(from_raw, args.min_s)
    m_ms, m_n = time_ms(from_m, args.min_s)
    raw_ms2, _ = time_ms(from_raw, args.min_s)        # alternate: a drift between the two windows shows here
    res = dict(card(), batch=B, image="%dx%d" % (H, W), points=args.points,
               fill_ms=round(fill_ms, 4), fill_calls=fill_n, fill_frames_per_s=round(B / fill_ms * 1e3, 1),
               index_build_from_raw_ms=round(raw_ms, 4), index_build_from_raw_ms_repeat=round(raw_ms2, 4),
               index_build_from_dpt_m_ms=round(m_ms, 4), index_build_calls=[raw_n, m_n])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
