"""Developer tool: GPU time of the segment sum (``ffb6d_segment_plan`` and ``ffb6d_segment_sum``, the backward of the
restructured fusion stage's gathered addend) at the seven p2r stage shapes, with the p2r indices of synthetic
480x640 frames from build_ffb6d_indices.  CUDA events, after warm-up, each timed window >= --min-s of work.  The sum
is HBM bound: its algorithmic bytes are dz read once (4 B C P), the plan's pixel list and offsets, and the output
(4 B C N'); they are reported as GB/s and as a fraction of the H100 SXM's 3.35 TB/s.  Prints one JSON line with the
card's name and power limit read in the same run.

usage: python tools/segment_sum_bench.py [--batch 8] [--min-s 1.0]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from fill_bench import card, time_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--min-s", type=float, default=1.0)
    args = ap.parse_args()
    from ffb6d_b200 import ops
    from ffb6d_b200 import tables as T
    from ffb6d_b200.schedule import build_ffb6d_indices
    from ffb6d_b200.synthetic import make_batch

    dev = torch.device("cuda:0")
    B = args.batch
    batch = make_batch(list(range(B)))
    inputs = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(dev), torch.from_numpy(batch["dpt_xyz"]).to(dev))
    n = [T.set_size(("cld", i)) for i in range(5)]
    stages = [("ds%d" % i, "p2r_ds_nei_idx%d" % i, T.DS_RGB_OC[i], n[i + 1]) for i in range(4)]
    stages += [("up%d" % i, "p2r_up_nei_idx%d" % i, T.UP_RGB_OC[i], n[3 - i]) for i in range(3)]
    g = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for name, key, C, na in stages:
        idx = inputs[key]
        P = idx.shape[1]
        grad = torch.randn((B, C, P), generator=g, device=dev)
        plan = ops.segment_plan(idx, na)
        largest = int(max(torch.bincount(idx[b].reshape(-1).long(), minlength=na).max() for b in range(B)))
        t_plan, _ = time_ms(lambda: ops.segment_plan(idx, na), args.min_s)
        t_sum, n_sum = time_ms(lambda: ops.segment_sum(grad, None, na, plan=plan), args.min_s)
        nbytes = B * (4 * C * P + 4 * P + 4 * (na + 1) + 4 * C * na)
        rows.append({"stage": name, "C": C, "P": P, "segments": na, "largest_segment": largest,
                     "plan_us": 1e3 * t_plan, "sum_us": 1e3 * t_sum, "sum_calls": n_sum,
                     "sum_GBps": nbytes / (t_sum * 1e-3) / 1e9,
                     "sum_hbm_fraction": nbytes / (t_sum * 1e-3) / HBM_BYTES_PER_S})
        print("%-4s C=%4d P=%6d N'=%5d largest=%5d  plan %8.1f us  sum %8.1f us  %7.1f GB/s  %.2f of 3.35 TB/s"
              % (name, C, P, na, largest, rows[-1]["plan_us"], rows[-1]["sum_us"], rows[-1]["sum_GBps"],
                 rows[-1]["sum_hbm_fraction"]), file=sys.stderr)
    line = {"metric": "segment plan + sum at the p2r stage shapes", "batch": B, "stages": rows}
    line.update(card())
    print(json.dumps(line))


if __name__ == "__main__":
    main()
