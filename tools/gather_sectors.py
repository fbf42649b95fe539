"""Developer tool: the HBM read floor of every gather of the pass, from the pass's actual indices.

For each gather of tables.gather_schedule it counts, per frame, the distinct 32-, 64- and 128-byte units of one
channel row that the frame's indices touch (NCHW rows: every channel reads the same positions), times C and the
batch.  A gather that fetches each touched unit from HBM once reads that unit's floor.  Next to it: the whole source
tensor and the bench's algorithmic bytes (tables.gather_alg_bytes), and, given the per-op table of
`bench.py --per-op` (its stderr), each gather's time, its rate over the 128 B floor and that floor's time at the HBM
peak as a fraction of the measured time.  On the B200 the sparse long-row gathers read from DRAM what their 128 B
floor says (DESIGN §4.2): whole 128-byte lines, each once.

Runs on the CPU from the synthetic frames: the indices come from an exact KNN (scipy) on the same point sets as
the pass (cloud levels = prefixes of the shuffled cloud, image levels = strided pixels of the depth map).

    python tools/gather_sectors.py [--frames 1] [--batch 32] [--per-op bench.err] [--peak-gbs 3350]
"""
import argparse
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ffb6d_b200.synthetic import make_frame, image_pyramid_np  # noqa: E402
from ffb6d_b200.tables import gather_alg_bytes, gather_schedule, knn_schedule, set_size  # noqa: E402


def frame_indices(seed, n_points):
    """{index key: [Q, K] int64} of one synthetic frame: the 22 searches of the schedule (exact KNN) + `choose`."""
    from scipy.spatial import cKDTree
    fr = make_frame(seed, n_points=n_points)
    sets = {("cld", i): fr["cld"][: set_size(("cld", i), n_points)] for i in range(5)}
    for sr, pts in image_pyramid_np(fr["dpt_xyz"]).items():
        sets[("img", sr)] = pts
    out = {"choose": fr["choose"].reshape(-1, 1).astype(np.int64)}
    trees = {}
    for key, s, q, k in knn_schedule(n_points):
        if s not in trees:
            trees[s] = cKDTree(sets[s].astype(np.float64))
        _, idx = trees[s].query(sets[q].astype(np.float64), k=k)
        out[key] = np.asarray(idx, dtype=np.int64).reshape(len(sets[q]), k)
    for i in range(4):             # cld_sub_idx_i = the first N_{i+1} rows of cld_nei_idx_i (schedule.py)
        out["cld_sub_idx%d" % i] = out["cld_nei_idx%d" % i][: set_size(("cld", i + 1), n_points)]
    return out


def read_per_op(path):
    """{index key: ms per step} from the per-op lines of `bench.py --per-op`."""
    ms = {}
    with open(path) as fh:
        for line in fh:
            m = re.match(r"gather:(\S+?):\S+\s+([0-9.]+) ms/step", line)
            if m:
                ms[m.group(1)] = float(m.group(2))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1, help="synthetic frames (seeds 0..n-1) averaged per frame")
    ap.add_argument("--batch", type=int, default=32, help="frames per step the floors are scaled to")
    ap.add_argument("--n-points", type=int, default=12288)
    ap.add_argument("--per-op", default=None, help="stderr of `bench.py --per-op` (per-gather ms per step)")
    ap.add_argument("--peak-gbs", type=float, default=3350.0, help="HBM peak for the floor's time (H100 SXM: 3350)")
    args = ap.parse_args()

    sched = gather_schedule(args.n_points)
    units = {}                    # key -> touched [32 B, 64 B, 128 B] units per channel row, summed over frames
    for seed in range(args.frames):
        idx = frame_indices(seed, args.n_points)
        for op, key, C, S, Q, K in sched:
            flat = idx[key][:Q].reshape(-1)
            u = units.setdefault(key, [0, 0, 0])
            for i, floats in enumerate((8, 16, 32)):
                u[i] += len(np.unique(flat // floats))
    ms = read_per_op(args.per_op) if args.per_op else {}
    scale = args.batch / float(args.frames)
    mb = 1e-6
    hdr = "%-18s %5s %7s %6s %3s %10s %10s %11s %10s %10s" % (
        "gather", "C", "S", "Q", "K", "floor32 MB", "floor64 MB", "floor128 MB", "tensor MB", "alg MB")
    if ms:
        hdr += " %9s %12s %13s" % ("ms/step", "GB/s @128B", "floor128/time")
    print(hdr)
    for op, key, C, S, Q, K in sched:
        f32, f64, f128 = (n * size * C * scale for n, size in zip(units[key], (32, 64, 128)))
        line = "%-18s %5d %7d %6d %3d %10.0f %10.0f %11.0f %10.0f %10.0f" % (
            key, C, S, Q, K, f32 * mb, f64 * mb, f128 * mb, 4.0 * C * S * args.batch * mb,
            gather_alg_bytes(C, S, Q, K) * args.batch * mb)
        if key in ms:
            t = ms[key] * 1e-3
            line += " %9.3f %12.0f %13.2f" % (ms[key], f128 / t * 1e-9, f128 / (args.peak_gbs * 1e9) / t)
        print(line)


if __name__ == "__main__":
    main()
