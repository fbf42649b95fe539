"""Developer tool: GPU time of the sampled points' item arrays (``ffb6d_point_item``, captured in a CUDA graph) and of
the whole batch ``get_item`` (``schedule.build_ffb6d_item``: depth completion, sampling, the 22 searches and the
point arrays) for a batch of 480x640 YCB-like frames.  CUDA events, after warm-up, each timed window >= --min-s of
work.  Prints one JSON line with the card's name and power limit read in the same run, and the bytes the point
kernel must move at least (from shapes: its stores, ``choose``, and one 32-byte sector per point of each of the
four images it reads) over its time.

usage: python tools/item_bench.py [--batch 32] [--points 12288] [--kps 8] [--min-s 1.0]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from fill_bench import capture, card, time_ms  # noqa: E402


def point_item_bytes(B, N, n_kps):
    stores = N * 4 * (9 + 1 + 3 * n_kps + 3)
    reads = N * 4 + 4 * 32 * N                       # choose; depth, rgb, labels, normal map: a sector per point
    return B * (stores + reads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--points", type=int, default=12288)
    ap.add_argument("--kps", type=int, default=8)
    ap.add_argument("--min-s", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("item_bench.py needs a GPU")
    import ffb6d_b200 as F
    from ffb6d_b200.item import pose_gt_objects
    from ffb6d_b200.ops import intrinsics_to_device
    from ffb6d_b200.synthetic import INTRINSICS, make_item_frame

    dev = torch.device("cuda:0")
    B, N, n_kps = args.batch, args.points, args.kps
    frames = [make_item_frame(s, n_kps=n_kps, cls_ids=(1, 4, 9, 15), blobs=(1, 4, 9, 15)) for s in range(B)]
    objs = [pose_gt_objects(f["poses"], f["cls_ids"], f["kps"], f["ctrs"], 22, n_kps) for f in frames]
    obj = {k: torch.from_numpy(np.stack([o[k] for o in objs])).to(dev) for k in objs[0]}
    raw = torch.from_numpy(np.stack([f["raw"] for f in frames])).to(dev)
    rgb = torch.from_numpy(np.stack([f["rgb"] for f in frames])).to(dev)
    labels = torch.from_numpy(np.stack([f["labels"] for f in frames])).to(dev)
    nrm = torch.from_numpy(np.stack([f["nrm"] for f in frames])).to(dev)
    K = intrinsics_to_device(INTRINSICS["ycb_K1"], dev)

    item = F.build_ffb6d_item(raw, 10000.0, K, rgb, labels, nrm, obj, N, seed=1)
    depth_m, choose = item["dpt_map_m"], item["choose"]

    def points():
        F.point_item(depth_m, K, choose, rgb, labels, nrm, obj["obj_cls"], obj["obj_kps"], obj["obj_ctr"])

    def whole():
        F.build_ffb6d_item(raw, 10000.0, K, rgb, labels, nrm, obj, N, seed=1)

    pt_ms, pt_n = time_ms(capture(points), args.min_s)
    item_ms, item_n = time_ms(whole, args.min_s)
    nbytes = point_item_bytes(B, N, n_kps)
    print(json.dumps(dict(card(), batch=B, points=N, n_kps=n_kps,
                          point_item_ms=round(pt_ms, 4), point_item_calls=pt_n,
                          point_item_min_bytes=nbytes, point_item_gbps=round(nbytes / pt_ms / 1e6, 1),
                          point_item_share_of_3350gbps=round(nbytes / pt_ms / 1e6 / 3350.0, 3),
                          build_item_ms=round(item_ms, 3), build_item_calls=item_n)))


if __name__ == "__main__":
    main()
