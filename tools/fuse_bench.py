"""LineMOD's fuse frames on the device (``fuse_rgbd``, DESIGN.md §4.34, §8): the compositor's device time per batch,
and what fused frames cost a LineMOD graphed training step.

    python tools/fuse_bench.py [--repeats 3] [--reps 50] [--steps 10] [--out results/fuse_bench.json]

* ``fuse_rgbd`` of B = 1, 8 and 32 frames of 480x640 with 13 slots each, drawn by ``draw_fuse_frame`` from a table of
  52 crops (13 classes, 4 crops each) cut from renders of the reference's example ape at seeded poses (0.3 to 0.8 m,
  LineMOD's camera), pasted over a background (``out=``, as the training path does): device time from CUDA events
  around ``--reps`` calls.
* ``GraphedFrameTrainStep`` at config 3 (LineMOD, B = 8, 2 classes, 12 800 points, fused image head): wall ms per
  step, each window ending in one synchronise, with half of the frames fused (``crops=``) against the same batches
  without fuse keys; both arms carry a per-frame ``K`` and use ``normals="device"`` (which ``crops=`` requires).

The arms alternate over ``--repeats`` windows; the median and range are reported with the card's name and power limit
read in the same run.  Weights are untrained and seeded."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ffb6d_b200 as F                                                        # noqa: E402
from ffb6d_b200.fuse_frames import FUSE_KEYS, FuseCropTable, draw_fuse_frame, unfused_keys   # noqa: E402
from ffb6d_b200.model import FFB6D                                            # noqa: E402
from ffb6d_b200.render import RenderMeshTable                                 # noqa: E402
from ffb6d_b200.synthetic import INTRINSICS                                   # noqa: E402
from frame_batches import CAM_SCALE, make_train_batch                         # noqa: E402

H, W, N = 480, 640, 480 * 640 // 24
K = INTRINSICS["linemod"]
N_CLS, PER_CLS, SLOTS = 13, 4, 13


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return dict(gpu=name, power_limit=power)


def summary(xs):
    s = sorted(xs)
    return dict(median=s[len(s) // 2], min=s[0], max=s[-1], windows=xs)


def ape():
    z = np.load(os.path.join(ROOT, "tests", "golden", "render_ape.npz"))
    return z["xyz"] / np.float32(1000.0), z["faces"], z["rgb"]


def poses(n, seed):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        q = rs.normal(size=4)
        q /= np.linalg.norm(q)
        a, b, c, d = q
        Rm = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                       [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                       [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
        t = [rs.uniform(-0.05, 0.05), rs.uniform(-0.05, 0.05), rs.uniform(0.3, 0.8)]
        out.append(np.concatenate([Rm, np.array(t)[:, None]], 1))
    return np.stack(out).astype(np.float32)[:, None]


def crop_table(h, w, n_cls):
    """Crops of ape renders at (h, w), ``PER_CLS`` per class over ``n_cls`` classes, over a random background."""
    n = n_cls * PER_CLS
    mesh = RenderMeshTable([ape()])
    Kh = K * np.array([[w / W], [h / H], [1.0]])
    out = (torch.zeros((n, h, w), dtype=torch.uint16, device="cuda"),
           torch.zeros((n, h, w, 3), dtype=torch.uint8, device="cuda"),
           torch.zeros((n, h, w), dtype=torch.uint8, device="cuda"))
    F.render_rgbd(mesh, np.zeros((n, 1), np.int32), poses(n, 7), np.full((n, 1), 255, np.uint8), Kh, h, w, out=out)
    dpt, rgb, lab = (t.cpu().numpy() for t in out)
    return FuseCropTable((rgb[k], dpt[k], lab[k], k % n_cls + 1) for k in range(n))


def draws(table, B, seed, h, w, Kb, fused=None):
    rs = np.random.RandomState(seed)
    rows, Ks = [], []
    for b in range(B):
        if fused is None or fused[b]:
            keys, K_f, _ = draw_fuse_frame(rs, table.meta, table.classes[b % len(table.classes)], Kb, h, w)
        else:
            keys, K_f = unfused_keys(table.meta), Kb
        rows.append(keys)
        Ks.append(K_f)
    out = {k: torch.from_numpy(np.stack([np.asarray(r[k]) for r in rows])) for k in FUSE_KEYS}
    out["K"] = torch.from_numpy(np.stack(Ks).astype(np.float64))
    return out


def kernel(repeats, reps):
    table = crop_table(H, W, N_CLS)
    res = dict(crops=len(table), table_bytes=int(table.nbytes), slots=SLOTS)
    cases = {}
    for B in (1, 8, 32):
        d = draws(table, B, 100 + B, H, W, K)
        args = tuple(d[k].cuda() for k in ("fuse_crop", "fuse_offset", "fuse_label"))
        # a background of depth 0: every pixel a crop covers has depth >= 1 mm (the renders' rule), so the nonzero
        # depths count the pasted pixels
        o = (torch.zeros((B, H, W), dtype=torch.uint16, device="cuda"),
             torch.randint(0, 255, (B, H, W, 3), device="cuda").to(torch.uint8),
             torch.zeros((B, H, W), dtype=torch.uint8, device="cuda"))
        for _ in range(3):
            F.fuse_rgbd(table, *args, H, W, out=o)
        cases[B] = dict(args=args, out=o, ms=[])
    torch.cuda.synchronize()
    for _ in range(repeats):                     # the batch sizes alternate within each window round
        for B, c in cases.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                F.fuse_rgbd(table, *c["args"], H, W, out=c["out"])
            e1.record()
            e1.synchronize()
            c["ms"].append(e0.elapsed_time(e1) / reps)
    for B, c in cases.items():
        res["B%d" % B] = dict(ms=summary(c["ms"]), pasted_pixels=int((c["out"][0].to(torch.int32) > 0).sum().item()),
                              target_pixels=int((c["out"][2] > 0).sum().item()))
    return res


def frame_train_step(repeats, steps):
    table = crop_table(H, W, 2)
    half = [i % 2 == 1 for i in range(8)]
    plain, fused = [], []
    for s in (1, 2):
        b = make_train_batch(s, "linemod", 8, H, W, 2)
        del b["nrm_map"]                         # both arms compute the normals on the device (crops= needs it)
        d = draws(table, 8, 50 + s, H, W, K, fused=half)
        plain.append(dict(b, K=d["K"]))
        fused.append(dict(b, **d))
    kw = dict(dataset="linemod", cam_scale=CAM_SCALE["linemod"], K=K, n_points=N, normals="device")
    arms = {}
    for arm, bs, crops in (("decoded", plain, None), ("half_fused", fused, table)):
        torch.manual_seed(0)
        model = FFB6D(n_classes=2, n_pts=N, n_kps=8, fused_image_head=True).cuda().train()
        opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device="cuda"), capturable=True)
        step = F.GraphedFrameTrainStep(model, opt, bs[0], crops=crops, **kw)
        for it in range(3):
            step(bs[it % 2], seed=it)
        arms[arm] = dict(step=step, batches=bs, ms=[])
    torch.cuda.synchronize()
    it = 0
    for _ in range(repeats):
        for a in arms.values():
            t0 = time.perf_counter()
            for _ in range(steps):
                loss, _ = a["step"](a["batches"][it % 2], seed=it)
                it += 1
            torch.cuda.synchronize()
            a["ms"].append((time.perf_counter() - t0) * 1e3 / steps)
            assert torch.isfinite(loss).item()
    return {k: dict(ms_per_step=summary(a["ms"]), captures=a["step"].captures) for k, a in arms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50, help="calls per window (kernel)")
    ap.add_argument("--steps", type=int, default=10, help="training steps per window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fuse_bench needs a GPU")
    res = dict(card(), fuse_rgbd=kernel(args.repeats, args.reps),
               frame_train_step_config3=frame_train_step(args.repeats, args.steps))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
