"""The rasteriser on the device (``render_rgbd``, DESIGN.md §4.31, §8): its device time per batch, the share of faces
the raster queue takes, and what render frames cost a LineMOD graphed training step.

    python tools/render_bench.py [--repeats 3] [--reps 20] [--steps 10] [--out results/render_bench.json]

* ``render_rgbd`` of B = 1, 8 and 32 frames of 480x640, one instance each at seeded poses (0.3 to 0.8 m, LineMOD's
  camera), for the reference's example ape (11 678 faces) and a UV sphere of about 10^6 faces (10 cm radius): device
  time from CUDA events around ``--reps`` calls, with the ``dpt_mm`` output the training path writes.
* The queue share: of the faces that reach the raster stage (not culled, non-zero area, a non-empty pixel box), those
  whose box exceeds FFB6D_RND_BIG_FACE_PIXELS and go to the queue, counted on the host from the oracle's vertex stage
  (the same integers the kernel computes).
* ``GraphedFrameTrainStep`` at config 3 (LineMOD, B = 8, 2 classes, 12 800 points, fused image head): wall ms per
  step, each window ending in one synchronise, with half of the frames rendered from the ape (``meshes=``) against
  the same batches without render keys, both with ``normals="device"`` (which ``meshes=`` requires).

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

import ffb6d_b200 as F                                        # noqa: E402
from ffb6d_b200 import _lib                                   # noqa: E402
from ffb6d_b200.model import FFB6D                            # noqa: E402
from ffb6d_b200.render import RenderMeshTable                 # noqa: E402
from ffb6d_b200.synthetic import INTRINSICS                   # noqa: E402
from frame_batches import CAM_SCALE, make_train_batch         # noqa: E402
from oracle import render_oracle as R                         # noqa: E402

H, W, N = 480, 640, 480 * 640 // 24
K = INTRINSICS["linemod"]
KD = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])


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


def sphere(n_faces=10 ** 6, radius=0.1):
    """A UV sphere of about ``n_faces`` faces, coloured by position."""
    n = int(np.sqrt(n_faces / 2))
    th, ph = np.meshgrid(np.linspace(0, np.pi, n + 1), np.linspace(0, 2 * np.pi, n + 1), indexing="ij")
    xyz = (radius * np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a, b, c, d = i * (n + 1) + j, i * (n + 1) + j + 1, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1
    faces = np.concatenate([np.stack([a, b, d], -1).reshape(-1, 3), np.stack([a, d, c], -1).reshape(-1, 3)])
    rgb = ((xyz / radius + 1) * 127.5).astype(np.uint8)
    return xyz.astype(np.float32), faces.astype(np.int32), rgb


def poses(B, seed):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(B):
        q = rs.normal(size=4)
        q /= np.linalg.norm(q)
        a, b, c, d = q
        Rm = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                       [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                       [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
        t = [rs.uniform(-0.05, 0.05), rs.uniform(-0.05, 0.05), rs.uniform(0.3, 0.8)]
        out.append(np.concatenate([Rm, np.array(t)[:, None]], 1))
    return np.stack(out).astype(np.float32)[:, None]


def queue_share(mesh, RTs):
    """Faces reaching the raster stage, and those sent to the queue, over the batch (host count)."""
    xyz, faces, _ = mesh
    drawn = queued = 0
    for RT in RTs[:, 0]:
        U, V, _, ok = R.vertex_stage(xyz, RT, KD)
        x, y = U[faces], V[faces]
        A = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
        i0, i1 = np.maximum(-((-x.min(1)) >> 8), 0), np.minimum(x.max(1) >> 8, W - 1)
        j0, j1 = np.maximum(-((-y.min(1)) >> 8), 0), np.minimum(y.max(1) >> 8, H - 1)
        live = ok[faces].all(1) & (A != 0) & (i0 <= i1) & (j0 <= j1)
        box = (i1 - i0 + 1) * (j1 - j0 + 1)
        drawn += int(live.sum())
        queued += int((live & (box > _lib.RND_BIG_FACE_PIXELS)).sum())
    return dict(faces_rastered=drawn, faces_queued=queued, share=queued / max(drawn, 1))


def kernel(repeats, reps):
    out = {}
    for name, mesh in (("ape", ape()), ("sphere_1M", sphere())):
        table = RenderMeshTable([mesh])
        res = dict(faces=int(len(mesh[1])))
        for B in (1, 8, 32):
            RTs = poses(B, 100 + B)
            midx = torch.zeros((B, 1), dtype=torch.int32, device="cuda")
            rts = torch.from_numpy(RTs).cuda()
            lab = torch.ones((B, 1), dtype=torch.uint8, device="cuda")
            intr = torch.from_numpy(KD).cuda()
            o = (torch.empty((B, H, W), dtype=torch.uint16, device="cuda"),
                 torch.empty((B, H, W, 3), dtype=torch.uint8, device="cuda"),
                 torch.empty((B, H, W), dtype=torch.uint8, device="cuda"))
            for _ in range(3):
                F.render_rgbd(table, midx, rts, lab, intr, H, W, out=o)
            ms = []
            for _ in range(repeats):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    F.render_rgbd(table, midx, rts, lab, intr, H, W, out=o)
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1) / reps)
            res["B%d" % B] = dict(ms=summary(ms), drawn_pixels=int((o[0].to(torch.int32) > 0).sum().item()),
                                  queue=queue_share(mesh, RTs))
        out[name] = res
    return out


def frame_train_step(repeats, steps):
    table = RenderMeshTable([ape()])
    batches = [make_train_batch(s, "linemod", 8, H, W, 2) for s in (1, 2)]
    for b in batches:
        del b["nrm_map"]                         # both arms compute the normals on the device (meshes= needs it)
    rendered = []
    for s, b in zip((1, 2), batches):
        r = dict(b, rendered=torch.tensor([i % 2 == 0 for i in range(8)]),
                 render_mesh=torch.zeros((8, 1), dtype=torch.int32), render_RTs=torch.from_numpy(poses(8, 50 + s)),
                 render_label=torch.ones((8, 1), dtype=torch.uint8))
        rendered.append(r)
    kw = dict(dataset="linemod", cam_scale=CAM_SCALE["linemod"], K=K, n_points=N, normals="device")
    arms = {}
    for arm, bs, meshes in (("decoded", batches, None), ("half_rendered", rendered, table)):
        torch.manual_seed(0)
        model = FFB6D(n_classes=2, n_pts=N, n_kps=8, fused_image_head=True).cuda().train()
        opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device="cuda"), capturable=True)
        step = F.GraphedFrameTrainStep(model, opt, bs[0], meshes=meshes, **kw)
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
    ap.add_argument("--reps", type=int, default=20, help="calls per window (kernel)")
    ap.add_argument("--steps", type=int, default=10, help="training steps per window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_bench needs a GPU")
    res = dict(card(), render_rgbd=kernel(args.repeats, args.reps),
               frame_train_step_config3=frame_train_step(args.repeats, args.steps))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
