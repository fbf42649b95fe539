"""Seeded inputs of the drawing cases (tests/golden/vis_cases.npz stores only the reference's outputs on them)."""
import hashlib

import numpy as np

from ffb6d_b200.synthetic import INTRINSICS, make_frame

K_YCB = INTRINSICS["ycb_K1"]
K_LM = INTRINSICS["linemod"]
K_INT = np.array([[2.0, 0.0, 3.0], [0.0, 4.0, -5.0], [0.0, 0.0, 1.0]])     # integer K: exact half-pixel ties
PROJ_SIZES = (1, 2, 3, 8, 9, 2621, 12288)
STORE_WHOLE = 1000              # projections of at most this many points are stored whole, larger ones as sha256
SMALL_H, SMALL_W = 64, 80


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def rotation(rs):
    q = rs.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose_in_front(rs, z=0.9):
    t = np.array([rs.uniform(-0.2, 0.2), rs.uniform(-0.15, 0.15), z + rs.uniform(-0.1, 0.3)])
    return np.concatenate((rotation(rs), t[:, None]), axis=1)


def mesh(rs, n, dtype):
    return (rs.normal(0, 0.04, (n, 3)) * [1.0, 0.8, 0.6]).astype(dtype)


def tie_points(rs, n, dtype):
    """Points whose pixel under K_INT is exactly k + 0.5 in u or v (both parities of k, both signs)."""
    z = 2.0 ** rs.randint(-2, 3, n)
    ku = rs.randint(-300, 300, n) + 0.5
    kv = rs.randint(-300, 300, n) + 0.5
    x = ((ku - 3.0) * z) / 2.0                    # 2 x / z + 3 = ku
    y = ((kv + 5.0) * z) / 4.0                    # 4 y / z - 5 = kv
    x[::3] = np.round(x[::3] * 4) / 4             # and some points off the tie
    return np.stack((x, y, z), axis=1).astype(dtype)


def edge_points(dtype):
    """Depths below 1e-8, negative and zero; NaN and inf coordinates; pixels beyond int32."""
    p = np.array([[0.1, 0.1, 1e-9], [0.1, 0.1, -0.5], [0.1, -0.2, 0.0], [0.0, 0.0, 0.0], [np.nan, 0.1, 1.0],
                  [0.1, np.nan, 1.0], [0.1, 0.1, np.nan], [np.inf, 0.1, 1.0], [0.1, -np.inf, 1.0], [0.1, 0.1, np.inf],
                  [1e12, 0.1, 1.0], [-1e12, 0.1, 1.0], [0.1, 3e6, 1.0], [2.1e6, -2.1e6, 1.0], [5.0, 5.0, 1e-7],
                  [1e-3, 1e-3, 1e-8]], np.float64)
    return p.astype(dtype)


def proj_cases():
    """{name: (p3d, cam_scale, K, pose or None)}."""
    rs = np.random.RandomState(11)
    out = {}
    for n in PROJ_SIZES:
        out["f32_%d" % n] = (mesh(rs, n, np.float32) + np.float32([0, 0, 0.9]), 1.0, K_YCB, None)
        out["f64_pose_%d" % n] = (mesh(rs, n, np.float64), 1.0, K_LM, pose_in_front(rs))
    out["f32_pose"] = (mesh(rs, 2621, np.float32), 1.0, K_YCB, pose_in_front(rs))
    out["f32_scale"] = ((mesh(rs, 500, np.float32) + np.float32([0, 0, 0.9])) / np.float32(1000.0), 1000.0, K_YCB,
                        None)
    out["f64_scale"] = (mesh(rs, 500, np.float64) + [0, 0, 0.9], 0.37, K_LM, None)
    for dt in (np.float32, np.float64):
        name = "f32" if dt == np.float32 else "f64"
        out["ties_" + name] = (tie_points(rs, 600, dt), 1.0, K_INT, None)
        out["edge_" + name] = (edge_points(dt), 1.0, K_YCB, None)
    out["ties_pose"] = (tie_points(rs, 600, np.float64), 1.0, K_INT, np.eye(3, 4))
    out["edge_pose"] = (edge_points(np.float64), 1.0, K_YCB, np.concatenate((np.eye(3), [[0.0], [0.0], [0.0]]), 1))
    return out


def small_background(seed):
    return np.random.RandomState(seed).randint(0, 256, (SMALL_H, SMALL_W, 3)).astype(np.uint8)


def draw_cases():
    """{name: (background [64,80,3] uint8, [(p2ds [n,2] int32, r, colour list)])}: the reference's draw_p2ds applied
    in order.  Borders, every radius of {0, 1, 2, 3, 4, 5, 64}, overlapping sets, per-row and single colours."""
    rs = np.random.RandomState(12)
    H, W = SMALL_H, SMALL_W
    xs = [-9, -1, 0, 1, 2, W // 2, W - 2, W - 1, W, W + 1, W + 30, -2 ** 31, 2 ** 31 - 1]
    ys = [-9, -1, 0, 1, 2, H // 2, H - 2, H - 1, H, H + 1, H + 30, -2 ** 31, 2 ** 31 - 1]
    border = np.array([(x, y) for x in xs for y in ys], np.int32)
    out = {}
    for r in (0, 1, 2, 3, 4, 5, 64):
        cols = [tuple(int(v) for v in c) for c in rs.randint(0, 256, (len(border), 3))]
        out["border_r%d" % r] = (small_background(r), [(border, r, cols)])
    sets = []
    for k in range(5):
        n = rs.randint(5, 60)
        p = np.stack((rs.randint(-5, W + 5, n), rs.randint(-5, H + 5, n)), 1).astype(np.int32)
        c = [tuple(int(v) for v in rs.randint(0, 256, 3))]
        if k % 2:
            c = [tuple(int(v) for v in cc) for cc in rs.randint(0, 256, (n, 3))]
        sets.append((p, [1, 3, 2, 4, 0][k], c))
    out["overlap"] = (small_background(20), sets)
    out["overlap_rev"] = (small_background(21), sets[::-1])
    same = np.repeat(np.array([[W // 3, H // 3]], np.int32), 4, 0)
    out["same_point"] = (small_background(22), [(same, 3, [(1, 2, 3), (4, 5, 6), (7, 8, 9), (10, 11, 12)]),
                                                 (same[:1], 1, [(200, 100, 50)])])
    return out


def demo_frames():
    """The demo's inputs on two 480 x 640 frames: {dataset: dict(rgb [3,H,W] float32, cls_ids [22,1], pred_cls_ids,
    pred_pose_lst, mesh_pts {id: [P,3]}, K, obj_id)}.  YCB meshes are float32 (``points.xyz``), LineMOD float64."""
    rs = np.random.RandomState(13)
    ycb_ids = [3, 7, 12, 15, 20]
    ids = np.zeros((22, 1), np.int32)
    ids[:5, 0] = ycb_ids
    ycb = dict(rgb=rs.randint(0, 256, (3, 480, 640)).astype(np.float32), cls_ids=ids,
               pred_cls_ids=np.array([3, 9, 12, 15, 20]), pred_pose_lst=[pose_in_front(rs) for _ in range(5)],
               mesh_pts={c: mesh(rs, 2621, np.float32) for c in ycb_ids + [9]}, K=K_YCB, obj_id=-1)
    lm_ids = np.zeros((22, 1), np.int32)
    lm_ids[0, 0] = 1
    lm = dict(rgb=rs.randint(0, 256, (3, 480, 640)).astype(np.float32), cls_ids=lm_ids, pred_cls_ids=None,
              pred_pose_lst=[pose_in_front(rs, 0.6)], mesh_pts={8: mesh(rs, 2000, np.float64)}, K=K_LM, obj_id=8)
    return {"ycb": ycb, "linemod": lm}


def view_labels_frame():
    """``(cld_cn [3,N] float32, labels [N] int64)``: a 12 288-point synthetic frame, YCB labels 0 .. 21."""
    fr = make_frame(14, intrinsics="ycb_K1")
    labels = np.random.RandomState(14).randint(0, 22, fr["cld"].shape[0])
    return fr["cld"].T.copy(), labels
