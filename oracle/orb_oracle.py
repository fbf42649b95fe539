"""numpy restatement of OpenCV's ORB keypoint detector at ``cv2.ORB_create()``'s defaults, and of the reference's lift
of those keypoints onto the mesh (utils/dataset_tools/rgbd_rnder_sift_kp3ds.py:138-166), DESIGN.md §4.32.

Each step is its own function so that each can be pinned to cv2 on its own (tests/golden/check_orb_opencv.py):

  grey            ``(3735 B + 19235 G + 9798 R + 2^14) >> 15``, exact integers (cvtColor's 15-bit BGR2GRAY)
  resize_exact    ``INTER_LINEAR_EXACT``: float64 source coordinates, 8-bit fixed-point weights, a horizontal then a
                  vertical pass in integers, ``(v + 2^15) >> 16``
  pyramid         8 levels, each resized from the previous level to ``cvRound(cols * (1 / s_l)) x
                  cvRound(rows * (1 / s_l))`` with ``s_l = float32(pow(double(1.2f), l))``, all in float32
  fast_scores     FAST-9/16 at threshold 20: ``M - 1`` where ``M`` is the larger of the best arc-of-9 minimum of
                  ``v - p`` and of ``p - v``, kept where ``M > 20`` (exact integers)
  nms             strict 3x3 maximum of the score map (0 where no corner)
  border          ``31 <= x < w - 31`` and ``31 <= y < h - 31``
  retain_best     every point whose response is >= the n-th best (the set; OpenCV's order is nth_element's)
  harris          7x7 Sobel sums in integers, the response in float32 with every operation rounded on its own
  level_budgets   ``nfeaturesPerLevel`` for 500 features, scale 1.2f, 8 levels, in float32 with cvRound
  level_to_image  ``float32(x_l) * float32(pow(double(1.2f), l))``

Output order is canonical, level then raster order; OpenCV's is not a contract (retainBest's nth_element), so the
keypoints are compared as sets.

The lift restates ``gen_one_zbuf_render`` after the render for a depth ``zbuf`` (float32 metres) and the tool's K
(an int64 array): the pixel ``(int(pt.y), int(pt.x))``, ``dpt_2_cld`` with ``cam_scale = 1`` -- under numpy >= 2 an
int64 scalar is not a weak operand, so ``(u - cx) * z / fx`` is float64 from float32 ``u`` and ``z`` --,
``filter_pcld`` (finite x, z > 1e-8) and ``(p - t) . R`` into the object frame, each output coordinate summed left
to right in float64 with every product rounded (no fused multiply-add).
"""
import math

import numpy as np

N_FEATURES = 500
N_LEVELS = 8
SCALE_FACTOR = float(np.float32(1.2))      # ORB_create's scaleFactor=1.2f, held as a double
FAST_THRESHOLD = 20
EDGE_THRESHOLD = 31
HARRIS_BLOCK = 7
HARRIS_K = np.float32(0.04)
MIN_RENDER_PIXELS = 500                    # gen_one_zbuf_render returns None below this many drawn pixels

# FAST's Bresenham circle of radius 3, (dx, dy), in order around it
CIRCLE = ((0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
          (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3))


def cv_round(x):
    """cvRound: round half to even (lrint in the default rounding mode)."""
    return int(np.rint(x))


def grey(rgb):
    """ORB's BGR->grey of an RGB uint8 image ``[H,W,3]`` (the tool passes BGR; this takes the channels by name)."""
    x = rgb.astype(np.int64)
    return ((3735 * x[..., 2] + 19235 * x[..., 1] + 9798 * x[..., 0] + (1 << 14)) >> 15).astype(np.uint8)


def _taps(src, dst):
    """Source index and the two 8-bit weights of each destination coordinate, clamped to the edge."""
    scale = float(src) / float(dst)
    f = (np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5
    s = np.floor(f).astype(np.int64)
    w1 = np.rint((f - s) * 256.0).astype(np.int64)
    lo, hi = s < 0, s >= src - 1
    s = np.where(lo, 0, np.where(hi, src - 1, s))
    w1 = np.where(lo | hi, 0, w1)
    s1 = np.minimum(s + 1, src - 1)
    return s, s1, 256 - w1, w1


def resize_exact(img, dw, dh):
    """cv2.resize(img, (dw, dh), interpolation=INTER_LINEAR_EXACT) of a uint8 image ``[h,w]``."""
    h, w = img.shape
    x0, x1, wx0, wx1 = _taps(w, dw)
    y0, y1, wy0, wy1 = _taps(h, dh)
    a = img.astype(np.int64)
    row = a[:, x0] * wx0 + a[:, x1] * wx1                     # [h, dw], 8 fractional bits
    v = row[y0, :] * wy0[:, None] + row[y1, :] * wy1[:, None]   # 16 fractional bits
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def level_scale(l):
    """The level's scale as a float32, ``float32(pow(double(1.2f), l))``."""
    return np.float32(math.pow(SCALE_FACTOR, l))


def level_sizes(h, w):
    """``[(h_l, w_l)]`` of the 8 levels."""
    out = []
    for l in range(N_LEVELS):
        s = level_scale(l)
        inv = np.float32(1) / s
        out.append((cv_round(np.float32(h) * inv), cv_round(np.float32(w) * inv)))
    return out


def pyramid(g):
    """The 8 level images of a grey image, each resized from the one before."""
    levels = [g]
    for h, w in level_sizes(*g.shape)[1:]:
        levels.append(resize_exact(levels[-1], w, h))
    return levels


def fast_scores(img, threshold=FAST_THRESHOLD):
    """FAST-9/16 corner score map ``[h,w]`` int: ``M - 1`` where ``M > threshold``, else 0.  Only pixels at least 3
    from every edge are tested."""
    h, w = img.shape
    out = np.zeros((h, w), np.int64)
    if h < 7 or w < 7:
        return out
    a = img.astype(np.int64)
    v = a[3:h - 3, 3:w - 3]
    d = np.stack([v - a[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] for dx, dy in CIRCLE])   # [16, ...]
    best = np.full(v.shape, -1 << 30, np.int64)
    for sign in (1, -1):
        e = sign * d
        for k in range(16):
            arc = np.min(np.stack([e[(k + i) % 16] for i in range(9)]), 0)
            best = np.maximum(best, arc)
    out[3:h - 3, 3:w - 3] = np.where(best > threshold, best - 1, 0)
    return out


def nms(score):
    """Strict 3x3 non-maximum suppression: a keypoint where the score is > 0 and > each of its eight neighbours."""
    h, w = score.shape
    p = np.zeros((h + 2, w + 2), score.dtype)
    p[1:-1, 1:-1] = score
    keep = score > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dy or dx:
                keep &= score > p[1 + dy:h + 1 + dy, 1 + dx:w + 1 + dx]
    return keep


def border(ys, xs, h, w, b=EDGE_THRESHOLD):
    """runByImageBorder's mask."""
    return (xs >= b) & (xs < w - b) & (ys >= b) & (ys < h - b)


def retain_best(response, n):
    """retainBest's kept set as a mask: everything when there are at most n, nothing for n = 0, else every point
    whose response is >= the n-th largest."""
    m = len(response)
    if m <= n:
        return np.ones(m, bool)
    if n == 0:
        return np.zeros(m, bool)
    cut = np.sort(response)[::-1][n - 1]
    return response >= cut


def harris(img, ys, xs):
    """HarrisResponses of 7x7 blocks at level coordinates, float32 [n]."""
    f = np.float32
    a = img.astype(np.int64)
    r = HARRIS_BLOCK // 2
    out = np.empty(len(ys), np.float32)
    scale = f(1.0) / (f(4.0) * f(HARRIS_BLOCK) * f(255.0))
    s4 = scale * scale * scale * scale
    for i, (y, x) in enumerate(zip(ys, xs)):
        blk = a[y - r - 1:y + r + 2, x - r - 1:x + r + 2]
        c = blk[1:-1, 1:-1]
        Ix = (blk[1:-1, 2:] - blk[1:-1, :-2]) * 2 + (blk[:-2, 2:] - blk[:-2, :-2]) + (blk[2:, 2:] - blk[2:, :-2])
        Iy = (blk[2:, 1:-1] - blk[:-2, 1:-1]) * 2 + (blk[2:, :-2] - blk[:-2, :-2]) + (blk[2:, 2:] - blk[:-2, 2:])
        assert c.shape == (HARRIS_BLOCK, HARRIS_BLOCK)
        A, B, C = f(np.sum(Ix * Ix)), f(np.sum(Iy * Iy)), f(np.sum(Ix * Iy))
        t = A + B
        out[i] = ((A * B - C * C) - HARRIS_K * t * t) * s4
    return out


def level_budgets(nfeatures=N_FEATURES, nlevels=N_LEVELS):
    """nfeaturesPerLevel."""
    f = np.float32
    factor = f(1.0 / SCALE_FACTOR)
    nd = f(nfeatures) * (f(1) - factor) / (f(1) - f(math.pow(float(factor), nlevels)))
    out, total = [], 0
    for _ in range(nlevels - 1):
        n = cv_round(nd)
        out.append(n)
        total += n
        nd = f(nd * factor)
    out.append(max(nfeatures - total, 0))
    return out


def level_to_image(xs, l):
    """Level coordinates -> full-image float32 coordinates."""
    return np.asarray(xs, np.float32) * level_scale(l)


def detect(rgb):
    """ORB keypoints of one RGB uint8 image ``[H,W,3]`` (or a grey ``[H,W]``): dict of ``pt [n,2]`` float32 (x, y),
    ``octave [n]`` int32 and ``response [n]`` float32 (Harris), in level then raster order."""
    g = grey(rgb) if rgb.ndim == 3 else rgb
    budgets = level_budgets()
    pts, octs, resp = [], [], []
    for l, img in enumerate(pyramid(g)):
        h, w = img.shape
        score = fast_scores(img)
        ys, xs = np.nonzero(nms(score))                           # raster order
        keep = border(ys, xs, h, w)
        ys, xs = ys[keep], xs[keep]
        sc = score[ys, xs].astype(np.float32)
        keep = retain_best(sc, 2 * budgets[l])
        ys, xs = ys[keep], xs[keep]
        hr = harris(img, ys, xs)
        keep = retain_best(hr, budgets[l])
        ys, xs, hr = ys[keep], xs[keep], hr[keep]
        pts.append(np.stack([level_to_image(xs, l), level_to_image(ys, l)], 1).reshape(-1, 2))
        octs.append(np.full(len(ys), l, np.int32))
        resp.append(hr)
    return dict(pt=np.concatenate(pts).astype(np.float32), octave=np.concatenate(octs), response=np.concatenate(resp))


# ---------------------------------------------------------------------------------------------------------- the lift

def camera_positions(n1, n2, r):
    """``PoseUtils.CameraPositions``: ``n1 x n2`` points on a sphere of radius r (float64)."""
    theta = np.linspace(0.1, np.pi, n1 + 1)[:-1]
    phi = np.linspace(0, 2 * np.pi, n2 + 1)[:-1]
    return [(r * math.sin(t) * math.cos(p), r * math.sin(t) * math.sin(p), r * math.cos(t))
            for t in theta for p in phi]


def camera_pose(T):
    """``PoseUtils.getCameraPose``: the OpenGL camera at T looking at the origin, [4,4]."""
    z = np.array(T)
    z = z / np.linalg.norm(z)
    x = -np.cross(z, np.array([0, 0, 1]))
    x = x / np.linalg.norm(x)
    y = np.cross(z, x)
    y = y / np.linalg.norm(y)
    pose = np.eye(4)
    pose[:3, :3] = np.array([x, y, z]).T
    pose[:3, 3] = T
    return pose


def o2c_pose(cam):
    """``PoseUtils.get_o2c_pose_cv(cam, np.eye(4))``: object (= world) to OpenCV camera, [4,4]."""
    R_bcam2cv = np.array([(1, 0, 0), (0, -1, 0), (0, 0, -1)])
    R_w2b = cam[:3, :3].T
    T_w2b = -1 * R_w2b @ cam[:3, 3]
    RT = np.eye(4)
    RT[:3, :3] = R_bcam2cv @ R_w2b
    RT[:3, 3] = R_bcam2cv @ T_w2b
    return np.matmul(RT, np.eye(4))


def sphere_poses(radius, n_longitude=3, n_latitude=3):
    """The tool's view poses for an object of box radius ``radius``: ``[n_longitude * n_latitude, 4, 4]`` float64."""
    sph_r = radius / 0.035 * 0.18
    return np.stack([o2c_pose(camera_pose(p)) for p in camera_positions(n_longitude, n_latitude, sph_r)])


def lift(pt, zbuf, K, RT):
    """One view's keypoints ``pt [n,2]`` (float32 image coordinates) on depth ``zbuf [H,W]`` (float32 metres, 0 where
    nothing is drawn) -> object-frame points ``[m,3]`` float64 and the mask of kept keypoints ``[n]``."""
    K = np.asarray(K, np.float64)
    xy = np.asarray(pt, np.float32).astype(np.int32)
    u, v = xy[:, 0], xy[:, 1]
    z = zbuf[v, u].astype(np.float64)
    x = (u.astype(np.float32).astype(np.float64) - K[0, 2]) * z / K[0, 0]
    y = (v.astype(np.float32).astype(np.float64) - K[1, 2]) * z / K[1, 1]
    ok = np.isfinite(x) & (z > 1e-8)
    p = np.stack([x, y, z], 1)[ok] - RT[:3, 3]
    R = RT[:3, :3]
    out = np.stack([(p[:, 0] * R[0, j] + p[:, 1] * R[1, j]) + p[:, 2] * R[2, j] for j in range(3)], 1)
    return out, ok
