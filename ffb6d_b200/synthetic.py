"""Seeded synthetic RGB-D frames shaped like the reference datasets' output.

Recipe: SURVEY.md §8(d).  Depth ``d(x,y) = 0.8 + 0.3 sin(x/57) cos(y/43) + 0.02 U[0,1)``
metres on a 480x640 grid, ``hole_frac`` of the pixels zeroed (holes become xyz =
(0,0,0), like ``dpt_2_pcld``'s mask, datasets/ycb/ycb_dataset.py:165-176), back-projected
with the LineMOD (or YCB) intrinsics of common.py:144-152; ``choose`` = the first
``n_points`` of a seeded permutation of the valid pixels (no 'wrap' padding, so no
duplicated cloud points: ycb_dataset.py:218-235 pads only when fewer valid pixels exist).
This is input generation (numpy, host); it is not part of the timed hot path.
"""
import numpy as np

INTRINSICS = {
    # common.py:144-152
    "linemod": np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]]),
    "ycb_K1": np.array([[1066.778, 0., 312.9869], [0., 1067.487, 241.3109], [0., 0., 1.]],
                       np.float32).astype(np.float64),
}


def depth_to_xyz(dpt, K):
    """``dpt_2_pcld`` (ycb_dataset.py:165-176) with cam_scale 1: organised cloud [H,W,3]
    float32, zero rows where depth <= 1e-8."""
    H, W = dpt.shape
    xmap, ymap = np.mgrid[:H, :W]          # xmap = row index, ymap = column index (:31-32)
    dpt = dpt.astype(np.float32)
    msk = (dpt > 1e-8).astype(np.float32)
    row = (ymap - K[0][2]) * dpt / K[0][0]
    col = (xmap - K[1][2]) * dpt / K[1][1]
    xyz = np.concatenate((row[..., None], col[..., None], dpt[..., None]), axis=2)
    return (xyz * msk[:, :, None]).astype(np.float32)


def make_frame(seed, n_points=12288, h=480, w=640, hole_frac=0.1, intrinsics="linemod"):
    """One synthetic frame.  Returns a dict with ``dpt_xyz [H,W,3] f32``, ``cld [N,3] f32``,
    ``choose [1,N] int32``, ``depth [H,W] f32`` (metres, 0 at holes), ``cld_rgb_nrm [9,N] f32`` (xyz | rgb in [0,255) | unit normals)."""
    rs = np.random.RandomState(seed)
    ys, xs = np.mgrid[:h, :w]
    d = 0.8 + 0.3 * np.sin(xs / 57.0) * np.cos(ys / 43.0) + 0.02 * rs.rand(h, w)
    d = d.astype(np.float32)
    if hole_frac > 0:
        d[rs.rand(h, w) < hole_frac] = 0.0
    xyz = depth_to_xyz(d, INTRINSICS[intrinsics])
    valid = (d.reshape(-1) > 1e-8).nonzero()[0]
    if len(valid) < n_points:
        raise ValueError("only %d valid pixels for %d points" % (len(valid), n_points))
    choose = valid[rs.permutation(len(valid))[:n_points]].astype(np.int32)
    cld = xyz.reshape(-1, 3)[choose]
    rgb = rs.uniform(0, 255, (n_points, 3)).astype(np.float32)
    nrm = rs.normal(size=(n_points, 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
    return dict(dpt_xyz=xyz, cld=cld, choose=choose[None, :], depth=d,
                cld_rgb_nrm=np.concatenate((cld, rgb, nrm), axis=1).T.copy())


def make_raw_depth(seed, h=480, w=640, cam_scale=10000.0, hole_frac=0.15, far_frac=0.03, block_holes=6,
                   empty_rows=0, empty_cols=()):
    """One raw ``uint16`` depth frame shaped like a YCB-Video ``-depth.png`` (``cam_scale`` raw units per
    metre): the smooth surface of :func:`make_frame` around 1.2 m with a near and a far object, a fraction
    ``hole_frac`` of random missing pixels, ``block_holes`` missing rectangles, ``far_frac`` of pixels
    beyond 3 m (what ``fill_missing`` leaves uninverted), ``empty_rows`` missing leading rows and the
    columns ``empty_cols`` missing entirely."""
    rs = np.random.RandomState(seed)
    ys, xs = np.mgrid[:h, :w]
    d = 1.2 + 0.3 * np.sin(xs / 57.0) * np.cos(ys / 43.0) + 0.02 * rs.rand(h, w)
    d[(ys - 0.6 * h) ** 2 + (xs - 0.3 * w) ** 2 < (0.15 * min(h, w)) ** 2] -= 0.5
    d[(ys > 0.2 * h) & (ys < 0.5 * h) & (xs > 0.6 * w) & (xs < 0.9 * w)] += 0.9
    raw = np.clip(np.round(d * cam_scale), 0, 65535).astype(np.uint16)
    far = rs.rand(h, w) < far_frac
    raw[far] = rs.randint(int(3.0 * cam_scale) + 1, 65536, far.sum())
    raw[rs.rand(h, w) < hole_frac] = 0
    for _ in range(block_holes):
        y0, x0 = rs.randint(0, h), rs.randint(0, w)
        raw[y0:y0 + rs.randint(1, max(2, h // 8)), x0:x0 + rs.randint(1, max(2, w // 8))] = 0
    raw[:empty_rows] = 0
    raw[:, list(empty_cols)] = 0
    return raw


FILL_CAM_SCALE = 10000.0      # YCB-Video's factor_depth


def fill_test_frames():
    """The raw depth frames of tests/golden/fill_cases.npz, by name: two full YCB-like frames and small ones
    for the edge cases of the depth completion (all holes, no holes, a constant frame, raw values at exactly
    1 m and 2 m, beyond 3 m and in 1..100, empty leading rows and columns, sizes that are multiples of no
    tile size, an image smaller than the 9x9 stencil)."""
    rs = np.random.RandomState(17)
    special = np.array([0, 1, 7, 50, 100, 9999, 10000, 10001, 19999, 20000, 20001, 29999, 30000, 30001, 40000,
                        65535], np.uint16)
    sv = rs.choice(special, (23, 29))
    sv[:, 17:] = rs.choice(special[-3:], (23, 12))      # a region beyond 3 m that no valid pixel reaches
    return {
        "full0": make_raw_depth(0),
        "full1": make_raw_depth(1, empty_rows=9, empty_cols=(0, 13, 14, 639)),
        "all_holes": np.zeros((6, 7), np.uint16),
        "constant": np.full((13, 17), 15000, np.uint16),
        "no_holes": make_raw_depth(2, h=21, w=33, hole_frac=0.0, far_frac=0.0, block_holes=0),
        "special_values": sv,
        "empty_top": make_raw_depth(3, h=37, w=91, empty_rows=5, empty_cols=(0, 40, 90)),
        "tiny": make_raw_depth(4, h=3, w=4, hole_frac=0.3, block_holes=0),
    }


def make_batch(seeds, **kw):
    """Stack frames: ``dpt_xyz [B,H,W,3]``, ``cld [B,N,3]``, ``choose [B,1,N]``, ``cld_rgb_nrm [B,9,N]``."""
    frames = [make_frame(s, **kw) for s in seeds]
    return {k: np.stack([f[k] for f in frames]) for k in frames[0]}


def image_pyramid_np(dpt_xyz):
    """numpy twin of schedule.image_pyramid for one frame: {sr: [(H//sr)*(W//sr), 3]}
    (ycb_dataset.py:253-267)."""
    H, W, _ = dpt_xyz.shape
    return {sr: np.ascontiguousarray(dpt_xyz[:(H // sr) * sr:sr, :(W // sr) * sr:sr, :].reshape(-1, 3))
            for sr in (1, 2, 4, 8)}
