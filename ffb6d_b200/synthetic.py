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
    "ycb_K2": np.array([[1077.836, 0., 323.7872], [0., 1078.189, 279.6921], [0., 0., 1.]],
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


def _rotation(rs):
    q, r = np.linalg.qr(rs.randn(3, 3))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def make_item_frame(seed, h=480, w=640, dataset="ycb", n_kps=8, cls_ids=(1, 5, 9), blobs=(1, 5, 9),
                    hole_frac=0.1, nrm_dtype=np.float32, intrinsics=None):
    """The decoded images and pose metadata of one dataset item, seeded: what ``get_item`` reads from disk.

    * ``raw [H,W] uint16``: raw depth (YCB 1e4, LineMOD 1e3 units per metre) around 0.8-1.4 m, ``hole_frac`` of
      the pixels missing;
    * ``rgb [H,W,3] uint8``; ``nrm [H,W,3]`` unit normals in ``nrm_dtype``;
    * ``labels [H,W] uint8``: background 0 and one elliptic blob per entry of ``blobs`` (later blobs paint over
      earlier ones); a class in ``cls_ids`` without a blob is an object with no points, a blob class not in
      ``cls_ids`` a label absent from the object list, a repeated class in ``cls_ids`` a duplicated object;
    * ``poses``: YCB ``meta['poses']`` ``[3,4,n]``, LineMOD ``RT [3,4]``; ``cls_ids``; per object the mesh
      keypoints ``kps [n_kps,3]`` and centre ``ctrs [3]`` of its class (float64, metres, a few cm across);
    * ``K`` (the dataset's intrinsics, float32 for YCB as the reference's config holds them) and ``cam_scale``.
    LineMOD frames hold one object of class 1 (``cls_ids=(1,)``, ``blobs=(1,)``)."""
    rs = np.random.RandomState(seed)
    ys, xs = np.mgrid[:h, :w]
    d = 1.1 + 0.3 * np.sin(xs / 57.0) * np.cos(ys / 43.0) + 0.02 * rs.rand(h, w)
    cam_scale = 10000.0 if dataset == "ycb" else 1000.0
    raw = np.round(d * cam_scale).astype(np.uint16)
    raw[rs.rand(h, w) < hole_frac] = 0
    rgb = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    nrm = rs.normal(size=(h, w, 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=2, keepdims=True)).astype(nrm_dtype)
    labels = np.zeros((h, w), np.uint8)
    for c in blobs:
        cy, cx = rs.uniform(0.1, 0.9) * h, rs.uniform(0.1, 0.9) * w
        ry, rx = rs.uniform(0.08, 0.3) * h, rs.uniform(0.08, 0.3) * w
        labels[((ys - cy) / ry) ** 2 + ((xs - cx) / rx) ** 2 < 1.0] = c
    n = len(cls_ids)
    Rt = [np.concatenate((_rotation(rs), rs.uniform(-0.2, 0.2, (3, 1)) + [[0.0], [0.0], [1.0]]), axis=1)
          for _ in range(n)]
    poses = np.stack(Rt, axis=2) if dataset == "ycb" else Rt[0]
    mesh = {c: (rs.uniform(-0.08, 0.08, (n_kps, 3)), rs.uniform(-0.01, 0.01, 3)) for c in sorted(set(cls_ids))}
    kps = [mesh[c][0] for c in cls_ids]
    ctrs = [mesh[c][1] for c in cls_ids]
    if intrinsics is None:
        intrinsics = "ycb_K1" if dataset == "ycb" else "linemod"
    K = INTRINSICS[intrinsics].astype(np.float32) if dataset == "ycb" else INTRINSICS[intrinsics]
    return dict(raw=raw, rgb=rgb, nrm=nrm, labels=labels, poses=poses, cls_ids=np.array(cls_ids, np.uint32),
                kps=kps, ctrs=ctrs, K=K, cam_scale=cam_scale)


def _far_votes(rs, n, anchors, min_dist=0.25, sep=0.0):
    """``n`` uniform votes at least ``min_dist`` from every anchor and ``sep`` from each other: nonsense that sits
    near no refinement or bandwidth boundary, and (with ``sep`` = 0.2 m) too far from anything to move under a
    0.04 m Gaussian kernel, so a mean shift over it stops after a few rounds."""
    out = []
    while len(out) < n:
        v = rs.uniform(-0.7, 0.7, 3) + [0.0, 0.0, 1.0]
        if np.linalg.norm(np.asarray(anchors) - v, axis=1).min() >= min_dist and \
                (not out or np.linalg.norm(np.asarray(out) - v, axis=1).min() >= sep):
            out.append(v)
    return np.array(out)


def make_pose_frame(seed, n_kps=8):
    """The network's per-point predictions for one frame, seeded: what ``cal_frame_poses`` reads.

    Four classes and background, 2000 points, class radii 8, 12, 10, 8 cm (``cls_radius``, indexed by ``cls - 1``;
    a fifth entry of 6 cm exists only so that indexing by ``cls`` is a wrong answer rather than an IndexError).
    Objects 1-3 are 150, 520 and 430 points; their points vote the object's centre and keypoints with 4 mm noise,
    5 % of them nonsense far from everything (none of class 1's centre votes).  Groups placed so that every rule of
    the centre-clustering refinement and of the centre-label filter moves some keypoint by millimetres:

    * 40 points of object 2 labelled 3: centre votes at object 2's centre, keypoint votes 1.8 cm off object 2's
      keypoints.  Refinement gives them to class 2, whose keypoints they pull.
    * 30 points labelled 3 whose centre votes lie 7.2 cm from object 1's centre (between 0.8 r of class 1, 6.4 cm,
      and 0.8 r of classes 2 and 3, 9.6 and 8 cm), keypoint votes 1.8 cm off object 3's keypoints.  They stay in
      class 3, where the centre-label filter drops them; kept, they pull class 3's keypoints.
    * 60 background points (class 0) whose centre votes lie 1.5 cm from object 2's centre and keypoint votes 2 cm
      off its keypoints: refinement must leave them alone (it only relabels object points).
    * class 4: a bit-exact copy of class 1's points (one object segmented twice).  Both vote the same centre, the
      distance tie goes to the lower class id, and refinement leaves class 4 without points.

    The other background points vote nonsense.  Returns ``pcld [N,3]``, ``mask [N] int64``, ``ctr_of [1,N,3]``,
    ``kp_of [n_kps,N,3]`` (float32), ``mesh {cls: [n_kps+1,3] float64}`` (centre last), ``cls_radius`` and
    ``poses {cls: [3,4]}`` the votes were made from."""
    rs = np.random.RandomState(seed)
    counts = {1: 150, 2: 520, 3: 430}
    radius = [0.08, 0.12, 0.10, 0.08, 0.06]
    mesh, poses, ctr_cam, kps_cam = {}, {}, {}, {}
    ctr_choices = [np.array([-0.25, 0.0, 1.0]), np.array([0.05, 0.15, 0.9]), np.array([0.25, -0.15, 1.1])]
    for c in (1, 2, 3):
        mesh[c] = np.concatenate((rs.uniform(-0.08, 0.08, (n_kps, 3)), rs.uniform(-0.01, 0.01, (1, 3))))
        t = ctr_choices[c - 1] + rs.uniform(-0.03, 0.03, 3)
        poses[c] = np.concatenate((_rotation(rs), t[:, None]), axis=1)
        cam = mesh[c] @ poses[c][:, :3].T + poses[c][:, 3]
        kps_cam[c], ctr_cam[c] = cam[:n_kps], cam[n_kps]
    anchors = np.concatenate([np.concatenate((kps_cam[c], ctr_cam[c][None])) for c in (1, 2, 3)])

    def votes(n, target, nonsense=0.05):
        v = target + rs.normal(0, 0.004, (n, 3))
        bad = rs.rand(n) < nonsense
        if bad.any():
            v[bad] = _far_votes(rs, int(bad.sum()), anchors, sep=0.2)
        return v

    def group(n, label, ctr_target, ctr_noise, kps_target):
        pts.append(ctr_target + rs.normal(0, 0.03, (n, 3)))
        lab.append(np.full(n, label))
        ctr_v.append(ctr_target + rs.normal(0, ctr_noise, (n, 3)))
        kp_v.append(np.stack([kps_target[k] + rs.normal(0, 0.004, (n, 3)) for k in range(n_kps)]))

    pts, lab, ctr_v, kp_v = [], [], [], []
    for c in (1, 2, 3):
        n = counts[c]
        pts.append(ctr_cam[c] + rs.normal(0, 0.03, (n, 3)))
        lab.append(np.full(n, c))
        ctr_v.append(votes(n, ctr_cam[c], 0.0 if c == 1 else 0.05))
        kp_v.append(np.stack([votes(n, kps_cam[c][k]) for k in range(n_kps)]))
    group(40, 3, ctr_cam[2], 0.004, kps_cam[2] + [0.015, -0.01, 0.0])                 # mislabelled object 2
    group(30, 3, ctr_cam[1] + [-0.072, 0.0, 0.0], 0.0015, kps_cam[3] + [0.0, 0.015, -0.01])   # between radii
    group(60, 0, ctr_cam[2] + [0.0, 0.0, 0.015], 0.004, kps_cam[2] + [-0.012, 0.0, 0.016])    # background
    nb = 2000 - sum(len(p) for p in pts) - counts[1]
    pts.append(rs.uniform(-0.5, 0.5, (nb, 3)) + [0.0, 0.0, 1.0])
    lab.append(np.zeros(nb, np.int64))
    ctr_v.append(_far_votes(rs, nb, anchors))
    kp_v.append(np.stack([_far_votes(rs, nb, anchors) for _ in range(n_kps)]))
    pcld = np.concatenate(pts).astype(np.float32)
    mask = np.concatenate(lab).astype(np.int64)
    ctr_of = (pcld - np.concatenate(ctr_v)).astype(np.float32)[None]
    kp_of = (pcld[None] - np.concatenate(kp_v, axis=1)).astype(np.float32)
    perm = rs.permutation(len(pcld))
    pcld, mask, ctr_of, kp_of = pcld[perm], mask[perm], ctr_of[:, perm], kp_of[:, perm]
    # class 4: a copy of class 1's points, in the same order, appended at the end
    one = np.flatnonzero(mask == 1)
    pcld = np.concatenate((pcld, pcld[one]))
    mask = np.concatenate((mask, np.full(len(one), 4)))
    ctr_of = np.concatenate((ctr_of, ctr_of[:, one]), axis=1)
    kp_of = np.concatenate((kp_of, kp_of[:, one]), axis=1)
    mesh[4], poses[4] = mesh[1], poses[1]
    return dict(pcld=pcld, mask=mask, ctr_of=ctr_of, kp_of=kp_of, mesh=mesh, cls_radius=radius, poses=poses)


def item_test_frames():
    """The frames of tests/golden/item_cases.npz by name, with the item shape each is sampled at:
    ``{name: (frame, dataset, n_points, n_objects)}``.  Two full 480x640 frames at 12288 points (YCB with 8
    keypoints, LineMOD with 16) and two small ones: a YCB frame with fewer valid pixels than points (the 'wrap'
    padding), an absent label, an object without points and a duplicated class id; a LineMOD frame with a point
    count that is no multiple of the kernel's tile."""
    return {
        "ycb_full": (make_item_frame(101, n_kps=8, cls_ids=(2, 7, 11, 7), blobs=(2, 7, 11, 4)), "ycb", 12288, 22),
        "lm_full": (make_item_frame(102, dataset="linemod", n_kps=16, cls_ids=(1,), blobs=(1,)), "linemod", 12288, 2),
        "ycb_small": (make_item_frame(103, h=24, w=40, n_kps=16, cls_ids=(3, 6, 3, 20), blobs=(3, 6, 9), hole_frac=0.4,
                                      intrinsics="ycb_K2"), "ycb", 700, 22),
        "lm_small": (make_item_frame(104, h=30, w=36, dataset="linemod", n_kps=8, cls_ids=(1,), blobs=(1,),
                                     nrm_dtype=np.float64), "linemod", 500, 2),
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


def make_aug_frame(seed, h=40, w=48, dataset="ycb", mask_channels=1):
    """A seeded frame and background frame for the augmentation (``rgb_add_noise`` / ``add_real_back``).

    The colour image mixes smooth gradients with noise and has bands of special pixels: saturated (S = 255 at
    V = 255 and below), grey (S = 0), black and white.  ``labels`` marks object blobs (YCB class ids, LineMOD 0/1);
    ``raw`` is uint16 depth with holes.  The background has its own colour, depth (with holes) and label image:
    YCB class ids, or a LineMOD 0/255 mask with ``mask_channels`` channels."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[:h, :w].astype(np.float64)
    base = np.stack([128 + 127 * np.sin(xx / 7.0 + k) * np.cos(yy / 5.0 - k) for k in range(3)], -1)
    rgb = np.clip(base + rs.randn(h, w, 3) * 20, 0, 255).astype(np.uint8)
    specials = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [200, 0, 90], [128, 128, 128],
                         [37, 37, 37], [0, 0, 0], [255, 255, 255], [255, 254, 255], [1, 0, 0], [254, 255, 0]],
                        np.uint8)
    rgb[0, : len(specials)] = specials
    rgb[h // 2, -len(specials):] = specials[::-1]
    rgb[-1, :] = rs.randint(0, 256, (w, 3)).astype(np.uint8)
    cls = rs.randint(1, 22, 3) if dataset == "ycb" else np.ones(3, np.int64)
    labels = np.zeros((h, w), np.uint8)
    for c in cls:
        cy, cx, r = rs.randint(0, h), rs.randint(0, w), rs.randint(4, 10)
        labels[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = c
    raw = (5000 + 3000 * rs.rand(h, w)).astype(np.uint16)
    raw[rs.rand(h, w) < 0.3] = 0
    back_rgb = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    back_dpt = (4000 + 4000 * rs.rand(h, w)).astype(np.uint16)
    back_dpt[rs.rand(h, w) < 0.2] = 0
    blob = (yy - h / 3) ** 2 + (xx - w / 2) ** 2 < (min(h, w) / 4) ** 2
    if dataset == "ycb":
        back_labels = np.where(blob, rs.randint(1, 22), 0).astype(np.uint8)
        back_labels[rs.rand(h, w) < 0.05] = 3
    else:
        m = np.where(blob, 255, 0).astype(np.uint8)
        m[rs.rand(h, w) < 0.05] = 254
        back_labels = m if mask_channels == 1 else np.repeat(m[..., None], 3, 2)
        if mask_channels == 3:
            back_labels[..., 1] = 255 - back_labels[..., 1]      # only channel 0 may matter
    return dict(rgb=rgb, labels=labels, raw=raw, back_rgb=back_rgb, back_labels=back_labels, back_dpt=back_dpt)
