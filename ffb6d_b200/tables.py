"""The per-frame KNN / gather / fusion-MLP schedules of FFB6D as plain data (no torch, no CUDA
library: importable by the CPU reference arm of bench.py and by the golden generator).

The reference builds 22 neighbour-index arrays per frame on the CPU inside the dataset
(datasets/ycb/ycb_dataset.py:269-309 == datasets/linemod/linemod_dataset.py:313-353) and consumes
them in ``FFB6D.forward`` through 22 gathers plus the ``choose`` gather (models/ffb6d.py:231-312)
and 28 fusion 1x1 MLPs (models/ffb6d.py:55-80, 104-129).
"""

# reference literals (ycb_dataset.py:269-271, 298)
RGB_DS_SR = (4, 8, 8, 8)
RGB_UP_SR = (4, 2, 2)
PCLD_SUB_S_R = (4, 4, 4, 4)
N_DS_LAYERS = 4
N_UP_LAYERS = 3
K_NEIGH = 16

# feature widths seen by the gathers (models/ffb6d.py:49-50, 89-95; common.py:26)
DS_RGB_OC = (64, 128, 512, 1024)
DS_RNDLA_OC = (64, 128, 256, 512)
UP_RGB_OC = (256, 64, 64)
UP_RNDLA_OC = (256, 128, 64, 64)


def knn_schedule(n_points=12288, h=480, w=640, k=K_NEIGH):
    """The 22 KNN calls of one frame as ``(key, support, query, K)`` where support /
    query name a point set: ``("cld", level)`` = first ``n_points / 4**level`` cloud
    points, ``("img", sr)`` = the stride-``sr`` image pyramid level (``h//sr * w//sr``
    points).  Order = the reference's call order."""
    calls = []
    for i in range(N_DS_LAYERS):
        sr = RGB_DS_SR[i]
        calls.append(("cld_nei_idx%d" % i, ("cld", i), ("cld", i), k))
        calls.append(("cld_interp_idx%d" % i, ("cld", i + 1), ("cld", i), 1))
        calls.append(("r2p_ds_nei_idx%d" % i, ("img", sr), ("cld", i + 1), k))
        calls.append(("p2r_ds_nei_idx%d" % i, ("cld", i + 1), ("img", sr), 1))
    for i in range(N_UP_LAYERS):
        sr = RGB_UP_SR[i]
        lvl = N_DS_LAYERS - i - 1
        calls.append(("r2p_up_nei_idx%d" % i, ("img", sr), ("cld", lvl), k))
        calls.append(("p2r_up_nei_idx%d" % i, ("cld", lvl), ("img", sr), 1))
    return calls


def derived_searches(calls):
    """``{child key: parent key}``: searches of the schedule that are row slices of another search.  Cloud level j
    is the first N_j rows of the shuffled cloud (ycb_dataset.py:278), so two searches of the same support with the
    same K whose query sets are cloud levels i < j answer the same questions on a prefix: ``r2p_ds_nei_idx2/3`` are
    the first 192 / 48 rows of ``r2p_ds_nei_idx1`` (support img8), ``r2p_up_nei_idx0`` of ``r2p_ds_nei_idx0`` (img4),
    ``r2p_up_nei_idx1`` of ``r2p_up_nei_idx2`` (img2)."""
    by_group, derived = {}, {}
    for key, s, q, kk in calls:
        if q[0] == "cld":
            by_group.setdefault((s, kk), []).append((q[1], key))
    for members in by_group.values():
        members.sort()
        for lvl, key in members[1:]:
            if lvl > members[0][0]:
                derived[key] = members[0][1]
    return derived


def derived_image_searches(calls, h=480, w=640):
    """``{child key: (parent key, f)}``: searches whose QUERIES are an image level that is a strided subset of a
    finer level searched against the same support with the same K.  The stride-``sr`` pyramid level is
    ``dpt_xyz[::sr, ::sr]`` (ycb_dataset.py:253-264), so level ``sr_c`` is every ``f = sr_c / sr_p``-th pixel of every
    ``f``-th row of level ``sr_p``: ``p2r_ds_nei_idx0`` (cld1 <- img4) is that subset of ``p2r_up_nei_idx2``
    (cld1 <- img2), ``p2r_ds_nei_idx1`` (cld2 <- img8) of ``p2r_up_nei_idx1`` (cld2 <- img2), ``p2r_ds_nei_idx2``
    (cld3 <- img8) of ``p2r_up_nei_idx0`` (cld3 <- img4).  Only when the image size is a multiple of ``sr_c``."""
    by_group, derived = {}, {}
    for key, s, q, kk in calls:
        if q[0] == "img":
            by_group.setdefault((s, kk), []).append((q[1], key))
    for members in by_group.values():
        members.sort()
        sr_p, parent = members[0]
        for sr_c, key in members[1:]:
            if sr_c > sr_p and sr_c % sr_p == 0 and h % sr_c == 0 and w % sr_c == 0:
                derived[key] = (parent, sr_c // sr_p)
    return derived


def set_size(name, n_points=12288, h=480, w=640):
    kind, a = name
    if kind == "cld":
        n = n_points
        for i in range(a):
            n //= PCLD_SUB_S_R[min(i, len(PCLD_SUB_S_R) - 1)]
        return n
    return (h // a) * (w // a)


def gather_schedule(n_points=12288, h=480, w=640):
    """The 23 gathers of ``FFB6D.forward`` as ``(op, index_key, C, S, Q, K)`` in call
    order (models/ffb6d.py:240-312; SURVEY.md App. A.2).  ``op`` is ``"random_sample"``,
    ``"nearest_interpolation"`` or ``"choose"``."""
    N = [set_size(("cld", i), n_points) for i in range(5)]
    HW = {sr: set_size(("img", sr), n_points, h, w) for sr in (1, 2, 4, 8)}
    k = K_NEIGH
    g = []
    for i in range(N_DS_LAYERS):
        sr = RGB_DS_SR[i]
        g.append(("random_sample", "cld_sub_idx%d" % i, DS_RNDLA_OC[i], N[i], N[i + 1], k))
        g.append(("nearest_interpolation", "p2r_ds_nei_idx%d" % i, DS_RGB_OC[i], N[i + 1], HW[sr], 1))
        g.append(("random_sample", "r2p_ds_nei_idx%d" % i, DS_RGB_OC[i], HW[sr], N[i + 1], k))
    up_in = (DS_RNDLA_OC[3], UP_RNDLA_OC[0], UP_RNDLA_OC[1])  # width entering each interp
    for i in range(N_UP_LAYERS):
        sr = RGB_UP_SR[i]
        lvl = N_DS_LAYERS - i - 1
        g.append(("nearest_interpolation", "cld_interp_idx%d" % lvl, up_in[i], N[lvl + 1], N[lvl], 1))
        g.append(("nearest_interpolation", "p2r_up_nei_idx%d" % i, UP_RGB_OC[i], N[lvl], HW[sr], 1))
        g.append(("random_sample", "r2p_up_nei_idx%d" % i, UP_RGB_OC[i], HW[sr], N[lvl], k))
    g.append(("nearest_interpolation", "cld_interp_idx0", UP_RNDLA_OC[2], N[1], N[0], 1))
    g.append(("choose", "choose", UP_RGB_OC[2], HW[1], N[0], 1))
    return g


def fusion_mlp_schedule(n_points=12288, h=480, w=640):
    """The 28 fusion 1x1 MLPs of ``FFB6D.forward`` as ``(name, P, C1, C2, Co)``: positions, the two
    concatenated input widths (C2 = 0 for the ``*_pre`` layers) and the output width
    (models/ffb6d.py:55-80, 104-129; SURVEY.md App. A.3)."""
    N = [set_size(("cld", i), n_points) for i in range(5)]
    HW = {sr: set_size(("img", sr), n_points, h, w) for sr in (1, 2, 4, 8)}
    layers = []
    for i in range(N_DS_LAYERS):
        cr, cp, n1, hw = DS_RGB_OC[i], DS_RNDLA_OC[i], N[i + 1], HW[RGB_DS_SR[i]]
        layers += [("ds%d_r2p_pre" % i, n1, cr, 0, cp), ("ds%d_r2p_fuse" % i, n1, cp, cp, cp),
                   ("ds%d_p2r_pre" % i, n1, cp, 0, cr), ("ds%d_p2r_fuse" % i, hw, cr, cr, cr)]
    for i in range(N_UP_LAYERS):
        cr, cp, n1, hw = UP_RGB_OC[i], UP_RNDLA_OC[i], N[N_DS_LAYERS - i - 1], HW[RGB_UP_SR[i]]
        layers += [("up%d_r2p_pre" % i, n1, cr, 0, cp), ("up%d_r2p_fuse" % i, n1, cp, cp, cp),
                   ("up%d_p2r_pre" % i, n1, cp, 0, cr), ("up%d_p2r_fuse" % i, hw, cr, cr, cr)]
    return layers


def knn_alg_bytes(S, Q, K):
    """Algorithmic HBM bytes of one KNN call (SURVEY.md §8d): xyz in once, int32 idx out."""
    return 12 * S + 12 * Q + 4 * Q * K


def gather_alg_bytes(C, S, Q, K):
    """Algorithmic HBM bytes of one gather (SURVEY.md §8d): touched rows once, int32 idx,
    output once."""
    return 4 * C * min(S, Q * K) + 4 * Q * K + 4 * C * Q


def frame_alg_bytes(n_points=12288, h=480, w=640, k=K_NEIGH):
    """(knn_bytes, gather_bytes) per frame; 8 239 296 + 160 186 368 at the defaults."""
    kb = sum(knn_alg_bytes(set_size(s, n_points, h, w), set_size(q, n_points, h, w), kk)
             for _, s, q, kk in knn_schedule(n_points, h, w, k))
    gb = 0
    for op, _, Cc, S, Q, K in gather_schedule(n_points, h, w):
        gb += gather_alg_bytes(Cc, S, Q, k if K == K_NEIGH else K)
    return kb, gb
