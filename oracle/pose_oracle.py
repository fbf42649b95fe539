"""oracle/pose_oracle.py -- TEST INFRASTRUCTURE ONLY. NOT A PRODUCT PATH.

CPU restatement (numpy, float32 like the reference's torch tensors) of the keypoint-voting step:

* ``mean_shift_fit``      -- MeanShiftTorch.fit, ffb6d/utils/meanshift_pytorch.py:33-57
* ``best_fit_transform``  -- ffb6d/utils/pvn3d_eval_utils_kpls.py:28-59
* ``cal_frame_poses`` (with ``refine_mask``), ``cal_frame_poses_lm`` -- pvn3d_eval_utils_kpls.py:65-160, 220-284,
  restated from their semantics; ``check_frame_poses`` is the frame-voting contract
* ``fit_catalogue`` / ``fit_errors`` -- degenerate rigid-fit problems and the contract a fit must meet on them

Pinned against the reference's own code executed on the CPU (oracle/ref_loader.pose_functions and
frame_pose_functions, fixtures in tests/golden/pose_cases.npz and pose_frame_cases.npz made by
tests/golden/make_golden.py).  Floating point: torch's reduction order is not
restated, so the pin is by tolerance, not bitwise.  The returned centre is ONE member of the winning collapsed
cluster -- the one with the most neighbours, and nearly all members tie on that count -- so two correct
implementations may return different members: when the iteration stops (max shift < bandwidth * 1e-3 = 4e-5 m, or the
iteration cap, which the outliers of realistic vote sets usually run into) the members of a cluster agree to about
1e-4 m.  The contract is therefore |centre - reference centre| < 2e-4 m (0.5 % of the 0.04 m bandwidth).
"""
import numpy as np


def mean_shift_fit(A, bandwidth=0.05, max_iter=300, return_modes=False):
    """``A [N,3]`` -> ``(centre [3] f32, labels [N] bool, iterations)`` (+ converged positions)."""
    A = np.asarray(A, np.float32)
    N = A.shape[0]
    bw = np.float32(bandwidth)
    stop = np.float32(bandwidth * 1e-3)                      # :31
    norm = np.float32(bandwidth * np.sqrt(2 * np.pi))
    C = A.copy()
    it = 0
    while True:                                              # :38-49
        it += 1
        diff = C[None, :, :] - C[:, None, :]
        dis = np.sqrt((diff * diff).sum(2, dtype=np.float32))
        w = np.exp(np.float32(-0.5) * (dis / bw) ** 2) / norm      # gaussian_kernel, :18-20
        new_C = (w[:, :, None] * C[None, :, :]).sum(1, dtype=np.float32) / w.sum(1, dtype=np.float32)[:, None]
        shift = np.sqrt(((new_C - C) ** 2).sum(1, dtype=np.float32))
        C = new_C.astype(np.float32)
        if shift.max() < stop or it > max_iter:
            break
    diff = C[:, None, :] - C[None, :, :]                     # :51-55
    dis = np.sqrt((diff * diff).sum(2, dtype=np.float32))
    num_in = (dis < bw).sum(1)
    max_idx = int(np.argmax(num_in))                         # first maximum, like torch.max on the CPU
    labels = dis[max_idx] < bw
    if return_modes:
        return C[max_idx].copy(), labels, it, C
    return C[max_idx].copy(), labels, it


def best_fit_transform(A, B):
    """``A, B [M,3]`` -> ``[3,4]`` float64 ``[R|t]`` mapping A onto B."""
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    ca, cb = A.mean(0), B.mean(0)
    H = (A - ca).T @ (B - cb)                                # :47
    U, S, Vt = np.linalg.svd(H)
    R = Vt.T @ U.T
    if np.linalg.det(R) < 0:                                 # :52-54
        Vt[2, :] *= -1
        R = Vt.T @ U.T
    T = np.zeros((3, 4))
    T[:, :3] = R
    T[:, 3] = cb - R @ ca
    return T


def _vote_object(pred_ctr, pred_kp, msk, radius, use_ctr, use_ctr_clus_flter):
    """Centre and keypoints of one object: cluster the centre votes, keep the points of the winning centre cluster
    (when filtering; at least one), cluster every keypoint's votes of those points; the centre goes last."""
    ctr, labels, _ = mean_shift_fit(pred_ctr[msk], radius, 300)
    if not labels.any():
        labels[0] = True
    keep = labels if use_ctr_clus_flter else np.ones_like(labels)
    kps = [mean_shift_fit(v[msk][keep], radius, 300)[0] for v in pred_kp]
    return np.stack(kps + [ctr] if use_ctr else kps).astype(np.float32)


def refine_mask(pred_ctr, mask, ids, cls_radius, radius):
    """The centre-clustering refinement: cluster every class's centre votes; an object point (class > 0) whose
    centre vote lies within 0.8 x ``cls_radius[cls - 1]`` of the nearest of those centres (class ``cls``; the lowest
    class id on distance ties) takes that class."""
    ctrs = np.stack([mean_shift_fit(pred_ctr[mask == c], radius, 300)[0] for c in ids])
    d = np.sqrt(((pred_ctr[:, None, :] - ctrs[None]) ** 2).sum(2, dtype=np.float32))
    j = d.argmin(1)                                          # first minimum: the lowest class id on ties
    near = ids[j]
    r = (np.asarray(cls_radius, np.float64)[near - 1] * 0.8).astype(np.float32)
    return np.where((mask > 0) & (d[np.arange(len(j)), j] < r), near, mask)


def cal_frame_poses(pcld, mask, ctr_of, pred_kp_of, use_ctr, use_ctr_clus_flter, mesh_kps, cls_radius, radius=0.04):
    """YCB frame voting (pvn3d_eval_utils_kpls.py:65-160) in numpy float32: ``(cls_ids, poses [3,4], kps)``.

    With ``use_ctr_clus_flter`` the mask is refined first: every class's centre votes are clustered, and an object
    point whose centre vote lies within 0.8 x the radius of the nearest of those centres (``cls_radius[cls - 1]``)
    takes that centre's class (lowest class id on distance ties).  A class left without points gets the identity
    pose and ``n_kps + 1`` zero keypoints.  ``mesh_kps[cls]`` is ``[n_kps+1,3]``, centre last."""
    pcld = np.asarray(pcld, np.float32)
    mask = np.asarray(mask)
    n_kps = pred_kp_of.shape[0]
    pred_ctr = pcld - ctr_of[0]
    pred_kp = pcld[None] - pred_kp_of
    ids = np.unique(mask[mask > 0])
    if use_ctr_clus_flter and len(ids):
        mask = refine_mask(pred_ctr, mask, ids, cls_radius, radius)
    poses, kps_lst = [], []
    for c in ids:
        msk = mask == c
        if not msk.any():
            poses.append(np.identity(4)[:3, :])
            kps_lst.append(np.zeros((n_kps + 1, 3)))
            continue
        kpc = _vote_object(pred_ctr, pred_kp, msk, radius, use_ctr, use_ctr_clus_flter)
        mesh = np.asarray(mesh_kps[int(c)], np.float64)
        poses.append(best_fit_transform(mesh if use_ctr else mesh[:n_kps], kpc))
        kps_lst.append(kpc)
    return ids, poses, kps_lst


def cal_frame_poses_lm(pcld, mask, ctr_of, pred_kp_of, use_ctr, use_ctr_clus_flter, mesh_kps, radius=0.04):
    """LineMOD frame voting (pvn3d_eval_utils_kpls.py:220-284): class 1 is the object, no mask refinement;
    ``[pose [3,4]]``, the identity when no point is of class 1."""
    pcld = np.asarray(pcld, np.float32)
    msk = np.asarray(mask) == 1
    if not msk.any():
        return [np.identity(4)[:3, :]]
    n_kps = pred_kp_of.shape[0]
    kpc = _vote_object(pcld - ctr_of[0], pcld[None] - pred_kp_of, msk, radius, use_ctr, use_ctr_clus_flter)
    mesh = np.asarray(mesh_kps, np.float64)
    return [best_fit_transform(mesh if use_ctr else mesh[:n_kps], kpc)]


def frame_input_sha256(frame):
    """sha256 over the arrays ``cal_frame_poses`` reads, to tie a fixture to its generator."""
    import hashlib
    h = hashlib.sha256()
    for k in ("pcld", "mask", "ctr_of", "kp_of"):
        h.update(np.ascontiguousarray(frame[k]).tobytes())
    for c in sorted(frame["mesh"]):
        h.update(np.ascontiguousarray(frame["mesh"][c], np.float64).tobytes())
    h.update(np.asarray(frame["cls_radius"], np.float64).tobytes())
    return h.hexdigest()


def check_frame_poses(ids, poses, kps, want, mesh, n_kps, use_ctr):
    """Frame-voting contract: class ids equal, empty-class entries exact, keypoints within 2e-4 m of the
    reference's, the mesh keypoints placed by T and by the reference's T within 2e-4 m on average."""
    assert np.array_equal(np.asarray(ids, np.int64), want["ids"])
    for k, c in enumerate(want["ids"]):
        w_kps, w_T = want["kps_%d" % c], want["poses"][k]
        if not w_kps.any():
            assert np.array_equal(kps[k], w_kps) and np.array_equal(poses[k], w_T), c
            continue
        assert kps[k].shape == w_kps.shape and np.abs(kps[k] - w_kps).max() < 2e-4, c
        m = np.asarray(mesh[int(c)], np.float64)[: n_kps + 1 if use_ctr else n_kps]
        placed = m @ poses[k][:, :3].T + poses[k][:, 3]
        w_placed = m @ w_T[:, :3].T + w_T[:, 3]
        assert np.linalg.norm(placed - w_placed, axis=1).mean() < 2e-4, c


def load_frame_golden(path):
    """tests/golden/pose_frame_cases.npz as ``{variant: {field: array}}`` (+ ``seed``, ``input_sha256``)."""
    z = np.load(path)
    out = {}
    for key in z.files:
        if "/" in key:
            g, f = key.split("/", 1)
            out.setdefault(g, {})[f] = z[key]
        else:
            out[key] = z[key]
    return out


FRAME_VARIANTS = [("TT", True, True), ("TF", True, False), ("FF", False, False)]


# ----------------------------------------------------------------------------- rigid-fit catalogue
def _rotation(rs):
    q, _ = np.linalg.qr(rs.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def _group(name, A, B):
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    return name, (A if A.ndim == 3 else A[None]), (B if B.ndim == 3 else B[None])


def fit_catalogue(seed=0):
    """Rigid-fit problems at the inputs where a hand-written 3x3 SVD goes wrong: ``[(name, A [G,M,3] f32,
    B [G,M,3] f32)]``, every group one batched call.  Degenerate point sets are built from float32-representable
    values (small-integer multiples of dyadic directions), so they stay exactly degenerate after the rounding."""
    rs = np.random.RandomState(seed)
    out = []

    def rigid(A, noise=0.0, t=None):
        R = _rotation(rs)
        t = rs.uniform(-0.5, 0.5, 3) + [0.0, 0.0, 1.0] if t is None else t
        return A @ R.T + t + (rs.normal(0, noise, A.shape) if noise else 0.0)

    # generic problems: 1000 of them, so 16 blocks of 64 threads and a partial last block
    A = rs.uniform(-0.1, 0.1, (1000, 9, 3))
    out.append(_group("generic", A, np.stack([rigid(a, 2e-3) for a in A])))
    for M in (1, 2, 3, 4, 9, 4096):
        A = rs.uniform(-0.1, 0.1, (4, M, 3))
        out.append(_group("M%d" % M, A, np.stack([rigid(a, 2e-3) for a in A])))
    # exactly collinear sets: k * d with small integers k and a dyadic direction d
    k = np.array([-4, -3, -1, 0, 1, 2, 5, 7, -7], np.float64)[:, None]
    d1, d2 = np.array([0.0625, -0.03125, 0.125]), np.array([-0.015625, 0.0625, 0.03125])
    line_a, line_b = k * d1, k[::-1] * d2 + [0.25, -0.125, 1.0]
    gen = rs.uniform(-0.1, 0.1, (9, 3))
    out.append(_group("collinear_A", line_a, rigid(line_a)))
    out.append(_group("collinear_B", gen, line_b))
    out.append(_group("collinear_AB", line_a, line_b))
    out.append(_group("collinear_AB_same", line_a, line_a + [0.5, 0.5, 0.5]))
    # collinear + 1e-8 relative noise: below float32 resolution at these magnitudes (|k d| >= 0.5, half an ulp
    # >= 3e-8), so the rounded points are still exactly collinear
    kk = np.array([4, 5, 6, 7, 8, 9, 10, 11, 12], np.float64)[:, None]
    big = kk * np.array([0.5, -1.0, 2.0])
    out.append(_group("collinear_noise1e-8", big + rs.normal(0, 1e-8, big.shape).clip(-2e-8, 2e-8), rigid(big)))
    # identical points
    out.append(_group("B_identical", gen, np.tile([0.1, -0.2, 0.9], (9, 1))))
    out.append(_group("AB_identical", np.tile([0.3, 0.1, 0.7], (9, 1)), np.tile([0.1, -0.2, 0.9], (9, 1))))
    # coplanar sets, with and without a mirrored target (the reflection branch)
    plane = rs.uniform(-0.1, 0.1, (9, 3))
    plane[:, 2] = 0.0
    mirror = np.array([1.0, 1.0, -1.0])
    out.append(_group("coplanar_A", plane, rigid(plane, 1e-3)))
    out.append(_group("coplanar_A_mirrored", plane, rigid(plane, 1e-3) * mirror))
    out.append(_group("coplanar_B", gen, rigid(plane, 1e-3)))
    out.append(_group("coplanar_B_mirrored", gen, rigid(plane, 1e-3) * mirror))
    out.append(_group("generic_mirrored", gen, rigid(gen, 1e-3) * mirror))
    # isotropic sets: all three singular values equal
    cube = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * 0.05
    tetra = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64) * 0.05
    out.append(_group("cube", cube, rigid(cube)))
    out.append(_group("tetrahedron", tetra, rigid(tetra)))
    # near-degenerate sets: collinear and coplanar with relative noise 1e-3 .. 1e-8.  sigma_2 / sigma_1 of a
    # near-collinear set goes roughly as the square of its thickness (6e-6 at 1e-3, 1e-11 at 1e-8): all below the
    # uniqueness gate of fit_errors, so these check orthonormality and the objective only.  The near-coplanar sets
    # keep sigma_2 / sigma_1 ~ 0.7 and are compared with numpy's T at every noise level.
    for e in range(3, 9):
        base = rs.uniform(-1, 1, (9, 1)) * rs.normal(size=3) * 0.1
        near_line = base + rs.normal(0, 0.1 * 10.0 ** -e, base.shape)
        near_plane = plane + np.outer(rs.normal(0, 0.1 * 10.0 ** -e, 9), [0.0, 0.0, 1.0])
        out.append(_group("near_collinear_1e-%d" % e, near_line, rigid(near_line, 1e-4)))
        out.append(_group("near_coplanar_1e-%d" % e, near_plane, rigid(near_plane, 1e-4)))
    # thicker near-collinear sets, whose sigma_2 / sigma_1 clears the 1e-4 uniqueness gate of fit_errors, so T is
    # compared with numpy's there too
    for name, rel in (("near_collinear_3e-2", 3e-2), ("near_collinear_1e-2", 1e-2)):
        base = rs.uniform(-1, 1, (9, 1)) * rs.normal(size=3) * 0.1
        near_line = base + rs.normal(0, 0.1 * rel, base.shape)
        out.append(_group(name, near_line, rigid(near_line, 1e-4)))
    # far from the origin, and a tiny spread
    out.append(_group("offset_1e3", gen, rigid(gen, 1e-4, t=np.array([1e3, -1e3, 1e3]))))
    small = rs.uniform(-1e-4, 1e-4, (9, 3))
    out.append(_group("spread_1e-4", small + [0.2, 0.1, 0.8], rigid(small)))
    # a spread of float32 subnormals (2^-145 steps): H's column norms multiply below fp64's range
    sub = rs.randint(-15, 16, (9, 3)).astype(np.float64) * 2.0 ** -145
    out.append(_group("subnormal_spread", sub, sub[:, [1, 2, 0]]))
    return out


def fit_objective(T, A, B):
    """``sum ||R a + t - b||^2`` in float64."""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    return float((((A @ T[:, :3].T) + T[:, 3] - B) ** 2).sum())


def fit_errors(T, A, B):
    """How far ``T`` is from a correct least-squares fit of ``A -> B``: ``(orth, det, excess, t_err)``.

    ``orth`` = max|R R^T - I|, ``det`` = |det R - 1|, ``excess`` = (objective - numpy's objective) divided by
    ``sum ||a - abar||^2 + sum ||b - bbar||^2`` (a correct fit has excess <= ~1e-15), ``t_err`` = max|T - T_numpy| /
    max(1, ||bbar||) where the minimiser is unique and well conditioned, else None: sigma_2 > 1e-4 sigma_1, and
    sigma_2 - sigma_3 > 1e-4 sigma_1 if the reflection branch is taken.  Below that gap the rotation about the weak
    axis is fixed only to about eps / (sigma_2 / sigma_1), and for rank <= 1 it is not unique at all: every
    completion of the basis is a proper rotation that reaches the same minimum."""
    A64, B64 = np.asarray(A, np.float64), np.asarray(B, np.float64)
    want = best_fit_transform(A64, B64)
    R = T[:, :3]
    orth = float(np.abs(R @ R.T - np.eye(3)).max())
    det = float(abs(np.linalg.det(R) - 1.0))
    scale = float(((A64 - A64.mean(0)) ** 2).sum() + ((B64 - B64.mean(0)) ** 2).sum())
    excess = (fit_objective(T, A64, B64) - fit_objective(want, A64, B64)) / max(scale, 1e-300)
    H = (A64 - A64.mean(0)).T @ (B64 - B64.mean(0))
    U, S, Vt = np.linalg.svd(H)
    reflect = np.linalg.det(Vt.T @ U.T) < 0
    unique = S[1] > 1e-4 * S[0] and (not reflect or S[1] - S[2] > 1e-4 * S[0])
    t_err = float(np.abs(T - want).max() / max(1.0, np.linalg.norm(B64.mean(0)))) if unique else None
    return orth, det, excess, t_err
