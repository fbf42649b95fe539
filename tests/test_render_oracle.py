"""CPU: the rasteriser's numpy oracle (oracle/render_oracle.py, DESIGN.md §4.31) against closed forms: the pixel set
of an axis-aligned quad under the top-left rule, the analytic depth of a slanted plane, watertight subdivided quads,
the depth tie, near-plane and guard-band culling, degenerate faces and both windings."""
import numpy as np
import pytest

from oracle import render_oracle as R

EYE = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
K256 = (256.0, 256.0, 0.0, 0.0)             # u = 256 x / z: camera points on a dyadic grid project exactly


def cam_points(uv, z, K=K256):
    """Camera-frame points that project to pixel positions ``uv [n,2]`` at depths ``z [n]`` (exact for dyadic
    values)."""
    uv, z = np.asarray(uv, np.float64), np.broadcast_to(np.asarray(z, np.float64), (len(uv),))
    fx, fy, cx, cy = K
    return np.stack([(uv[:, 0] - cx) / fx * z, (uv[:, 1] - cy) / fy * z, z], 1).astype(np.float32)


def one(mesh, H, W, K=K256, RT=EYE, z_near=0.01, coverage=True, label=7):
    return R.render_frame([mesh], [0], RT[None], [label], K, H, W, z_near, coverage=coverage)


def colours(n, seed=0):
    return np.random.RandomState(seed).randint(0, 256, (n, 3)).astype(np.uint8)


def quad(u0, v0, u1, v1, z=1.0):
    xyz = cam_points([(u0, v0), (u1, v0), (u1, v1), (u0, v1)], z)
    return xyz, np.array([[0, 1, 2], [0, 2, 3]]), colours(4)


def test_axis_aligned_quad_covers_the_top_left_pixel_set():
    H, W = 16, 20
    for (u0, v0, u1, v1) in ((2, 3, 7, 9), (0, 0, 5, 4), (2.5, 3.25, 7.5, 9.75), (-3, -2, 25, 30)):
        depth, rgb, labels, cov = one(quad(u0, v0, u1, v1), H, W)
        jj, ii = np.mgrid[:H, :W]
        # left and top edges drawn, right and bottom edges not: u0 <= i < u1, v0 <= j < v1
        want = (ii >= u0) & (ii < u1) & (jj >= v0) & (jj < v1)
        assert np.array_equal(cov, want.astype(np.int64)), (u0, v0, u1, v1)
        assert np.all(depth[want] == np.float32(1.0)) and np.all(depth[~want] == 0)
        assert np.all(labels[want] == 7) and np.all(labels[~want] == 0) and np.all(rgb[~want] == 0)


def test_slanted_plane_depth_within_an_ulp():
    # the plane z = 1 + x / 2 seen by fx = fy = 256, cx = cy = 100: its vertices are exact float32 and project to
    # exact pixel positions, so the only error is the interpolation's rounding
    K = (256.0, 256.0, 100.0, 100.0)
    xyz = np.array([[0, -0.25, 1], [0, 0.25, 1], [2, 0.5, 2], [2, -0.5, 2]], np.float32)
    mesh = (xyz, np.array([[0, 1, 2], [0, 2, 3]]), colours(4))
    depth, _, _, cov = one(mesh, 200, 400, K=K)
    drawn = cov > 0
    assert drawn.sum() > 10000 and cov.max() == 1
    ii = np.mgrid[:200, :400][1]
    exact = 1.0 / (1.0 - 0.5 * (ii - 100.0) / 256.0)
    f32 = exact.astype(np.float32)
    ulp = np.spacing(f32)
    assert np.all(np.abs(depth[drawn].astype(np.float64) - f32[drawn]) <= ulp[drawn])


@pytest.mark.parametrize("jitter", [0.0, 0.3])
def test_subdivided_quad_is_watertight(jitter):
    # an n x n grid of cells over [4, 36) x [3, 27), the interior vertices jittered (0: every edge passes through
    # pixel samples, diagonals included); every pixel of the square is covered exactly once, none outside it
    rs = np.random.RandomState(1)
    n, (u0, v0, u1, v1) = 12, (4, 3, 36, 27)
    gu, gv = np.linspace(u0, u1, n + 1), np.linspace(v0, v1, n + 1)
    uv = np.stack(np.meshgrid(gu, gv), -1).reshape(-1, 2)
    inner = ((uv[:, 0] > u0) & (uv[:, 0] < u1) & (uv[:, 1] > v0) & (uv[:, 1] < v1))
    uv[inner] += rs.uniform(-jitter, jitter, (inner.sum(), 2)) * (u1 - u0) / n
    uv = np.round(uv * 256) / 256
    xyz = cam_points(uv, rs.uniform(0.5, 2.0, len(uv)).astype(np.float32).astype(np.float64))
    faces = []
    for r in range(n):
        for c in range(n):
            a, b, d, e = r * (n + 1) + c, r * (n + 1) + c + 1, (r + 1) * (n + 1) + c, (r + 1) * (n + 1) + c + 1
            faces += [[a, b, e], [a, e, d]] if (r + c) % 2 else [[a, b, d], [b, e, d]]
    faces = np.array(faces)
    faces[::3] = faces[::3, ::-1]                    # mixed windings
    _, _, _, cov = one((xyz, faces, colours(len(uv))), 32, 40)
    jj, ii = np.mgrid[:32, :40]
    want = (ii >= u0) & (ii < u1) & (jj >= v0) & (jj < v1)
    assert np.array_equal(cov, want.astype(np.int64))


def test_depth_tie_goes_to_the_lower_slot_and_face():
    xyz, faces, rgb = quad(2, 2, 10, 10)
    # two slots of one mesh at the same pose: the lower slot's label wins
    d, c, lab = R.render_frame([(xyz, faces, rgb)], [0, 0], np.stack([EYE, EYE]), [3, 5], K256, 12, 12)
    assert set(np.unique(lab)) == {0, 3}
    # the same face twice in one mesh, on vertices of different colours: the lower face's colours win
    xyz2 = np.concatenate([xyz, xyz])
    rgb2 = np.concatenate([np.full((4, 3), 10, np.uint8), np.full((4, 3), 200, np.uint8)])
    for order in ([[4, 5, 6], [4, 6, 7], [0, 1, 2], [0, 2, 3]], [[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]]):
        _, c, _ = one((xyz2, np.array(order), rgb2), 12, 12, coverage=False)
        first = 200 if order[0][0] == 4 else 10
        assert set(np.unique(c[2:10, 2:10])) == {first}
    # a nearer slot wins whatever its index
    near = EYE.copy()
    near[2, 3] = -0.5
    d, c, lab = R.render_frame([(xyz, faces, rgb)], [0, 0], np.stack([EYE, near]), [3, 5], K256, 12, 12)
    # the nearer quad covers [4, 20)^2, the farther [2, 10)^2: where both cover, the nearer draws
    assert np.all(lab[4:10, 4:10] == 5) and np.all(d[lab == 5] == np.float32(0.5))
    assert np.all(d[lab == 3] == np.float32(1.0)) and (lab == 3).sum() == 8 * 8 - 6 * 6


def test_near_plane_and_guard_band_cull_whole_faces():
    xyz = cam_points([(1, 1), (9, 1), (1, 9)], [1.0, 1.0, 1.0])
    mesh = lambda p: (p, np.array([[0, 1, 2]]), colours(3))                       # noqa: E731
    assert one(mesh(xyz), 12, 12)[3].sum() > 0
    for z_near, drawn in ((1.0, True), (1.0 + 2 ** -20, False)):                 # z >= z_near is drawn
        assert (one(mesh(xyz), 12, 12, z_near=z_near)[3].sum() > 0) == drawn, z_near
    # a vertex behind the camera culls the face, even where the other two vertices project onto the image
    behind = xyz.copy()
    behind[2, 2] = -1.0
    assert one(mesh(behind), 12, 12)[3].sum() == 0
    # a vertex whose Z is not finite culls the face (only non-finite poses or vertices reach this)
    for bad in (np.inf, -np.inf, np.nan):
        p = xyz.copy()
        p[1, 2] = bad
        assert one(mesh(p), 12, 12)[3].sum() == 0, bad
    far = EYE.copy()
    far[2, 3] = np.inf
    assert R.render_frame([mesh(xyz)], [0], far[None], [1], K256, 12, 12)[0].sum() == 0
    # the guard band is |u|, |v| <= 2^14, inclusive
    for u, drawn in ((16384.0, True), (16384.0 + 2 ** -8, False), (-16384.0, True), (-16384.0 - 2 ** -8, False)):
        p = cam_points([(1, 1), (u, 1), (1, 9)], 1.0)
        assert (one(mesh(p), 12, 12)[3].sum() > 0) == drawn, u


def test_degenerate_faces_draw_nothing():
    xyz = cam_points([(1, 1), (5, 5), (9, 9), (1, 9)], 1.0)
    rgb = colours(4)
    for face in ([0, 1, 2], [0, 0, 3], [3, 3, 3], [0, 3, 0]):
        assert one((xyz, np.array([face]), rgb), 12, 12)[3].sum() == 0, face
    # a face that snaps to zero area at 1/256 pixel
    tiny = cam_points([(1, 1), (1 + 2 ** -10, 1), (1, 9)], 1.0)
    assert one((tiny, np.array([[0, 1, 2]]), rgb[:3]), 12, 12)[3].sum() == 0


def test_both_windings_draw_the_same_pixels():
    rs = np.random.RandomState(3)
    for _ in range(20):
        uv = np.round(rs.uniform(-2, 18, (3, 2)) * 256) / 256
        xyz = cam_points(uv, rs.uniform(0.5, 3.0, 3).astype(np.float32).astype(np.float64))
        rgb = colours(3, rs.randint(1 << 30))
        a = one((xyz, np.array([[0, 1, 2]]), rgb), 16, 16)
        b = one((xyz, np.array([[0, 2, 1]]), rgb), 16, 16)
        c = one((xyz, np.array([[1, 2, 0]]), rgb), 16, 16)
        for o in (b, c):
            assert np.array_equal(a[3], o[3])
            drawn = a[3] > 0
            ulp = np.spacing(a[0][drawn])
            assert np.all(np.abs(a[0][drawn] - o[0][drawn]) <= ulp)
            assert np.all(np.abs(a[1].astype(int) - o[1].astype(int)) <= 1)


def test_dpt_mm_is_the_float32_product_truncated():
    z = np.array([0.001, 0.0010000000474974513, 0.5, 0.7654321, 65.535, 65.536, 100.0], np.float32)
    want = [int(min(np.trunc(np.float32(v) * np.float32(1000.0)), 65535)) for v in z]
    assert R.dpt_mm(z).tolist() == want and R.dpt_mm(z).dtype == np.uint16
    # a face at the nearest admitted plane is drawn at >= 1 mm: add_real_back's dpt > 0 is the reference's
    # dpt_mm > 1e-6 on the float map
    xyz = cam_points([(1, 1), (9, 1), (1, 9)], [0.001, 0.0015, 0.001]).astype(np.float32)
    xyz[:, 2] = np.maximum(xyz[:, 2], np.float32(0.001))
    d, _, _, cov = one((xyz, np.array([[0, 1, 2]]), colours(3)), 12, 12, z_near=0.001)
    assert cov.sum() > 0 and np.all(R.dpt_mm(d)[cov > 0] >= 1) and np.all(R.dpt_mm(d)[cov == 0] == 0)


def test_batch_render_and_inactive_frames():
    mesh = quad(2, 2, 10, 10)
    RTs = np.stack([EYE, EYE])[:, None]
    d, c, lab = R.render([mesh], [[0], [0]], RTs, [[1], [2]], np.array([K256, K256]), 12, 12, active=[True, False])
    assert lab[0].max() == 1 and not lab[1].any() and not d[1].any()
    d2, _, _ = R.render([mesh], [[-1], [0]], RTs, [[1], [2]], K256, 12, 12)
    assert not d2[0].any() and np.array_equal(d2[1], d[0])
