"""CPU: the textured rasteriser's oracle (DESIGN.md §4.35) against closed forms: a constant texture, a screen-aligned
quad that reproduces its texture (rho = 1) and its half-size copy that samples level 1 alone, a slanted plane's UVs
against ray-plane intersection, REPEAT wrapping, and mip chains against a direct restatement."""
import numpy as np
import pytest

from oracle import render_oracle as R
from oracle import textured_render_oracle as T
import textured_cases as TC


def _frame(mesh, H, W, K=TC.UNIT_K, RT=TC.IDENTITY):
    return T.render_frame([mesh], [0], RT[None], [7], K, H, W)


def test_constant_texture_draws_its_colour():
    xyz, faces, uv, _ = TC.box_mesh(4)
    tex = np.empty((64, 32, 3), np.uint8)
    tex[:] = (201, 17, 90)
    RT = np.array(np.concatenate([np.eye(3), [[0.0], [0.0], [0.6]]], 1), np.float32)
    RT[:3, :3] = np.array([[0.8, 0.0, 0.6], [0.0, 1.0, 0.0], [-0.6, 0.0, 0.8]])     # the box turned about y
    depth, rgb, lab = _frame((xyz, faces, uv, tex), 60, 80, (100.0, 100.0, 40.0, 30.0), RT)
    drawn = depth > 0
    assert drawn.sum() > 500
    assert (rgb[drawn] == (201, 17, 90)).all() and (rgb[~drawn] == 0).all()
    assert (lab[drawn] == 7).all()


def test_depth_and_labels_are_the_vertex_coloured_renders():
    xyz, faces, uv, tex = TC.box_mesh(4)
    RT = np.array(np.concatenate([np.eye(3), [[0.01], [-0.02], [0.5]]], 1), np.float32)
    K = (120.0, 110.0, 39.5, 31.0)
    d, _, lab = T.render_frame([(xyz, faces, uv, tex)], [0], RT[None], [3], K, 64, 80)
    d2, _, lab2 = R.render_frame([(xyz, faces, np.zeros_like(xyz, np.uint8))], [0], RT[None], [3], K, 64, 80)
    assert np.array_equal(d.view(np.uint32), d2.view(np.uint32)) and np.array_equal(lab, lab2)


@pytest.mark.parametrize("H, W", [(12, 16), (7, 5), (1, 9)])
def test_screen_quad_reproduces_its_texture(H, W):
    tex = TC.noise_texture(max(H, W), 3)[:H, :W]
    xyz, faces, uv = TC.screen_quad(W, H)
    _, rgb, _ = _frame((xyz, faces, uv, tex), H, W)
    assert np.array_equal(rgb, tex)


def test_half_size_quad_samples_level_one():
    H, W = 24, 32
    tex = TC.noise_texture(32, 4)[:H, :W]
    xyz, faces, uv = TC.screen_quad(W, H, x1=W / 2 - 0.5, y1=H / 2 - 0.5)
    _, rgb, _ = _frame((xyz, faces, uv, tex), H, W)
    assert np.array_equal(rgb[:H // 2, :W // 2], T.mip_chain(tex)[1])
    # the rule at rho = 2 exactly: level 1, t = 0
    rho, la, lb, t, blend = T.lod(np.array([2.0 / W]), np.array([0.0]), np.array([0.0]), np.array([2.0 / H]), H, W)
    assert rho[0] == 2.0 and la[0] == 1 and lb[0] == 2 and t[0] == 0.0 and blend[0]


def test_lod_rule():
    # below 1 or NaN: level 0 alone; at or past 2^(L-1): the last level alone; linear in rho between
    z = np.zeros(5)
    ux = np.array([0.5, 1.0, 1.5, 3.999, 4.0]) / 64.0
    rho, la, lb, t, blend = T.lod(ux, z, z, z, 5, 64)          # L = 7 levels for 64 wide
    assert list(la) == [0, 0, 0, 1, 2] and not blend[0] and not blend[1]
    assert t[2] == 0.5 and blend[2] and lb[2] == 1
    rho, la, _, _, blend = T.lod(np.array([64.0, np.inf, np.nan]) / 64.0, z[:3], z[:3], z[:3], 64, 64)
    assert list(la) == [6, 6, 0] and not blend.any()


def test_slanted_plane_uv_is_ray_plane_intersection():
    # vertices on the 1/256-pixel grid (camera (1, 1, 0, 0), Z a power of two), so the projected triangle is exact
    scr = np.array([[2.5, 3.25], [40.75, 5.5], [10.125, 30.0]])
    Z = np.array([1.0, 2.0, 4.0])
    P = np.column_stack([scr * Z[:, None], Z])
    uv = np.array([[0.1, 0.2], [0.9, 0.3], [0.4, 0.95]], np.float32)
    U, V, iz, ok = R.vertex_stage(P.astype(np.float32), TC.IDENTITY, TC.UNIT_K)
    assert ok.all() and np.array_equal(U, np.rint(scr[:, 0] * 256)) and np.array_equal(V, np.rint(scr[:, 1] * 256))
    face = np.array([0, 1, 2])
    ii, jj, w, _ = R.face_pixels(U, V, face, 40, 48)
    n = len(ii)
    fa = np.tile(face, (n, 1))
    u, v, ux, uy, vx, vy = T.attributes(uv, fa, U[fa], V[fa], iz[fa], w)

    def closed(i, j):
        # the ray (i, j, 1) against the plane of P, then the barycentrics of the hit point in 3D
        nrm = np.cross(P[1] - P[0], P[2] - P[0])
        d = np.stack([i, j, np.ones_like(i)], -1).astype(np.float64)
        hit = d * ((P[0] @ nrm) / (d @ nrm))[:, None]
        area = np.linalg.norm(nrm)
        lam = [np.linalg.norm(np.cross(P[(k + 1) % 3] - hit, P[(k + 2) % 3] - hit), axis=1) / area for k in range(3)]
        return sum(l[:, None] * uv[k].astype(np.float64) for k, l in enumerate(lam))

    want = closed(ii, jj)
    assert n > 200
    assert np.abs(u - want[:, 0]).max() < 1e-12 and np.abs(v - want[:, 1]).max() < 1e-12
    # the analytic derivatives against central differences of the closed form
    h = 1e-4
    dx = (closed(ii + h, jj) - closed(ii - h, jj)) / (2 * h)
    dy = (closed(ii, jj + h) - closed(ii, jj - h)) / (2 * h)
    assert np.abs(ux - dx[:, 0]).max() < 1e-7 and np.abs(vy - dy[:, 1]).max() < 1e-7
    assert np.abs(uy - dy[:, 0]).max() < 1e-7 and np.abs(vx - dx[:, 1]).max() < 1e-7


def test_repeat_wrapping():
    tex = TC.noise_texture(8, 5)
    lv = T.mip_chain(tex)[0]
    u = np.arange(-64, 64) / 64.0 + 1.0 / 128
    v = np.full_like(u, 0.3125)
    base = T.bilinear(lv, u, v)
    for k in (-3.0, -1.0, 1.0, 2.0):
        assert np.array_equal(T.bilinear(lv, u + k, v + k), base)
    # a texel centre on the wrap: x = -0.5 blends the last and first columns equally
    c = T.bilinear(lv, np.array([0.0]), np.array([1.0 - 0.5 / 8]))
    assert np.array_equal(c[0], 0.5 * lv[0, 7].astype(np.float64) + 0.5 * lv[0, 0])
    # a quad whose UVs run past [0, 1] draws the texture tiled
    H, W = 8, 16
    xyz, faces, uv = TC.screen_quad(W, H, uv0=(-1.0, 1.0), uv1=(1.0, 2.0))
    _, rgb, _ = _frame((xyz, faces, uv, tex), H, W)
    assert np.array_equal(rgb, np.concatenate([tex, tex], 1))


def _direct_mips(tex):
    out = [tex.astype(np.int64)]
    while out[-1].shape[0] > 1 or out[-1].shape[1] > 1:
        s = out[-1]
        h, w = s.shape[:2]
        d = np.zeros((max(1, h >> 1), max(1, w >> 1), 3), np.int64)
        for j in range(d.shape[0]):
            for i in range(d.shape[1]):
                acc = 0
                for (x, y) in ((2 * i, 2 * j), (2 * i + 1, 2 * j), (2 * i, 2 * j + 1), (2 * i + 1, 2 * j + 1)):
                    acc = acc + s[min(y, h - 1), min(x, w - 1)]
                d[j, i] = (acc + 2) >> 2
        out.append(d)
    return out


@pytest.mark.parametrize("h, w", [(3, 5), (7, 1), (1, 4097), (4097, 1), (6, 6)])
def test_mip_chain_direct(h, w):
    tex = np.random.default_rng(h * 10000 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    got = T.mip_chain(tex)
    want = _direct_mips(tex)
    assert len(got) == max(h, w).bit_length() == len(want)
    for g, x in zip(got, want):
        assert np.array_equal(g, x)
