"""GPU: every path of the uniform-grid KNN (ffb6d_b200/csrc/knn_grid.cu) against the exact oracle.

Under the default tuning nearly every query is certified within two rings, so most of the grid's
code rarely runs in tests/test_gpu_knn.py: rings 3-4 and the ring jump, the new-shell scan of old
rows, the cell-cap loop, the geometric fallbacks, the single-cell grid, and overflow lists where the
duplicate list (back) meets the plain one (front).  The
cases here drive the tuning knobs and the geometry onto those paths, read back the grid's
``GridParams`` and the query's ``QueryState`` to prove they got there, and require results
bitwise equal to ``oracle.cpu_oracle.knn_search`` (fp32 reference arithmetic, ties in
(distance, index) order) in int32 and int64."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200._lib import lib, check
from conftest import GOLDEN
from oracle import cpu_oracle as O

pytestmark = pytest.mark.gpu

# knn_grid.cu: struct GridParams (64 B, at offset 0 of the grid) and struct QueryState (16 B, at
# offset 0 of a query's scratch), one per batch item
GRID_PARAMS = np.dtype([("lo", "<f4", 3), ("h", "<f4"), ("inv_h", "<f4"), ("slack", "<f4"), ("n", "<i4", 3),
                        ("ncells", "<i4"), ("hi", "<f4", 3), ("pad", "<i4", 3)])
QUERY_STATE = np.dtype([("ovf", "<i4"), ("dup", "<i4"), ("rep", "<i4"), ("finished", "<i4")])
assert GRID_PARAMS.itemsize == 64 and QUERY_STATE.itemsize == 16

DEFAULTS = (1.0, 17, 2.5)            # cell_scale, quantile, K = 1 cell_scale (include/ffb6d_b200.h)
RMAX = 4                             # widest block the search tries: 9 x 9 x 9 cells
N_SAMPLES = 32                       # sample points of the build's K-th-distance estimate


def max_cells(S):
    """Cell cap of a grid over S points (knn_grid.cu max_cells_for)."""
    m = min(max(8 * S, 4096), 1 << 22)
    return (m + 4095) // 4096 * 4096


def sample_indices(S):
    """Support rows whose K-th-neighbour distance the build estimates."""
    return {(smp * S) // N_SAMPLES + S // (2 * N_SAMPLES) for smp in range(N_SAMPLES)}


def single_cell(p):
    return p["ncells"] == 1 and p["inv_h"] == 0 and np.isinf(p["h"])


class Grid:
    """``ffb6d_knn_grid_build`` / ``ffb6d_knn_grid_query_organized`` with test-owned grid and scratch
    memory; ``params`` and ``query``'s second result are the per-item GridParams / QueryState."""

    def __init__(self, sup, k_hint):
        self.sup = sup
        self.B, self.S = sup.shape[0], sup.shape[1]
        self.nbytes = int(lib.ffb6d_knn_grid_bytes(self.B, self.S))
        self.mem = torch.zeros(self.nbytes, dtype=torch.uint8, device=sup.device)
        check(lib.ffb6d_knn_grid_build(sup.data_ptr(), self.B, self.S, int(k_hint), self.mem.data_ptr(), self.nbytes,
                                       torch.cuda.current_stream().cuda_stream))
        self.params = self.mem[: self.B * 64].cpu().numpy().view(GRID_PARAMS)

    def query(self, qry, k, dtype=torch.int32, query_width=0):
        Q = qry.shape[1]
        out = torch.full((self.B, Q, k), -7, dtype=dtype, device=qry.device)
        sb = int(lib.ffb6d_knn_grid_query_bytes(self.B, Q))
        scratch = torch.full((sb,), 0x55, dtype=torch.uint8, device=qry.device)
        check(lib.ffb6d_knn_grid_query_organized(self.sup.data_ptr(), qry.data_ptr(), self.B, self.S, Q, int(k),
                                                 out.data_ptr(), int(dtype == torch.int64), self.mem.data_ptr(),
                                                 self.nbytes, scratch.data_ptr(), sb, int(query_width),
                                                 torch.cuda.current_stream().cuda_stream))
        return out.cpu().numpy(), scratch[: self.B * 16].cpu().numpy().view(QUERY_STATE)


def set_knobs(scale, quantile, scale_k1):
    lib.ffb6d_knn_grid_tune(float(scale), int(quantile))
    lib.ffb6d_knn_grid_tune_k1(float(scale_k1))


@pytest.fixture
def knobs():
    """Sets the cell-size knobs for one test (documented defaults first) and always restores the
    defaults afterwards."""
    set_knobs(*DEFAULTS)
    try:
        yield set_knobs
    finally:
        set_knobs(*DEFAULTS)


def _width(Q):
    """An image row width under which Q queries take the organised K = 1 path (0 if none)."""
    for w in (64, 48, 40, 32, 16, 8):
        if Q % w == 0 and Q // w >= 4:
            return w
    return 0


def _eq(got, want, sup, qry, what):
    assert np.array_equal(got.astype(np.int64), want.astype(np.int64)), "%s: %s" % (
        what, O.knn_matches(sup, qry, got, want)[3])


def run_all_kernels(sup, qry, ks, hint, label, tiled=True, width=None):
    """Searches ``qry`` (None: self search) in the grid of ``sup`` for every K of ``ks`` through the
    kernel of its K class, in int32 and int64, plus the organised K = 1 path (rows of ``width``
    queries) and the tiled scan (algo 1); every result must equal the oracle.  Returns the
    GridParams and {K: QueryState}."""
    ts = torch.from_numpy(np.ascontiguousarray(sup, np.float32)).cuda()
    tq = ts if qry is None else torch.from_numpy(np.ascontiguousarray(qry, np.float32)).cuda()
    q_np = sup if qry is None else qry
    g = Grid(ts, hint)
    states = {}
    for k in ks:
        want = O.knn_search(sup, q_np, k)
        for dt in (torch.int32, torch.int64):
            got, st = g.query(tq, k, dt)
            _eq(got, want, sup, q_np, "%s K=%d %s" % (label, k, dt))
        states[k] = st
        w = width or _width(q_np.shape[1])
        if k == 1 and qry is not None and w:
            for dt in (torch.int32, torch.int64):
                got, st = g.query(tq, 1, dt, query_width=w)
                _eq(got, want, sup, q_np, "%s organised K=1 %s" % (label, dt))
            states["organised"] = st
        if tiled:
            got = F.knn_search(ts, tq, k, algo=1).cpu().numpy()
            _eq(got, want, sup, q_np, "%s tiled scan K=%d" % (label, k))
    return g.params, states


# ------------------------------------------------------------------------------------------ adversarial clouds
def _f32(x):
    return np.ascontiguousarray(x, dtype=np.float32)


def _nudge(v, steps):
    """v moved by `steps` ulps (elementwise, steps in -2..2)."""
    v = _f32(v).copy()
    for s in (-2, -1, 1, 2):
        m = steps == s
        for _ in range(abs(s)):
            v[m] = np.nextafter(v[m], np.float32(np.inf if s > 0 else -np.inf))
    return v


def _faces(p, axis):
    """Interior cell faces lo + c*h along one axis, rounded as the kernels may compute them (product
    rounded or fused into the add)."""
    c = np.arange(1, int(p["n"][axis]), dtype=np.float64)
    lo, h = np.float32(p["lo"][axis]), np.float32(p["h"])
    plain = (lo + (c.astype(np.float32) * h).astype(np.float32)).astype(np.float32)
    fused = (np.float64(lo) + c * np.float64(h)).astype(np.float32)
    return np.unique(np.concatenate([plain, fused]))


def _snap(pts, p, rs):
    """Moves one to three coordinates of every point onto a read-back cell face, +-0..2 ulps."""
    pts = _f32(pts).copy()
    lo, hi = p["lo"], p["hi"]
    for a in range(3):
        fa = _faces(p, a)
        sel = rs.rand(len(pts)) < (1.0 if a == 0 else 0.6)
        if len(fa) == 0:
            continue
        v =_nudge(fa[rs.randint(0, len(fa), sel.sum())], rs.randint(-2, 3, sel.sum()))
        pts[sel, a] = np.clip(v, lo[a], hi[a])
    return pts


def _snap_nearest(pts, p, rs, frac=0.7):
    """Moves a fraction of the coordinates onto their NEAREST read-back cell face, +-0..2 ulps
    (neighbouring points stay neighbours)."""
    pts = _f32(pts).copy()
    for a in range(3):
        fa = _faces(p, a)
        if len(fa) == 0:
            continue
        sel = rs.rand(len(pts)) < frac
        j = np.clip(np.searchsorted(fa, pts[sel, a]), 1, len(fa) - 1)
        near = np.where(np.abs(fa[j - 1] - pts[sel, a]) < np.abs(fa[j] - pts[sel, a]), fa[j - 1], fa[j])
        pts[sel, a] = np.clip(_nudge(near, rs.randint(-2, 3, sel.sum())), p["lo"][a], p["hi"][a])
    return pts


def _lattice(n, spacing, offset):
    i = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).reshape(-1, 3)
    return _f32(np.float32(offset) + (i * spacing).astype(np.float32))


def face_cloud(offset, spacing, rs):
    """A 20^3 lattice, shuffled, with its 8 corners repeated in rows 0, 2, ..., 14."""
    base = _lattice(20, spacing, offset)
    base = base[rs.permutation(len(base))]
    lo, hi = base.min(0), base.max(0)
    base[0:16:2] = np.array([[(lo, hi)[(c >> a) & 1][a] for a in range(3)] for c in range(8)], np.float32)
    return base


def wide_needle(rs, S=16384):
    """A needle from x = -1024 to +1024 (ends in rows 0 and 4) whose other points lie in [990, 1010]: the cell
    cap stretches ~10^5 cells along x, and cell_of's (p - lo) * inv_h rounds by more than the float spacing
    at p, so points near a face may be binned on either side of it."""
    x = np.sort(rs.rand(S) * 20.0 + 990.0)
    x[0], x[4] = -1024.0, 1024.0
    return _f32(np.c_[x, np.zeros((S, 2))])


def test_face_placed_clouds(cuda, knobs):
    """Support points and queries exactly on the read-back cell faces and 1-2 ulps off them: lattices near
    the origin and 10^3 m from it at mm spacing, and a needle 2 km long whose dense end is 10^3 m from the
    origin.  The support's rows other than the build's sample rows and its subsample (even rows: stride
    <= 4 for these S and K_hint 8) are moved onto the faces of the unmoved cloud's grid; the box is pinned
    by rows that stay, so the moved cloud has the same grid, which is asserted."""
    rs = np.random.RandomState(11)
    ks = (1, 3, 8, 16, 17, 24, 28, 32, 40, 64)
    for name, base in (("lattice 0.25 m", face_cloud(0.0, 0.25, rs)), ("lattice 1 mm at 1 km", face_cloud(1000.0, 1e-3, rs)),
                       ("lattice 2^-10 m at -1 km", face_cloud(-1024.0, 2.0 ** -10, rs)), ("wide needle", wide_needle(rs))):
        S, hint = len(base), 8
        p = Grid(torch.from_numpy(base[None]).cuda(), hint).params[0]
        assert p["ncells"] > 8 and not single_cell(p)
        keep = sample_indices(S) | set(range(0, S, 2))
        moved = np.array([i for i in range(S) if i not in keep])
        sup = base.copy()
        sup[moved] = _snap_nearest(base[moved], p, rs)
        box =lambda n: rs.rand(n, 3) * (p["hi"] - p["lo"]) + p["lo"]
        qry = _f32(np.concatenate([_snap(box(6144), p, rs), _snap_nearest(box(4096), p, rs), sup[rs.randint(0, S, 2048)]]))
        if name == "wide needle":
            qry[:, 1:] = 0.0
            qry[:6144, 0] = sup[rs.randint(0, S, 6144), 0] + (rs.rand(6144) - 0.5).astype(np.float32) * p["h"] * 4
        params, _ = run_all_kernels(sup[None], qry[None], ks, hint, name)
        for f in ("lo", "hi", "h", "inv_h", "n", "slack"):
            assert np.array_equal(params[0][f], p[f]), (name, f)          # the moved cloud kept its grid
        # an image of neighbouring queries (the organised K = 1 tiles share candidate boxes) on snapped planes
        H, W = 96, 128
        u, v = np.meshgrid((np.arange(W) + 0.5) / W, (np.arange(H) + 0.5) / H)
        img = np.c_[u.reshape(-1), v.reshape(-1), np.repeat(rs.rand(H // 4), 4 * W)] * (p["hi"] - p["lo"]) + p["lo"]
        img = _snap_nearest(img, p, rs)
        run_all_kernels(sup[None], img[None], (1, 2, 16, 32), hint, name + " image", width=W)
        run_all_kernels(sup[None], None, (1, 8, 16, 24, 32, 64), hint, name + " self", tiled=False)


def test_sparse_support_under_dense_image(cuda, knobs):
    """The organised K = 1 tiles where their stop test is tight: a sparse random sheet under a dense image of
    pixels on the same plane, with K = 1 cells of 0.4 ... 1.3 point spacings, so a pixel's nearest point is
    often about as far as the face of its tile's box and the next point just beyond it."""
    rs = np.random.RandomState(12)
    sup = _f32(np.c_[rs.rand(2000, 2), np.zeros(2000)])
    H, W = 128, 160
    u, v = np.meshgrid((np.arange(W) + 0.5) / W, (np.arange(H) + 0.5) / H)
    img = _f32(np.c_[u.reshape(-1), v.reshape(-1), np.zeros(H * W)])
    ts, tq = torch.from_numpy(sup[None]).cuda(), torch.from_numpy(img[None]).cuda()
    want = O.knn_search(sup[None], img[None], 1)
    for scale_k1 in (0.4, 0.55, 0.7, 0.85, 1.0, 1.3):
        knobs(DEFAULTS[0], DEFAULTS[1], scale_k1)
        g = Grid(ts, 1)
        assert g.params[0]["n"][2] == 1 and g.params[0]["ncells"] > 1000, g.params
        for dt in (torch.int32, torch.int64):
            got, _ = g.query(tq, 1, dt, query_width=W)
            _eq(got, want, sup[None], img[None], "sparse sheet, image, scale_k1 %g %s" % (scale_k1, dt))


def test_tile_stop_test_at_its_margin(cuda, knobs):
    """Organised K = 1 tiles whose best candidate inside the shared box is 0-0.5 % farther than the box face,
    with the true nearest point just beyond that face.  A needle of duplicated points has an estimate of 0,
    so its cells are h = l1 / S = 2^-7 exactly; tile t's 32 pixels sit at x = (4t + 2.75 +- 0.01) h, its box
    spans cells 4t + 1 ... 4t + 3, the outside point is at (4t + 4) h and the inside one at (4t + 1.4975) h.
    The support is small (S = 100) because the stop test's slack, 1e-5 (|x|max + l1), grows with S h here."""
    rs = np.random.RandomState(13)
    h = 2.0 ** -7
    B, T, W = 16, 24, 64                                      # T tiles per item: an image of 64 x 12 pixels
    S = 4 * T + 4
    c = 4 * np.arange(T) + 2
    xs = np.concatenate([(c + 2) * h, (c - 0.5025) * h, [0.0, S * h]])
    sup = _f32([np.c_[np.repeat(xs, 2), np.zeros((S, 2))][rs.permutation(S)] for _ in range(B)])
    tile = np.arange(T * 32) // 32                            # pixel order: tile rows of 8 x 4 pixels
    lane = np.arange(T * 32) % 32
    pix = (tile // (W // 8) * 4 + lane // 8) * W + tile % (W // 8) * 8 + lane % 8
    t_of = np.empty(T * 32, np.int64)
    t_of[pix] = tile
    qx = (c[t_of] + 0.75 + (rs.rand(B, T * 32) - 0.5) * 0.02) * h
    qry = _f32(np.stack([qx, np.zeros_like(qx), np.zeros_like(qx)], -1))
    params, _ = run_all_kernels(sup, qry, (1, 2), 1, "tile margin", width=W)
    assert (params["h"] == np.float32(h)).all() and (params["n"][:, 0] == S + 1).all(), params   # the line fallback


def test_power_of_two_lattice_ties(cuda, knobs):
    """16^3 lattice with spacing 2^-3: squared distances are exact, so queries on lattice points, edge and
    face midpoints, cell centres and the grid's own cell faces have up to dozens of exactly tied
    neighbours; ties must resolve to the lowest index, like the oracle's, for K up to 64."""
    rs = np.random.RandomState(2)
    sup = _lattice(16, 0.125, 0.0)
    sup = sup[rs.permutation(len(sup))]
    g = Grid(torch.from_numpy(sup[None]).cuda(), 16)
    p = g.params[0]
    assert not single_cell(p)
    pick = rs.randint(0, len(sup), 1536)
    half = rs.randint(0, 2, (1536, 3)).astype(np.float32) * np.float32(0.0625)
    qry = _f32(np.concatenate([sup[pick], sup[pick[:1024]] + half[:1024], _snap(sup[pick[:512]], p, rs)]))
    for hint in (16, 1, 64):
        run_all_kernels(sup[None], qry[None], (1, 6, 16, 27, 32, 33, 64), hint, "lattice hint %d" % hint)
    run_all_kernels(sup[None], None, (1, 7, 19, 64), 16, "lattice self", tiled=False)


def test_dense_cluster_in_sparse_shell(cuda, knobs):
    """6000 points in a 1 mm ball inside 200 points on a 10 m sphere (density ratio > 10^12): the estimate
    sees the cluster, the cell cap stretches the cells, and nearly every query of the surrounding box
    is sent to the overflow pass."""
    rs = np.random.RandomState(4)
    v = rs.randn(6200, 3)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    sup = np.concatenate([v[:6000] * rs.rand(6000, 1) ** (1 / 3) * 1e-3, v[6000:] * 10.0])
    sup = _f32(sup[rs.permutation(len(sup))])
    qry = _f32(np.concatenate([rs.rand(4800, 3) * 20.0 - 10.0, sup[rs.randint(0, len(sup), 320)]]))
    params, states = run_all_kernels(sup[None], qry[None], (1, 2, 16, 32, 64), 16, "cluster in shell")
    p = params[0]
    assert max_cells(len(sup)) / 2 < p["ncells"] <= max_cells(len(sup)), p      # at the cell cap
    for k in (16, 32, 64):
        st = states[k][0]
        assert st["ovf"] + st["dup"] > 0.9 * len(qry), (k, st)            # mostly overflow
    run_all_kernels(sup[None], None, (1, 16, 64), 16, "cluster in shell self", tiled=False)


def test_sheets_and_needles(cuda, knobs):
    """Flat sheets (one axis of zero extent, and a tilted plane) and needles (two axes of zero extent, and
    a diagonal), including a needle of repeated points that takes the points-on-a-line cell size."""
    rs = np.random.RandomState(6)
    flat = _f32(np.c_[rs.rand(6000, 2), np.zeros(6000)])
    uv = rs.rand(6000, 2)
    tilted = _f32(np.c_[uv, 1.0 - uv.sum(1) * 0.5])
    needle = _f32(np.c_[np.arange(4096) / np.float32(256), np.zeros((4096, 2))])
    diag = _f32(np.repeat(rs.rand(5000, 1), 3, 1) * np.array([1.0, 2.0, -0.5]))
    # 256 distinct points, each repeated 20 times in consecutive rows: every sampled point has >= 4 exact
    # duplicates in the build's subsample, the estimate is 0, and l2 = 0 leaves h = l1 * K / S
    rep = _f32(np.repeat(np.c_[np.arange(256) / np.float32(64), np.zeros((256, 2))], 20, 0))
    for name, sup in (("flat", flat), ("tilted", tilted), ("needle", needle), ("diagonal", diag), ("repeated", rep)):
        lo, hi = sup.min(0), sup.max(0)
        qry = _f32(np.concatenate([sup[rs.randint(0, len(sup), 2048)] + rs.randn(2048, 3).astype(np.float32) * 0.01,
                                   rs.rand(1024, 3) * (hi - lo + 0.1) + lo - 0.05]))
        qry[:256, 1:] = sup[:256, 1:]                                     # y, z of support points: on the flat ones
        params, _ = run_all_kernels(sup[None], qry[None], (1, 4, 16, 32, 64), 16, name)
        if name == "repeated":
            p = params[0]
            l1 = np.float32(hi[0] - lo[0])
            assert np.isclose(p["h"], l1 * np.float32(16) / np.float32(len(sup)), rtol=1e-6), p
        run_all_kernels(sup[None], None, (1, 16, 64), 16, name + " self", tiled=False)


def _fallback_h(sup, K):
    """The 2-D geometric cell edge sqrt(K l1 l2 / S) in the build's float32 arithmetic."""
    L = (sup.max(0) - sup.min(0)).astype(np.float32)
    l1, l3 = L.max(), L.min()
    l2 = np.float32(np.float32(np.float32(L[0] + L[1]) + L[2]) - l1) - l3
    return np.sqrt(np.float32(np.float32(np.float32(K) * l1) * l2) / np.float32(len(sup)))


def test_hole_pixel_supports(cuda, knobs):
    """Image levels that are 60-95 % hole pixels at +0.0 / -0.0: most sampled points estimate 0, so the cell
    edge is the 2-D geometric fallback (times 1.2 per step of the cell cap); the self searches of the holes
    rank thousands of exactly tied neighbours."""
    from ffb6d_b200.synthetic import make_frame, image_pyramid_np
    rs = np.random.RandomState(8)
    fr = make_frame(5, n_points=3072)
    img = image_pyramid_np(fr["dpt_xyz"])[8]                          # 60 x 80, 10 % holes
    samples = np.array(sorted(sample_indices(len(img))))
    for frac in (0.6, 0.8, 0.95):
        sup = img.copy()
        holes = rs.rand(len(sup)) < frac
        holes[samples[:20]] = True                                    # >= 18 of the 32 estimates are 0
        sup[holes] = 0.0
        neg = holes[:, None] & (rs.rand(len(sup), 3) < 0.5)
        sup[neg] = -0.0
        qry = _f32(np.concatenate([img, sup[rs.randint(0, len(sup), 1600)]]))
        for hint in (16, 1):
            params, states = run_all_kernels(sup[None], qry[None], (1, 5, 16, 32, 64), hint, "holes %g" % frac)
            p, hf = params[0], _fallback_h(sup, hint)
            assert any(np.isclose(p["h"], hf * 1.2 ** j, rtol=1e-5) for j in range(60)), (frac, hint, p["h"], hf)
        run_all_kernels(sup[None], None, (1, 16, 64), 16, "holes self %g" % frac, tiled=False)


def test_mixed_batch_items_equal_their_solo_search(cuda, knobs):
    """A batch that mixes normal items with degenerate ones (all points equal, a single cell, a needle, a far
    support): every item equals its own B = 1 search and the oracle, through every kernel."""
    rs = np.random.RandomState(9)
    S, Q = 2048, 1024
    items = [rs.randn(S, 3), np.full((S, 3), 0.5), rs.rand(S, 3) * 1e-6,
             np.c_[np.linspace(0, 1, S), np.zeros((S, 2))], rs.rand(S, 3) + 500.0]
    sup = _f32(np.stack(items))
    qry = _f32(np.concatenate([rs.randn(len(items), Q - 64, 3), np.zeros((len(items), 64, 3))], 1))
    qry[:, -32:, 2] = -0.0
    ts, tq = torch.from_numpy(sup).cuda(), torch.from_numpy(qry).cuda()
    for hint in (1, 16):
        g = Grid(ts, hint)
        assert single_cell(g.params[1]) and not single_cell(g.params[0])
        for k in (1, 3, 16, 32, 64):
            for w in ((0, 32) if k == 1 else (0,)):
                got, _ = g.query(tq, k, query_width=w)
                for b in range(len(items)):
                    solo, _ = Grid(ts[b:b + 1].contiguous(), hint).query(tq[b:b + 1].contiguous(), k, query_width=w)
                    assert np.array_equal(got[b], solo[0]), (hint, k, w, b)
                _eq(got, O.knn_search(sup, qry, k), sup, qry, "mixed batch K=%d width %d" % (k, w))
    for k in (1, 16, 64):
        got = F.knn_search(ts, ts, k).cpu().numpy()
        _eq(got, O.knn_search(sup, sup, k), sup, sup, "mixed batch self K=%d" % k)


def far_queries(rs, S=3000, Q=1536):
    """Items whose every query is far from the support: two far points that differ in ONE coordinate
    (z, y and x in items 0, 1, 2), each repeated hundreds of times, with +0.0 / -0.0 variants; which one
    becomes the item's representative depends on the race, so either way the other must not be
    mistaken for its duplicate."""
    sup = _f32(rs.rand(3, S, 3))
    qry = np.empty((3, Q, 3), np.float32)
    base = np.array([40.0, 0.5, 0.0], np.float32)
    for b, (axis, alt) in enumerate(((2, 0.9), (1, 0.9), (0, 41.0))):
        other = base.copy()
        other[axis] = alt
        pick = rs.rand(Q) < 0.5
        qry[b] = np.where(pick[:, None], base, other)
    qry[:, 1::7, 2] = np.where(qry[:, 1::7, 2] == 0, np.float32(-0.0), qry[:, 1::7, 2])
    return sup, qry


def test_every_query_overflows(cuda, knobs):
    """The overflow lists full: every query overflows, the duplicates fill the list from the back and the
    rest from the front until they meet (K = 1 without a row width: the per-thread search); K > 32 takes the
    tiled overflow scan and the separate row copy."""
    rs = np.random.RandomState(10)
    sup, qry = far_queries(rs)
    Q = qry.shape[1]
    for hint in (1, 16):
        params, states = run_all_kernels(sup, qry, (1, 2, 16, 31, 32, 33, 64), hint, "all far hint %d" % hint)
        for k, st in states.items():
            for b in range(3):
                assert st[b]["rep"] > 0 and st[b]["ovf"] >= 2, (k, b, st[b])
                if k != "organised":
                    assert st[b]["ovf"] + st[b]["dup"] == Q and st[b]["dup"] > Q // 4, (k, b, st[b])
                else:
                    assert st[b]["dup"] == 0, st[b]                      # far duplicates take the sentinel path


# ------------------------------------------------------------------------------------------ tuning invariance
SCALES = (0.02, 0.25, 1.0, 3.0, 30.0, 1e4)
QUANTILES = (0, 17, 31)
SCALES_K1 = (0.05, 2.5, 1e3)


@pytest.fixture(scope="module")
def frame_cases():
    """A synthetic frame's cloud and image levels in every K class, self and not, plus the organised K = 1
    searches, with the oracle's indices and K-th distances."""
    from ffb6d_b200.synthetic import make_frame, image_pyramid_np
    fr = make_frame(23, n_points=12288)
    cld0, cld1 = fr["cld"], fr["cld"][:3072]
    pyr = image_pyramid_np(fr["dpt_xyz"])
    cases = [  # name, support, query (None: self), K, query_width
        ("cld0 self K=1", cld0, None, 1, 0), ("cld0 self K=16", cld0, None, 16, 0),
        ("cld1 self K=32", cld1, None, 32, 0), ("cld1 self K=64", cld1, None, 64, 0),
        ("cld1->cld0 K=1", cld1, cld0, 1, 0), ("img8->cld1 K=9", pyr[8], cld1, 9, 0),
        ("img8->cld1 K=32", pyr[8], cld1, 32, 0), ("img8->cld1 K=64", pyr[8], cld1, 64, 0),
        ("cld0->img4 K=1", cld0, pyr[4], 1, 160), ("cld1->img8 K=1", cld1, pyr[8], 1, 80),
    ]
    out = []
    for name, s, q, k, w in cases:
        qq = s if q is None else q
        idx, dist = O.knn_batch(s[None], qq[None], k, return_dist=True)
        ts = torch.from_numpy(s[None]).cuda()
        tq = ts if q is None else torch.from_numpy(q[None]).cuda()
        out.append((name, s, qq, ts, tq, k, w, idx.astype(np.int32), np.sqrt(dist[0, :, k - 1])))
    return out


def test_results_never_depend_on_the_tuning(cuda, knobs, frame_cases):
    """cell_scale x quantile x K = 1 scale, and grids built for another K than the one queried: identical to
    the oracle at every setting.  The extremes must really give capped grids and single cells, and some
    queries must be certified at rings 3-4."""
    seen = {"cap": 0, "single": 0, "deep": 0}
    settings = [(s, qt, SCALES_K1[(i + j) % 3]) for i, s in enumerate(SCALES) for j, qt in enumerate(QUANTILES)]
    for scale, quantile, scale_k1 in settings:
        knobs(scale, quantile, scale_k1)
        for name, s, qq, ts, tq, k, w, want, kth in frame_cases:
            for hint in (k, 64 if k == 1 else 1):
                g = Grid(ts, hint)
                p = g.params[0]
                for dt in (torch.int32, torch.int64):
                    got, st = g.query(tq, k, dt, query_width=w)
                    _eq(got, want, s[None], qq[None], "%s hint %d at %s" % (name, hint, (scale, quantile, scale_k1)))
                cell_scale = scale_k1 if hint == 1 else scale
                # the clouds have no duplicate points, so every estimate is positive
                if name.startswith("cld") and (cell_scale == 1e4 or (cell_scale >= 1e3 and quantile >= 17)):
                    assert single_cell(p), (name, hint, p)
                    seen["single"] += 1
                if cell_scale <= 0.05 and quantile >= 17:
                    assert max_cells(s.shape[0]) / 2 < p["ncells"] <= max_cells(s.shape[0]), (name, hint, p)
                    seen["cap"] += 1
                if single_cell(p):
                    assert st[0]["ovf"] + st[0]["dup"] == 0, (name, st)
                elif not w:
                    # a K-th distance beyond 3 cells is certified at ring 3 or 4, or overflows
                    deep = int((kth > 3.001 * p["h"]).sum()) - int(st[0]["ovf"] + st[0]["dup"])
                    seen["deep"] = max(seen["deep"], deep)
    assert seen["single"] and seen["cap"] and seen["deep"] > 0, seen


# ------------------------------------------------------------------------------------------ the whole schedule
@pytest.mark.parametrize("setting", [(0.1, 0, 0.08), (12.0, 31, 40.0), (0.4, 5, 1e3)])
def test_schedule_digest_under_perturbed_tuning(cuda, knobs, setting):
    """The 22 arrays of the index build, Python scheduler and single C entry point, still equal the
    reference's (sha256) for all three digest frames with the cell-size knobs far from their defaults."""
    from ffb6d_b200.schedule import image_pyramid
    from ffb6d_b200.synthetic import make_frame
    knobs(*setting)
    frames = json.load(open(os.path.join(GOLDEN, "schedule_digest.json")))["frames"]
    for fname, d in sorted(frames.items()):
        fr = make_frame(d["seed"], n_points=d["n_points"])
        cld = torch.from_numpy(fr["cld"])[None].cuda()
        xyz = torch.from_numpy(fr["dpt_xyz"])[None].cuda()
        py = F.build_ffb6d_indices(cld, xyz)
        nat = F.build_ffb6d_indices_native(cld, image_pyramid(xyz, (2, 4, 8)), xyz.shape[1:3])
        for key, meta in d["keys"].items():
            for which, res in (("python", py), ("native", nat)):
                got = np.ascontiguousarray(res[key][0].cpu().numpy().astype(np.int32))
                assert list(got.shape) == meta["shape"], (fname, which, key)
                assert hashlib.sha256(got.tobytes()).hexdigest() == meta["sha256"], (fname, which, key, setting)
