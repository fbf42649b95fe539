"""Edge cases of voxel-grid subsampling, shared by the device test (tests/test_gpu_grid_edges.py) and the
oracle test (tests/test_grid_oracle_edges.py).  Both compare an implementation with the reference's own
compiled ``grid_subsampling`` (``oracle/_ref/libgrid_ref.so``, built by ``make -C oracle ref``).

The reference computes, in float32 (grid_subsampling.cpp:25-56, cloud.cpp:27-67):

    min, max   = min_point / max_point: start from point 0, replace on a strict '<' / '>'
    origin     = floor(min * (1 / dl)) * dl
    NX, NY     = (size_t)floor((max - origin) / dl) + 1
    iX, iY, iZ = (size_t)floor((p - origin) / dl)
    key        = iX + NX * iY + NX * NY * iZ            (mod 2^64)

``(size_t)`` of a float is what x86-64 compilers emit for it (:func:`size_t_of`), not a saturating cast: an
index of -1 wraps to 2^64 - 1, NaN gives 2^63.  :func:`voxel_keys` restates this in numpy, so that each row of
every implementation can be given its voxel key, and rows are compared key by key.
"""
import numpy as np

INT_MIN, INT_MAX = np.iinfo(np.int32).min, np.iinfo(np.int32).max
TWO63 = np.float32(2.0 ** 63)
INDEFINITE = np.uint64(1 << 63)           # what cvttss2si returns for NaN and out-of-range input


# ----------------------------------------------------------------------------- the reference's arithmetic
def size_t_of(f):
    """``(size_t)f`` for float32 ``f`` as x86-64 code computes it: below 2^63 a signed ``cvttss2si``; from 2^63
    up, ``cvttss2si(f - 2^63)`` with the top bit flipped.  ``cvttss2si`` gives 2^63 for NaN and for values
    outside [-2^63, 2^63), so NaN and -inf map to 2^63, +inf and values >= 2^64 to 0, -1 to 2^64 - 1."""
    f = np.asarray(f, np.float32)
    hi = f >= TWO63
    g = np.where(hi, f - TWO63, f).astype(np.float32)
    ok = (g >= -TWO63) & (g < TWO63)
    out = np.full(f.shape, INDEFINITE, np.uint64)
    out[ok] = g[ok].astype(np.int64).view(np.uint64)
    return np.where(hi, out ^ INDEFINITE, out)


def limits(pts):
    """min_point / max_point (cloud.cpp:27-67): a NaN at point 0 stays the limit, later NaNs are never taken,
    and among equal values (+0 and -0) the first in input order wins."""
    mn, mx = np.empty(3, np.float32), np.empty(3, np.float32)
    for a in range(3):
        v = pts[:, a]
        if np.isnan(v[0]):
            mn[a] = mx[a] = v[0]
            continue
        ok = ~np.isnan(v)
        for out, ext in ((mn, np.min), (mx, np.max)):
            e = ext(v[ok])
            out[a] = v[np.flatnonzero(v == e)[0]]
    return mn, mx


def grid_frame(pts, dl):
    """(origin [3], NX, NY) as grid_subsampling.cpp:25-31 computes them."""
    dl = np.float32(dl)
    mn, mx = limits(pts)
    with np.errstate(invalid="ignore", over="ignore"):
        org = (np.floor(mn * (np.float32(1) / dl)) * dl).astype(np.float32)
        NX = size_t_of(np.floor((mx[0] - org[0]) / dl)) + np.uint64(1)
        NY = size_t_of(np.floor((mx[1] - org[1]) / dl)) + np.uint64(1)
    return org, NX, NY


def voxel_indices(pts, dl):
    """[N, 3] uint64 (iX, iY, iZ) of grid_subsampling.cpp:53-55."""
    org, _, _ = grid_frame(pts, dl)
    with np.errstate(invalid="ignore", over="ignore"):
        return size_t_of(np.floor(((pts - org).astype(np.float32) / np.float32(dl)).astype(np.float32)))


def voxel_keys(pts, dl):
    """[N] uint64 voxel key of every point (grid_subsampling.cpp:56, wrapping mod 2^64)."""
    _, NX, NY = grid_frame(pts, dl)
    ijk = voxel_indices(pts, dl)
    with np.errstate(over="ignore"):
        return ijk[:, 0] + NX * ijk[:, 1] + NX * NY * ijk[:, 2]


def negative_index_minima(dl, lo=-5.0, hi=5.0, ulps=4):
    """Every float32 ``m`` in [lo, hi] within ``ulps`` below a multiple ``fl(k·dl)`` whose origin
    ``fl(floor(fl(m·fl(1/dl)))·dl)`` lies above ``m``: a cloud whose minimum is ``m`` has points at voxel
    index -1.  These sit next to multiples of dl, so the search walks them instead of sampling at random."""
    d = np.float32(dl)
    k = np.arange(np.floor(lo / dl), np.ceil(hi / dl) + 1).astype(np.float32)
    m = (k * d).astype(np.float32)
    cands = [m]
    for _ in range(ulps):
        m = np.nextafter(m, np.float32(-np.inf))
        cands.append(m)
    m = np.concatenate(cands)
    m = m[(m >= lo) & (m <= hi)]
    org = (np.floor(m * (np.float32(1) / d)) * d).astype(np.float32)
    return np.unique(m[org > m])


# ----------------------------------------------------------------------------- cases
class Case:
    def __init__(self, pts, dl, feats=None, labels=None):
        self.pts = np.ascontiguousarray(pts, np.float32)
        self.dl = float(np.float32(dl))
        self.feats = None if feats is None else np.ascontiguousarray(feats, np.float32)
        self.labels = None if labels is None else np.ascontiguousarray(labels, np.int32)
        if self.labels is not None and self.labels.ndim == 1:
            self.labels = self.labels[:, None]


def _feats_labels(rs, n, fdim=3, ldim=1):
    return rs.rand(n, fdim).astype(np.float32), rs.randint(-3, 9, (n, ldim)).astype(np.int32)


FOUR_POINTS = np.array([[-3.7, 0, 0], [-3.69, 0, 0], [-3.61, 0.05, 0], [-3.5, 0.05, 0]], np.float32)
NEG_DLS = (0.02, 0.06, 0.1)
NEG_AXES = ("x", "y", "z", "xyz")


def negative_index_case(dl, axes, seed):
    """A dense cloud of 8 voxels per side whose minimum on ``axes`` is a searched value with origin > min, so
    that the points at the minimum have index -1 and their wrapped key lands in an occupied voxel."""
    rs = np.random.RandomState(seed)
    found = negative_index_minima(dl)
    assert len(found) >= 3, "no (min, dl) pair with origin above the minimum found at dl=%g" % dl
    d = np.float32(dl)
    mins = rs.uniform(-4, 4, 3).astype(np.float32)
    neg = ["xyz".index(a) for a in axes]
    mins[neg] = rs.choice(found, len(neg), replace=False)
    n = 4000
    pts = (mins + rs.rand(n, 3).astype(np.float32) * (np.float32(8) * d)).astype(np.float32)
    pts[rs.choice(n, 40, replace=False)] = mins           # whole points at the minimum corner
    for a in neg:
        pts[rs.choice(n, 40, replace=False), a] = mins[a]  # and points at the minimum of one axis
    assert np.array_equal(limits(pts)[0], mins)
    ijk = voxel_indices(pts, dl).view(np.int64)
    for a in range(3):
        assert (ijk[:, a] == -1).any() == (a in neg), "axis %d: the cloud misses the case it is built for" % a
    return Case(pts, dl, *_feats_labels(rs, n, ldim=2))


def negative_index_pair_clouds(dl):
    """For every searched minimum ``m`` at ``dl`` and every axis ``a``, three points: A at ``m`` on axis a and
    one voxel up on axis b = a + 1, B at the far end of axis a in the first voxel of axis b, C holding the
    minimum of axis b.  A's index -1 wraps its key to B's voxel (to a key near 2^64 when a is z, which has no
    slab below it)."""
    d = np.float32(dl)
    for m in negative_index_minima(dl):
        for a in range(3):
            b = (a + 1) % 3
            pts = np.zeros((3, 3), np.float32)
            pts[:, a] = [m, m + np.float32(5.5) * d, m + np.float32(2.5) * d]
            pts[:, b] = [np.float32(1.5) * d, np.float32(0.5) * d, 0]
            yield m, a, Case(pts, dl)


FAR_OFFSETS = (1e3, -1e4, 1e5)
FAR_DLS = (0.02, 0.1, 1.0)


def far_case(offset, dl, seed, lattice):
    """A cloud 1e3 - 1e5 m from the origin, where p - origin keeps few bits.  ``lattice``: the points lie at
    ``origin + k·dl`` and half-way between (on and inside voxel faces), as float32 rounds them."""
    rs = np.random.RandomState(seed)
    d = np.float32(dl)
    base = (np.float32(offset) + rs.uniform(-1, 1, 3).astype(np.float32) * d * 50).astype(np.float32)
    if lattice:
        org = (np.floor(base * (np.float32(1) / d)) * d).astype(np.float32)
        k = rs.randint(0, 24, (3000, 3)).astype(np.float32) * np.float32(0.5)
        pts = (org + (k * d).astype(np.float32)).astype(np.float32)
    else:
        pts = (base + rs.rand(3000, 3).astype(np.float32) * d * np.float32(12)).astype(np.float32)
    return Case(pts, dl, *_feats_labels(rs, len(pts)))


def key_collision_case(e, seed):
    """dl = 2^-e with NX = NY = 2^24, so NX·NY·iZ wraps 2^64 at iZ = 2^16: the voxels (i, j, k) and
    (i, j, k + 2^16) share a key and the reference merges them.  All coordinates are exact in float32."""
    rs = np.random.RandomState(seed)
    d = np.float32(2.0 ** -e)
    ix = np.array([0, 1, 2 ** 24 - 1], np.float32)
    iz = np.array([0, 1, 2 ** 16, 2 ** 16 + 1, 2 ** 17, 3], np.float32)
    g = np.stack(np.meshgrid(ix, ix, iz, indexing="ij"), -1).reshape(-1, 3)
    g = np.repeat(g, 3, 0)
    g = g[rs.permutation(len(g))]
    pts = ((g - np.float32(37)) * d).astype(np.float32)     # origin -37·dl, exact
    org, NX, NY = grid_frame(pts, d)
    assert org[0] == np.float32(-37) * d and NX == NY == 2 ** 24
    nvox = len(np.unique(voxel_indices(pts, d), axis=0))
    assert len(np.unique(voxel_keys(pts, d))) < nvox, "no two voxels share a key"
    return Case(pts, d, *_feats_labels(rs, len(pts), fdim=2, ldim=1))


WIDE = ((1e-6, 1000.0), (1e-7, 1000.0), (1e-9, 1000.0))


def wide_case(dl, extent, seed):
    """A cloud so wide against dl that NX·NY·NZ (and for dl <= 1e-7 NX·NY) passes 2^64.  Clusters of points a
    few float32 ulps across (an ulp there spans many voxels), with repeats, so that voxels hold several points."""
    rs = np.random.RandomState(seed)
    c = np.repeat(rs.uniform(-extent / 2, extent / 2, (60, 3)).astype(np.float32), 40, 0)
    pts = (c + rs.randint(-3, 4, c.shape).astype(np.float32) * np.spacing(np.abs(c))).astype(np.float32)
    _, NX, NY = grid_frame(pts, dl)
    ijk = voxel_indices(pts, dl)
    NZ = int(ijk[:, 2].max()) + 1
    assert int(NX) * int(NY) * NZ >= 2 ** 64
    return Case(pts, dl, *_feats_labels(rs, len(pts)))


def non_finite_case(kind, seed):
    """NaN at point 0 (one axis or all three), NaN at later points, +inf / -inf / both among the coordinates.
    The reference's output is whatever it computes; the comparison takes it as it is."""
    rs = np.random.RandomState(seed)
    n = 600
    pts = (rs.rand(n, 3) * 0.5).astype(np.float32)
    rows = rs.choice(np.arange(1, n), 12, replace=False)
    if kind == "nan_point0_x":
        pts[0, 0] = np.nan
    elif kind == "nan_point0_xyz":
        pts[0] = np.nan
    elif kind == "nan_later":
        pts[rows, rs.randint(0, 3, 12)] = np.nan
        pts[rows[:3]] = np.nan
    elif kind == "pos_inf":
        pts[rows, rs.randint(0, 3, 12)] = np.inf
    elif kind == "neg_inf":
        pts[rows, rs.randint(0, 3, 12)] = -np.inf
    elif kind == "both_inf":
        pts[rows[:6], rs.randint(0, 3, 6)] = np.inf
        pts[rows[6:], rs.randint(0, 3, 6)] = -np.inf
        pts[rows[0]] = [np.inf, -np.inf, np.inf]
    else:
        raise ValueError(kind)
    return Case(pts, 0.1, *_feats_labels(rs, n))


NON_FINITE = ("nan_point0_x", "nan_point0_xyz", "nan_later", "pos_inf", "neg_inf", "both_inf")


def one_voxel_case(n, seed, dl=0.1):
    """n points inside one voxel (M = 1).  Features of ones: once n > 2^24 their fp32 sum stops at 2^24 and
    (float)n rounds, so the mean is 2^24 / fl(n), not 1."""
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 3), dtype=np.float32)
    pts *= np.float32(0.08)
    pts += np.float32(0.01)
    labels = np.zeros((n, 1), np.int32)
    labels[rng.integers(0, n, n // 3)] = 7
    return Case(pts, dl, np.ones((n, 1), np.float32), labels)


FDIMS = (1, 2, 7, 64)


def features_case(fdim, dl, seed):
    """fdim-channel features with magnitudes spread over 2^-40 - 2^40 and both signs, so the fp32 sums depend
    on their order; about 5 points per voxel."""
    rs = np.random.RandomState(seed)
    n = 6000
    pts = (rs.rand(n, 3).astype(np.float32) * np.float32(dl * 10)).astype(np.float32)
    mag = np.exp2(rs.uniform(-40, 40, (n, fdim)))
    feats = (mag * rs.choice([-1.0, 1.0], (n, fdim)) * rs.uniform(1, 2, (n, fdim))).astype(np.float32)
    return Case(pts, dl, feats, rs.randint(0, 4, n))


LDIMS = (1, 3, 5)


def labels_case(ldim, dl, seed):
    """ldim label columns drawn from {INT_MIN, INT_MAX, -1, 0, 3}, a few points per voxel: many voxels hold
    INT_MIN, INT_MAX, -1 and 0 together, with and without a tie for the top count."""
    rs = np.random.RandomState(seed)
    n = 5000
    pts = (rs.rand(n, 3).astype(np.float32) * np.float32(dl * 12)).astype(np.float32)
    vals = np.array([INT_MIN, INT_MAX, -1, 0, 3], np.int32)
    labels = vals[rs.randint(0, len(vals), (n, ldim))]
    # a voxel of its own, past the others, with nine points: the four extremes twice each, and a ninth that
    # breaks the tie by column
    pts[:9] = np.float32(dl * 12.5)
    labels[:8] = np.tile(vals[:4], 2)[:, None]
    labels[8] = [(INT_MAX, -1, 0, INT_MIN, 0)[l] for l in range(ldim)]
    return Case(pts, dl, (rs.rand(n, 2)).astype(np.float32), labels)


# ----------------------------------------------------------------------------- comparison
def run(fn, case, with_keys=True):
    """Run ``fn(points, features, labels [N, ld], dl) -> (points, features or None, labels)`` on ``case``.
    With ``with_keys`` two label columns carrying the high and low halves of each point's voxel key
    (:func:`voxel_keys`) are appended: every point of a voxel has the same key, so each output row's vote
    returns its voxel's key exactly.  Returns (points, features, labels, keys) with keys None otherwise."""
    labels = case.labels
    if with_keys:
        k = voxel_keys(case.pts, case.dl)
        kl = np.stack([(k >> np.uint64(32)).astype(np.uint32), k.astype(np.uint32)], 1).view(np.int32)
        labels = kl if labels is None else np.concatenate([labels, kl], 1)
    sp, sf, sl = fn(case.pts, case.feats, labels, case.dl)
    keys = None
    if with_keys:
        kk = sl[:, -2:].view(np.uint32).astype(np.uint64)
        keys = (kk[:, 0] << np.uint64(32)) | kk[:, 1]
        sl = sl[:, :-2] if case.labels is not None else None
    return sp, sf, sl, keys


def same_bits(got, want, what):
    """Bit for bit, signed zeros included; NaNs at the same positions (their payloads are the hardware's)."""
    assert got.shape == want.shape, "%s: shape %s vs %s" % (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    bad = (gn != wn) | (~gn & (got.view(np.uint32) != want.view(np.uint32)))
    if bad.any():
        r = np.argwhere(bad)[0]
        raise AssertionError("%s: %d of %d values differ, first at %s: %r vs %r"
                             % (what, bad.sum(), bad.size, tuple(r), got[tuple(r)], want[tuple(r)]))


def vote_tables(case):
    """Per voxel (ascending key) and label column: (smallest label of top count, set of top-count labels as
    int64 codes voxel·2^32 + label, number of labels tied at the top)."""
    keys = voxel_keys(case.pts, case.dl)
    uk, inv = np.unique(keys, return_inverse=True)
    out = []
    for l in range(case.labels.shape[1]):
        lab = case.labels[:, l].astype(np.int64)
        o = np.lexsort((lab, inv))
        g, v = inv[o], lab[o]
        start = np.flatnonzero(np.r_[True, (g[1:] != g[:-1]) | (v[1:] != v[:-1])])
        cnt = np.diff(np.r_[start, len(o)])
        rg, rv = g[start], v[start]
        top = np.zeros(len(uk), np.int64)
        np.maximum.at(top, rg, cnt)
        is_top = cnt == top[rg]
        first = np.full(len(uk), INT_MAX, np.int64)
        np.minimum.at(first, rg[is_top], rv[is_top])
        codes = rg[is_top] * (1 << 32) + (rv[is_top] - INT_MIN)
        out.append((first, codes, np.bincount(rg[is_top], minlength=len(uk))))
    return uk, out


def assert_matches_reference(got, want, case, ordered=True):
    """``got`` (the implementation under test) against ``want`` (the reference), both from :func:`run`.
    Rows are matched by voxel key; barycentres and mean features must be bitwise equal.  Labels: ``got`` takes
    the smallest of the labels tied for the top count (DESIGN.md §4.3), the reference the first in its hash-map
    order, so where the top count is unique both equal it and otherwise the reference's is one of the tied.
    ``ordered``: ``got``'s rows come by ascending voxel key."""
    gp, gf, gl, gk = got
    wp, wf, wl, wk = want
    assert len(gk) == len(wk), "%d voxels, the reference has %d" % (len(gk), len(wk))
    uk = np.unique(voxel_keys(case.pts, case.dl))
    ow = np.argsort(wk, kind="stable")
    assert np.array_equal(wk[ow], uk), "the reference's voxels are not those of the key restatement"
    if ordered:
        assert np.array_equal(gk, uk), "rows are not by ascending voxel key, or not the reference's voxels"
    og = np.argsort(gk, kind="stable")
    assert np.array_equal(gk[og], uk)
    same_bits(gp[og], wp[ow], "barycentres")
    if case.feats is not None:
        same_bits(gf[og], wf[ow], "mean features")
    if case.labels is not None:
        _, tables = vote_tables(case)
        gl, wl = gl[og], wl[ow]
        for l, (smallest, codes, ntop) in enumerate(tables):
            assert np.array_equal(gl[:, l], smallest), "labels[:, %d]: not the smallest label of top count" % l
            assert np.array_equal(wl[ntop == 1, l], smallest[ntop == 1]), "labels[:, %d]: unique top" % l
            wc = np.arange(len(uk)) * (1 << 32) + (wl[:, l].astype(np.int64) - INT_MIN)
            assert np.isin(wc, codes).all(), "labels[:, %d]: the reference's label is not of top count" % l
