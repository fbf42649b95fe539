"""The clouds of the farthest point sampling cases, regenerated from seeds (tests/golden/make_fps_golden.py stores
only the reference's indices for them in tests/golden/fps_cases.npz).

CASES: name -> (builder, S).  Every cloud runs with ``init_center`` (``<name>:ic``) and from the reference's random
start (``<name>:rs``, whose first index is the start the device run is given).
"""
import numpy as np

MAX_POINTS = 8 * 14336          # FFB6D_FPS_MAX_POINTS
MAX_SAMPLES = MAX_POINTS


def _rand(seed, n, scale=1.0):
    return (np.random.RandomState(seed).rand(n, 3) * scale).astype(np.float32)


def _lattice(seed, k, step=0.01):
    g = np.stack(np.meshgrid(*[np.arange(k)] * 3, indexing="ij"), -1).reshape(-1, 3) * step
    return g[np.random.RandomState(seed).permutation(len(g))].astype(np.float32)


def _box_surface(seed, n):
    """Vertices on the faces of a 0.16 x 0.21 x 0.07 m box, like a YCB mesh's points.xyz."""
    rs = np.random.RandomState(seed)
    half = np.array([0.08, 0.105, 0.035])
    p = (rs.rand(n, 3) * 2 - 1) * half
    ax = rs.randint(0, 3, n)
    p[np.arange(n), ax] = np.where(rs.rand(n) < 0.5, -1, 1) * half[ax]
    return p.astype(np.float32)


def _dups(seed):
    p = _rand(seed, 200)
    return np.repeat(p, 3, 0)[np.random.RandomState(seed + 1).permutation(600)]


def _collinear(seed):
    t = np.random.RandomState(seed).rand(300)
    return (np.array([0.3, -0.2, 0.1]) + t[:, None] * np.array([1.0, 2.0, -0.5])).astype(np.float32)


def _coplanar(seed):
    p = _rand(seed, 500)
    p[:, 2] = 0.25
    return p


CASES = {
    "n1": (lambda: _rand(1, 1), 3),
    "n2": (lambda: _rand(2, 2), 4),
    "n31": (lambda: _rand(31, 31), 33),
    "n32": (lambda: _rand(32, 32), 32),
    "n33": (lambda: _rand(33, 33), 16),
    "n1024": (lambda: _rand(1024, 1024), 64),
    "n1025": (lambda: _rand(1025, 1025), 64),
    "n14336_one_cta": (lambda: _rand(14336, 14336), 64),
    "n14337_two_ctas": (lambda: _rand(14337, 14337), 64),
    "ycb_2621_kps": (lambda: _box_surface(7, 2621), 8),
    "ycb_2621_all": (lambda: _box_surface(7, 2621), 2621),
    "linemod_40000": (lambda: _box_surface(8, 40000), 64),
    "max_points": (lambda: _rand(9, MAX_POINTS), 64),
    "max_samples": (lambda: _rand(10, 1000), MAX_SAMPLES),
    "all_equal": (lambda: np.tile(np.float32([[0.1, -0.2, 0.3]]), (50, 1)), 10),
    "lattice_ties": (lambda: _lattice(11, 8), 100),
    "lattice_ties_5_ctas": (lambda: _lattice(12, 40), 100),
    "duplicates": (lambda: _dups(13), 700),
    "s_gt_p": (lambda: _rand(14, 5), 12),
    "collinear": (lambda: _collinear(15), 50),
    "coplanar": (lambda: _coplanar(16), 80),
    "scale_1e4": (lambda: _rand(17, 3000, 1e4), 32),
    "scale_1e-4": (lambda: _rand(18, 3000, 1e-4), 32),
}

# one batch of G clouds of P points, and the prefix lengths of its ragged form (n_points_per_cloud)
BATCH_G, BATCH_P = 5, 700
BATCH_N = (700, 1, 350, 699, 33)


def batch_clouds():
    return np.stack([_rand(100 + g, BATCH_P) for g in range(BATCH_G)])


# arrays the object-info restatement is compared on (float32 meshes, as read from .ply, and one float64)
def objinfo_arrays():
    return {"box": _box_surface(7, 2621), "small": _rand(18, 3000, 1e-4),
            "f64": np.random.RandomState(19).randn(400, 3) * 0.05}
