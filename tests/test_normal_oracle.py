"""CPU: the depth-normal oracle (``oracle/normal_oracle.py``, DESIGN.md §4.30) against closed forms: constant depth,
integer ramps, both thresholds at their edges, holes, border pixels with 3 and 5 neighbours, a fit left with one axis,
``point_into_surface`` and per-frame focal lengths."""
import numpy as np

from oracle.normal_oracle import depth_normal, ycb_mm

FX, FY = 1066.778, 1067.487


def _ulps(a, b):
    """Per-component distance in float32 ulps (sign-magnitude order)."""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


def _closed(g, h, d, fx=FX, fy=FY):
    """normalize(fx g, fy h, -d) in float64, rounded once to float32."""
    v = np.stack(np.broadcast_arrays(np.float64(fx) * g, np.float64(fy) * h, -np.asarray(d, np.float64)), -1)
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)


def test_constant_depth_faces_the_camera():
    n = depth_normal(np.full((23, 31), 812, np.uint16), FX, FY)
    assert n.dtype == np.float32 and n.shape == (23, 31, 3)
    assert np.array_equal(n, np.broadcast_to(np.float32([0, 0, -1]), n.shape))


def test_integer_ramps():
    y, x = np.mgrid[:40, :50]
    for g, h in ((1, 0), (0, 1), (2, -1), (-3, 1)):       # (|g| + |h|) r < 20 with r = 5: every neighbour accepted
        d = 900 + g * x + h * y
        n = depth_normal(d.astype(np.uint16), FX, FY)
        assert _ulps(n, _closed(g, h, d)).max() <= 1, (g, h)


def test_difference_threshold_is_strict():
    r, y, x = 5, 12, 12
    for t, accepted in ((19, True), (20, False), (-19, True), (-20, False)):
        D = np.full((25, 25), 1000, np.uint16)
        D[y, x + r] = 1000 + t
        n = depth_normal(D, FX, FY)[y, x]
        if accepted:    # A0 = A2 = 6 r^2, A1 = 0, b0 = r t, b1 = 0: ddx = 6 r^3 t, det = 36 r^4
            assert _ulps(n, _closed(t / (6.0 * r), 0.0, 1000)).max() <= 1, t
        else:           # the neighbour left out, b = 0
            assert np.array_equal(n, np.float32([0, 0, -1])), t


def test_distance_threshold_and_holes():
    D = np.full((15, 15), 1999, np.uint16)
    assert np.array_equal(depth_normal(D, FX, FY)[7, 7], np.float32([0, 0, -1]))
    D[7, 7] = 2000
    n = depth_normal(D, FX, FY)
    assert np.array_equal(n[7, 7], np.zeros(3, np.float32))
    D[7, 7] = 0
    assert np.array_equal(depth_normal(D, FX, FY)[7, 7], np.zeros(3, np.float32))
    # a hole is a neighbour like any other: delta = -d, accepted while d < difference_threshold
    D = np.full((15, 15), 10, np.uint16)
    D[7, 12] = 0
    assert depth_normal(D, FX, FY)[7, 7][0] != 0
    assert np.array_equal(depth_normal(np.zeros((9, 9), np.uint16), FX, FY), np.zeros((9, 9, 3), np.float32))


def test_border_pixels():
    r = 5
    D = np.full((20, 20), 1000, np.uint16)
    a, b, c = 7, -4, 3
    D[0, r], D[r, 0], D[r, r] = 1000 + a, 1000 + b, 1000 + c
    # corner (0,0): neighbours (r,0), (0,r), (r,r); A0 = A2 = 2 r^2, A1 = r^2, b0 = r (a + c), b1 = r (b + c)
    A0, A1, A2, b0, b1 = 2 * r * r, r * r, 2 * r * r, r * (a + c), r * (b + c)
    det, ddx, ddy = A0 * A2 - A1 * A1, A2 * b0 - A1 * b1, A0 * b1 - A1 * b0
    v = np.array([FX * ddx, FY * ddy, -(det * 1000.0)])
    assert np.array_equal(depth_normal(D, FX, FY)[0, 0], (v / np.sqrt((v[0] ** 2 + v[1] ** 2) + v[2] ** 2)).astype(np.float32))
    # edge pixel (0, x): 5 neighbours, y in {0, r}; on a ramp the fit is exact
    y, x = np.mgrid[:20, :20]
    d = 700 + 2 * x - y
    n = depth_normal(d.astype(np.uint16), FX, FY)
    for py, px in ((0, 9), (19, 9), (9, 0), (9, 19), (0, 0), (19, 19)):
        assert _ulps(n[py, px], _closed(2, -1, d[py, px])).max() <= 1, (py, px)


def test_one_axis_gives_zero():
    # rows alternate by 100 mm with r = 1: every neighbour off the row is rejected, A2 = A1 = 0, det = 0
    y = np.arange(12)[:, None]
    D = np.broadcast_to(1000 + 100 * (y % 2) + np.arange(16)[None, :], (12, 16)).astype(np.uint16)
    assert np.array_equal(depth_normal(D, FX, FY, k_size=1), np.zeros((12, 16, 3), np.float32))


def test_point_into_surface():
    y, x = np.mgrid[:30, :30]
    D = (1200 + x - 2 * y).astype(np.uint16)
    D[4, 4] = 0
    out, into = depth_normal(D, FX, FY), depth_normal(D, FX, FY, point_into_surface=True)
    valid = D != 0
    assert np.array_equal(into[valid], -out[valid])
    assert np.array_equal(into[~valid], np.zeros((1, 3), np.float32))


def test_per_frame_focal_lengths():
    y, x = np.mgrid[:25, :35]
    d = 1500 + x + y
    D = np.stack([d, d]).astype(np.uint16)
    fx, fy = [FX, 572.4114], [FY, 573.57043]
    n = depth_normal(D, fx, fy)
    for b in range(2):
        assert _ulps(n[b], _closed(1, 1, d, fx[b], fy[b])).max() <= 1
        assert np.array_equal(n[b], depth_normal(D[b], fx[b], fy[b]))
    assert not np.array_equal(n[0], n[1])


def test_ycb_millimetres():
    v = np.float32([0, 9.999999, 10, 19.99999, 123456.7, 29999.998, 30000.0])
    assert ycb_mm(v).tolist() == [int(np.float32(a) / np.float32(10)) for a in v]
