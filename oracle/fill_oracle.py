"""oracle/fill_oracle.py -- plain-numpy restatement of the YCB dataset's depth completion.

``fill_missing(dpt_raw, cam_scale)`` is ``Basic_Utils.fill_missing(dpt, cam_scale, 1)`` as
``datasets/ycb/ycb_dataset.py:204`` calls it (utils/basic_utils.py:467-487): ip_basic's
``fill_in_multiscale`` (utils/ip_basic/ip_basic/depth_map_utils_ycb.py:290-443) with
``max_depth=3.0``, ``extrapolate=False`` and ``blur_type='bilateral'``.  No OpenCV: dilation and
erosion are shifted max/min with out-of-image pixels ignored, the 5x5 median is the 13th of 25
sorted edge-replicated values, the top masks come from ``argmax``, and the bilateral filter uses
exact float64 weights where OpenCV interpolates a float32 look-up table.  Every stage before the
bilateral is bit-identical to the reference; the bilateral differs from OpenCV's in the last bits
(DESIGN.md §4.10).  Used as the CPU oracle of the CUDA path (ffb6d_b200/csrc/depth_fill.cu).
"""
import numpy as np

F32 = np.float32
T = F32(0.01)             # every `> 0.01` / `< 0.01` of fill_in_multiscale, cast to float32 by numpy
MAX_DEPTH = F32(3.0)
FLT_EPSILON = float(np.finfo(np.float32).eps)
BILATERAL_SIGMA_COLOR = 0.5
BILATERAL_SIGMA_SPACE = 2.0
BILATERAL_RADIUS = 2      # d = 5


def cross(r):
    return [(dy, 0) for dy in range(-r, r + 1)] + [(0, dx) for dx in range(-r, r + 1) if dx]


def square(r):
    return [(dy, dx) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]


def _morph(x, offsets, op, pad_value):
    r = max(max(abs(dy), abs(dx)) for dy, dx in offsets)
    H, W = x.shape
    p = np.pad(x, r, mode="constant", constant_values=pad_value)
    out = None
    for dy, dx in offsets:
        v = p[r + dy:r + dy + H, r + dx:r + dx + W]
        out = v.copy() if out is None else op(out, v)
    return out


def dilate(x, offsets):
    """Max over the structuring element; pixels outside the image take no part."""
    return _morph(x, offsets, np.maximum, -np.inf)


def erode(x, offsets):
    return _morph(x, offsets, np.minimum, np.inf)


def median5(x):
    """5x5 median with replicated edges."""
    H, W = x.shape
    p = np.pad(x, 2, mode="edge")
    stack = np.stack([p[2 + dy:2 + dy + H, 2 + dx:2 + dx + W] for dy, dx in square(2)])
    return np.sort(stack, axis=0)[12]


def top_mask(x):
    """False above the first row of each column with a value > 0.01; a column without one is all
    True (argmax of an all-False column is 0)."""
    first = np.argmax(x > T, axis=0)
    return np.arange(x.shape[0])[:, None] >= first[None, :]


def reflect101(i, n):
    """Index ``i`` folded into ``[0, n)`` by reflection without repeating the edge."""
    if n == 1:
        return np.zeros_like(i)
    period = 2 * (n - 1)
    i = np.mod(i, period)
    return np.where(i >= n, period - i, i)


def bilateral(x):
    """Bilateral filter of diameter 5, sigma_color 0.5, sigma_space 2.0 over reflect-101 borders,
    exact float64 weights; returns ``x`` unchanged when the frame's max - min < FLT_EPSILON."""
    if abs(float(x.max()) - float(x.min())) < FLT_EPSILON:
        return x.copy()
    H, W = x.shape
    rows, cols = np.arange(H), np.arange(W)
    x64 = x.astype(np.float64)
    num = np.zeros((H, W), np.float64)
    den = np.zeros((H, W), np.float64)
    cc = -0.5 / (BILATERAL_SIGMA_COLOR * BILATERAL_SIGMA_COLOR)
    sc = -0.5 / (BILATERAL_SIGMA_SPACE * BILATERAL_SIGMA_SPACE)
    r = BILATERAL_RADIUS
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            r2 = dy * dy + dx * dx
            if r2 > r * r:
                continue
            v = x64[reflect101(rows + dy, H)][:, reflect101(cols + dx, W)]
            d = v - x64
            w = np.exp(r2 * sc) * np.exp(d * d * cc)
            num += v * w
            den += w
    return (num / den).astype(np.float32)


def fill_in_multiscale(depths_in):
    """The stages of fill_in_multiscale on float32 metres; returns the dict of its
    ``show_process`` names (s1 ... s8; s7 and s8 after the bilateral)."""
    x = np.asarray(depths_in, dtype=np.float32)
    near = (x > T) & (x <= F32(1.0))
    med = (x > F32(1.0)) & (x <= F32(2.0))
    far = x > F32(2.0)
    s1 = x.copy()
    v = s1 > T
    s1[v] = MAX_DEPTH - s1[v]

    d_far = dilate(s1 * far, cross(1))
    d_med = dilate(s1 * med, cross(2))
    d_near = dilate(s1 * near, cross(3))
    s2 = s1.copy()
    for d in (d_far, d_med, d_near):
        m = d > T
        s2[m] = d[m]

    s3 = erode(dilate(s2, square(2)), square(2))

    s4 = s3.copy()
    m = s3 > T
    s4[m] = median5(s3)[m]

    empty = ~(s4 > T) & top_mask(s4)
    s5 = s4.copy()
    s5[empty] = dilate(s4, square(4))[empty]

    s6 = s5.copy()
    top = top_mask(s5)

    s7 = s6.copy()
    for _ in range(6):
        empty = (s7 < T) & top
        s7[empty] = dilate(s7, square(2))[empty]

    valid = (s7 > T) & top
    s7[valid] = median5(s7)[valid]
    s7_median = s7.copy()
    s7[valid] = bilateral(s7)[valid]

    s8 = s7.copy()
    m = s8 > T
    s8[m] = MAX_DEPTH - s8[m]
    return dict(s1_inverted_depths=s1, s2_dilated_depths=s2, s3_closed_depths=s3, s4_blurred_depths=s4,
                s5_combined_depths=s5, s6_extended_depths=s6, s7_median_depths=s7_median,
                s7_blurred_depths=s7, s8_inverted_depths=s8, bilateral_mask=valid)


def fill_missing(dpt_raw, cam_scale, return_stages=False):
    """``bs_utils.fill_missing(dpt_raw, cam_scale, 1)``: raw uint16 depth ``[H,W]`` (or ``[B,H,W]``) ->
    completed depth in raw units, float32.  ``return_stages`` adds the dict of
    :func:`fill_in_multiscale` (single frame only)."""
    raw = np.asarray(dpt_raw)
    cs = F32(cam_scale)
    if raw.ndim == 3:
        if return_stages:
            raise ValueError("return_stages needs a single frame")
        return np.stack([fill_missing(f, cs) for f in raw])
    x = raw.astype(np.float32) / cs
    st = fill_in_multiscale(x)
    out = st["s8_inverted_depths"] / F32(1) * cs
    return (out, st) if return_stages else out
