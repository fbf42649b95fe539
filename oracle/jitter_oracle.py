"""numpy restatement of the colour jitter (ffb6d_b200/csrc/color_jitter.cu): torchvision 0.26's
``ColorJitter(0.2, 0.2, 0.2, 0.05)`` on a PIL RGB image with Pillow 12.2, applied from a plan of
:func:`ffb6d_b200.augment.draw_color_jitter`.  No Pillow: every op is written out with Pillow's integer, float32 and
float64 arithmetic (numpy's float32 ops round each result, as C on x86-64 does).  Pinned to the real library by
tests/golden/jitter_cases.npz and checked exhaustively by tests/golden/check_jitter_pil.py."""
import numpy as np

f32, f64 = np.float32, np.float64
OPS = ("brightness", "contrast", "saturation", "hue")


def luma(rgb):
    """``convert("L")``: (19595 R + 38470 G + 7471 B + 0x8000) >> 16, int64."""
    x = rgb.astype(np.int64)
    return (19595 * x[..., 0] + 38470 * x[..., 1] + 7471 * x[..., 2] + 0x8000) >> 16


def blend(a, b, factor):
    """``Image.blend(a, b, factor)`` per byte: the factor as a C float, a + f * (b - a) in float32 (product and sum
    rounded separately); truncated for 0 <= f <= 1, else clipped to [0, 255] first."""
    f = f32(factor)
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    t = a.astype(f32) + f * (b - a).astype(f32)
    if 0 <= f <= 1:
        return np.trunc(t).astype(np.uint8)
    with np.errstate(invalid="ignore"):
        return np.where(t <= 0, 0, np.where(t >= 255, 255, np.trunc(t))).astype(np.uint8)


def rgb2hsv(rgb):
    """``convert("HSV")`` (Pillow's rgb2hsv_row): float32 ratios, the hue's sum and fmod in float64 stored to float32,
    H and S truncated from float64 products with 255.  Returns uint8 [..., 3]."""
    x = rgb.astype(np.int64)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    mx = np.maximum(np.maximum(r, g), b)
    mn = np.minimum(np.minimum(r, g), b)
    grey = mx == mn
    with np.errstate(divide="ignore", invalid="ignore"):
        cr = (mx - mn).astype(f32)
        s = cr / mx.astype(f32)
        rc, gc, bc = ((mx - c).astype(f32) / cr for c in (r, g, b))
        h = np.where(r == mx, (bc - gc).astype(f64),
                     np.where(g == mx, (2.0 + rc.astype(f64)) - bc.astype(f64),
                              (4.0 + gc.astype(f64)) - rc.astype(f64))).astype(f32)
        h = np.fmod(h.astype(f64) / 6.0 + 1.0, 1.0).astype(f32)
        H = np.clip(np.where(grey, 0, h.astype(f64) * 255.0).astype(np.int64), 0, 255)
        S = np.clip(np.where(grey, 0, s.astype(f64) * 255.0).astype(np.int64), 0, 255)
    return np.stack([H, S, mx], -1).astype(np.uint8)


def _round_away(x):
    """C's round() for x >= 0: half away from zero."""
    t = np.trunc(x)
    return t + (x - t >= 0.5)


def hsv2rgb(hsv):
    """``convert("RGB")`` of an HSV image (Pillow's hsv2rgb): sextant i = floor(h * 6 / 255) and the remainder in
    float64 (remainder stored to float32), fs = (float)(s / 255), p, q, t in float64 (fs * f a float32 product)
    rounded half away from zero.  Returns uint8 [..., 3]."""
    x = hsv.astype(np.int64)
    h, s, v = x[..., 0], x[..., 1], x[..., 2]
    hh = h.astype(f64) * 6.0 / 255.0
    i = np.floor(hh)
    f = (hh - i).astype(f32)
    fs = (s.astype(f64) / 255.0).astype(f32)
    dv = v.astype(f64)
    p = _round_away(dv * (1.0 - fs.astype(f64)))
    q = _round_away(dv * (1.0 - (fs * f).astype(f64)))
    t = _round_away(dv * (1.0 - fs.astype(f64) * (1.0 - f.astype(f64))))
    p, q, t = (np.clip(a, 0, 255).astype(np.int64) for a in (p, q, t))
    table = np.stack([np.stack(c, -1) for c in ((v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q))])
    out = np.take_along_axis(np.moveaxis(table, 0, -2), (i.astype(np.int64) % 6)[..., None, None], -2)[..., 0, :]
    out = np.where((s == 0)[..., None], v[..., None], out)
    return out.astype(np.uint8)


def hue_shift(hue):
    """``np.int32(hue_factor * 255)``, the shift adjust_hue adds to H (mod 256)."""
    return int(np.int32(f64(hue) * 255))


def adjust_brightness(img, f):
    return blend(0, img, f)


def adjust_contrast(img, f):
    L = luma(img)
    mean = int(float(L.sum()) / L.size + 0.5)
    return blend(mean, img, f)


def adjust_saturation(img, f):
    return blend(luma(img)[..., None], img, f)


def adjust_hue(img, hue):
    hsv = rgb2hsv(img)
    hsv[..., 0] = (hsv[..., 0].astype(np.int64) + hue_shift(hue)) & 255
    return hsv2rgb(hsv)


def color_jitter(img, plan):
    """One frame [H,W,3] uint8 through a plan [8]: the four ops in the plan's order."""
    fns = (adjust_brightness, adjust_contrast, adjust_saturation, adjust_hue)
    for op in plan[:4].astype(np.int64):
        img = fns[op](img, plan[4 + op])
    return img
