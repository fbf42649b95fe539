"""numpy restatement of the augmentation kernels (ffb6d_b200/csrc/augment.cu): the datasets' ``rgb_add_noise`` and
``add_real_back`` applied from a record of :mod:`ffb6d_b200.augment` and given normal fields.  Bitwise the device's
arithmetic; pinned to the reference's own functions by tests/golden/aug_cases.npz."""
import numpy as np

from ffb6d_b200 import augment as A

f32, f64 = np.float32, np.float64
_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def _reflect101(i, n):
    i = np.where(i < 0, -i, i)
    return np.where(i >= n, 2 * n - 2 - i, i)


def fma32(a, b, c):
    """float32 fma(a, b, c), correctly rounded: the product of two float32 is exact in float64, the float64 sum is
    rounded to odd (its error recovered by TwoSum), and rounding that to float32 is then a single rounding."""
    p = np.asarray(a, f32).astype(f64) * np.asarray(b, f32).astype(f64)
    c = np.asarray(c, f32).astype(f64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(np.int64) & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def bgr2hsv(img):
    """COLOR_BGR2HSV on 8U (OpenCV's integer path); channel 0 plays blue.  Returns int64 (h, s, v)."""
    x = img.astype(np.int64)
    b, g, r = x[..., 0], x[..., 1], x[..., 2]
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    i = np.arange(256, dtype=f64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i > 0, np.rint((255 << 12) / i), 0).astype(np.int64)
        hdiv = np.where(i > 0, np.rint((180 << 12) / (6.0 * i)), 0).astype(np.int64)
    s = (diff * sdiv[v] + (1 << 11)) >> 12
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * hdiv[diff] + (1 << 11)) >> 12
    h = h + np.where(h < 0, 180, 0)
    return h, s, v


def hsv2bgr(h, s, v):
    """COLOR_HSV2BGR on 8U (h < 180), as OpenCV 4.13 computes it on x86-64 with AVX2 / AVX-512: float32, fused
    1 - s*f, and the product with 255 truncated in the 32-pixel vector loop, rounded in the scalar loop over the last
    W % 32 pixels of each row (the last axis of h is the row)."""
    h, s, v = (np.asarray(t, np.int64) for t in (h, s, v))
    fs = s.astype(f32) * f32(1.0 / 255.0)
    fv = v.astype(f32) * f32(1.0 / 255.0)
    hh = h.astype(f32) * f32(6.0 / 180.0)
    sector = np.floor(hh).astype(np.int64)
    fr = hh - sector.astype(f32)
    one = f32(1)
    tab = np.stack([fv, fv * (one - fs), fv * fma32(-fs, fr, one), fv * fma32(-fs, one - fr, one)], -1)
    out = np.take_along_axis(tab, _SECTOR[np.where((sector >= 0) & (sector < 6), sector, 0)], -1)
    out = np.where((s == 0)[..., None], fv[..., None], out) * f32(255)
    W = h.shape[-1]
    simd = np.arange(W) < W - W % 32
    out = np.where(simd[:, None], np.trunc(out), np.rint(out))
    return np.clip(out, 0, 255).astype(np.uint8)


def hsv(img, sf, vf):
    """The HSV stage: BGR2HSV, S*sf and V*vf in float64 truncated into uint16 and clipped to 255, HSV2BGR."""
    h, s, v = bgr2hsv(img)
    s = np.minimum(255, (s * f64(sf)).astype(np.uint16).astype(np.int64))
    v = np.minimum(255, (v * f64(vf)).astype(np.uint16).astype(np.int64))
    return hsv2bgr(h, s, v)


def filter2d(img, kern):
    """filter2D(img, -1, kern) on 8U by direct summation: the kernel rounded to float32, a running fma over its
    nonzero taps in row-major order, rounded half to even (OpenCV's non-DFT path)."""
    k = np.asarray(kern, f64).astype(f32)
    a = k.shape[0]
    H, W = img.shape[:2]
    acc = np.zeros(img.shape, f32)
    for i in range(a):
        rows = _reflect101(np.arange(H) + i - a // 2, H)
        for j in range(a):
            if k[i, j] == 0:
                continue
            cols = _reflect101(np.arange(W) + j - a // 2, W)
            acc = fma32(img[rows][:, cols].astype(f32), k[i, j], acc)
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def gaussian(img, taps):
    """GaussianBlur on 8U: OpenCV's fixed-point separable sum, (sum + 2^15) >> 16."""
    n = len(taps)
    H, W = img.shape[:2]
    x = img.astype(np.int64)
    row = sum(int(taps[j]) * x[:, _reflect101(np.arange(W) + j - n // 2, W)] for j in range(n))
    col = sum(int(taps[i]) * row[_reflect101(np.arange(H) + i - n // 2, H)] for i in range(n))
    return np.minimum(255, (col + (1 << 15)) >> 16).astype(np.uint8)


def add_noise(img, z, sigma):
    """``clip(img + z * sigma, 0, 255)`` in float64, truncated to uint8."""
    return np.clip(img + z * sigma, 0, 255).astype(np.uint8)


def rgb_add_noise(img, rec, z_noise=None, z_final=None):
    """One frame [H,W,3] uint8 through a record; z_noise / z_final: [H,W,3] float64 normals of its noise stages."""
    if rec[A.I_HSV]:
        img = hsv(img, rec[A.I_S_FACTOR], rec[A.I_V_FACTOR])
    if rec[A.I_SHARPEN]:
        img = filter2d(img, rec[A.I_SHARPEN_K:A.I_SHARPEN_K + 9].reshape(3, 3))
    a = int(rec[A.I_MOTION_A])
    if a:
        img = filter2d(img, rec[A.I_MOTION_K:A.I_MOTION_K + a * a].reshape(a, a))
    n = int(rec[A.I_GAUSS_K])
    if n:
        img = gaussian(img, rec[A.I_GAUSS_TAPS:A.I_GAUSS_TAPS + n].astype(np.int64))
    if rec[A.I_NOISE]:
        img = add_noise(img, z_noise, int(rec[A.I_NOISE_SIGMA]))
    if rec[A.I_FINAL]:
        img = add_noise(img, 0.0 + 7.0 * z_final, 1)
    return img


def keep_mask(back_labels, dataset):
    """The background frame's kept pixels: label <= 0 (YCB), mask channel 0 < 255 (LineMOD)."""
    bl = back_labels if back_labels.ndim == 2 else back_labels[..., 0]
    return bl <= 0 if dataset == "ycb" else bl < 255


def add_real_back(rgb, labels, dpt, back_rgb, back_labels, back_dpt, apply_rgb, dataset):
    """One frame: (rgb [H,W,3] uint8, dpt [H,W] uint16) after add_real_back."""
    keep = keep_mask(back_labels, dataset)
    out = rgb.copy()
    if apply_rgb:
        hole = labels <= 0
        out[hole] = np.where(keep[hole][:, None], back_rgb[hole], 0)
    d = np.where(dpt > 0, dpt, np.where(keep, back_dpt, 0)).astype(np.uint16)
    return out, d
