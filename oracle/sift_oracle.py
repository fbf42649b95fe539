"""numpy restatement of OpenCV's SIFT keypoint detector at ``cv2.SIFT_create()``'s defaults (nfeatures 0, 3 octave
layers, contrast 0.04, edge 10, sigma 1.6), DESIGN.md §4.33.  Keypoints only: the reference's textured keypoint tool
reads ``kp.pt`` and nothing else, so descriptors are not restated.

Each step is its own function so that each can be pinned to cv2 on its own (tests/golden/check_sift_opencv.py):

  grey            ORB's 15-bit BGR2GRAY (oracle/orb_oracle.py), as float32
  upscale         the 2x INTER_LINEAR resize of the grey image (weights 3/4 and 1/4, clamped at the edges; exact)
  gaussian_taps   getGaussianKernel(ks, sigma, CV_32F), ks = cvRound(8 sigma + 1) | 1, in its bit-exact form
  blur            the separable float32 GaussianBlur, BORDER_REFLECT_101: a row pass ``acc = k0 s[-r]``, then
                  ``acc = fma(k_j, s[j - r], acc)`` in tap order, and a column pass ``acc = k_r s[0]``, then
                  ``acc = fma(k_{r+j}, s[-j] + s[j], acc)``; the last ``W mod 8`` columns take OpenCV's narrower
                  paths: 4 columns with an fma row pass and a plain column pass (when 4 or more remain), then the
                  rest with plain passes (``acc + k s``, two roundings)
  octave_sizes    ``cvRound(log2(min side of the upscaled image) - 2) + 1`` octaves, each halving the last
                  (integer division); 6 Gaussian layers with buildGaussianPyramid's incremental sigmas; an octave's
                  base is the previous octave's layer 3 at even pixels; DoG is a float32 subtract
  extrema         ``|v| > 1`` (``floor(0.5 0.04 / 3 255)``) and ``v >=`` (``<=`` for negative v) each of its 26
                  neighbours, 5 pixels from every edge, DoG layers 1..3
  refine          adjustLocalExtrema: at most 5 Newton steps, the 3x3 solve by Cramer's rule in float32
                  (``Matx33f::solve``'s fast path), contrast and edge tests, with the fused multiply-adds OpenCV's
                  build contracts them into (``_fms``, ``solve3``)
  orientations    calcOrientationHist and its peaks: weights by ``exp32``, angles by ``atan32``, magnitudes by
                  ``mag32``, 36 bins accumulated in pixel order, the 5-tap smoothing, then every strict local peak
                  ``>= 0.8 max`` with a parabolic fit
  dedup           removeDuplicatedSorted: of keypoints with equal ``pt``, ``size`` and ``angle``, the one of
                  larger response, then larger packed octave, is kept

``exp32``, ``atan32`` and ``mag32`` are specified here; OpenCV 4.13's ``hal`` versions differ from them in the
last bits (DESIGN.md §4.33 gives the measured counts), so angles agree with OpenCV's to ~1e-4 degrees, not bitwise.

Output order is canonical: octave, DoG layer where the extremum was found, raster order, then peaks in histogram
order.  OpenCV's order comes from ``parallel_for_`` and a sort and is not a contract.
"""
import math

import numpy as np

from oracle.aug_oracle import fma32
from oracle.orb_oracle import grey as _grey8

f32, f64 = np.float32, np.float64

N_LAYERS = 3
SIGMA = 1.6
CONTRAST = f32(0.04)
EDGE = f32(10.0)
BORDER = 5
MAX_STEPS = 5
N_BINS = 36
THRESHOLD = math.floor(0.5 * 0.04 / N_LAYERS * 255)      # = 1
MAX_COPIES = N_BINS // 2                                  # strict peaks of 36 circular bins
HIST_LANES = 16                                           # calcOrientationHist's vector width (AVX-512)


def cv_round(x):
    """cvRound: round half to even."""
    return int(np.rint(x))


def grey(rgb):
    """Float32 grey of an RGB uint8 image ``[H,W,3]`` (the tool passes BGR; this takes the channels by name)."""
    return _grey8(rgb).astype(f32)


def _up_taps(n):
    d = np.arange(2 * n)
    s = np.where(d % 2 == 0, d // 2 - 1, d // 2)
    a1 = np.where(d % 2 == 0, f32(0.75), f32(0.25)).astype(f32)
    a1 = np.where((s < 0) | (s >= n - 1), f32(0), a1).astype(f32)
    return np.clip(s, 0, n - 1), np.clip(s + 1, 0, n - 1), (f32(1) - a1).astype(f32), a1


def upscale(g):
    """The 2x INTER_LINEAR resize of a float32 grey image ``[h,w]`` (integers in, multiples of 1/16 out: exact)."""
    h, w = g.shape
    x0, x1, wx0, wx1 = _up_taps(w)
    y0, y1, wy0, wy1 = _up_taps(h)
    r = g[:, x0] * wx0 + g[:, x1] * wx1
    return (r[y0] * wy0[:, None] + r[y1] * wy1[:, None]).astype(f32)


def base_sigma():
    """createInitialImage's blur: ``sqrtf(max(1.6f^2 - 4 0.5^2, 0.01f))`` as a double."""
    s = f32(SIGMA)
    return float(np.sqrt(np.maximum(s * s - f32(0.5) * f32(0.5) * f32(4), f32(0.01))))


def layer_sigmas():
    """buildGaussianPyramid's incremental sigmas of layers 1..5 (float64)."""
    k = math.pow(2.0, 1.0 / N_LAYERS)
    out = []
    for i in range(1, N_LAYERS + 3):
        prev = math.pow(k, i - 1) * SIGMA
        tot = prev * k
        out.append(math.sqrt(tot * tot - prev * prev))
    return out


def gaussian_taps(sigma):
    """getGaussianKernel(ks, sigma, CV_32F) with ks = cvRound(8 sigma + 1) | 1 (its bit-exact double form)."""
    n = cv_round(sigma * 8 + 1) | 1
    sc = -0.125 / (sigma * sigma)
    vals = [math.exp(float(x * x) * sc) for x in range(1 - n, 0, 2)]
    s = 0.0
    for v in vals:
        s += v
    mul = 1.0 / (s * 2 + 1.0)
    half = [v * mul for v in vals]
    return np.array(half + [mul] + half[::-1]).astype(f32)


def _reflect101(i, n):
    i = np.asarray(i)
    if n == 1:
        return np.zeros_like(i)
    while np.any((i < 0) | (i >= n)):
        i = np.where(i < 0, -i, i)
        i = np.where(i >= n, 2 * n - 2 - i, i)
    return i


def column_modes(w):
    """Per column: 0 fma row and column passes, 1 fma row pass and plain column pass, 2 plain passes."""
    m = np.zeros(w, np.int64)
    v = w // 8 * 8
    m[v:] = 2
    if w - v >= 4:
        m[v:v + 4] = 1
    return m


def blur(img, k):
    """GaussianBlur of a float32 image ``[h,w]`` with taps ``k``."""
    h, w = img.shape
    r = len(k) // 2
    x, y = np.arange(w), np.arange(h)
    m = column_modes(w)
    rf, cf = m <= 1, m == 0
    acc = img[:, _reflect101(x - r, w)] * k[0]
    for j in range(1, len(k)):
        s = img[:, _reflect101(x + j - r, w)]
        acc = np.where(rf, fma32(k[j], s, acc), (acc + k[j] * s).astype(f32))
    t = acc.astype(f32)
    acc = t * k[r]
    for j in range(1, r + 1):
        s = (t[_reflect101(y - j, h)] + t[_reflect101(y + j, h)]).astype(f32)
        acc = np.where(cf, fma32(k[r + j], s, acc), (acc + k[r + j] * s).astype(f32))
    return acc.astype(f32)


def n_octaves(H, W):
    """Octave count of an H x W input: ``cvRound(log(min(2H, 2W)) / log(2) - 2) + 1``."""
    return cv_round(math.log(float(min(2 * H, 2 * W))) / math.log(2.0) - 2) + 1


def octave_sizes(H, W):
    """``[(h_o, w_o)]`` of the octaves (octave 0 is the upscaled image)."""
    h, w = 2 * H, 2 * W
    out = []
    for _ in range(n_octaves(H, W)):
        out.append((h, w))
        h, w = h // 2, w // 2
    return out


def pyramids(rgb):
    """Gaussian (6 layers) and DoG (5 layers) images of every octave of an RGB uint8 image: two lists of
    ``[layers, h_o, w_o]`` float32 arrays."""
    H, W = rgb.shape[:2]
    g = blur(upscale(grey(rgb)), gaussian_taps(base_sigma()))
    taps = [gaussian_taps(s) for s in layer_sigmas()]
    gauss, dog = [], []
    for o, (h, w) in enumerate(octave_sizes(H, W)):
        if o:
            g = gauss[-1][N_LAYERS][::2, ::2][:h, :w]
        layers = [g]
        for k in taps:
            layers.append(blur(layers[-1], k))
        L = np.stack(layers)
        gauss.append(L)
        dog.append((L[1:] - L[:-1]).astype(f32))
    return gauss, dog


def extrema(D):
    """Candidates of one octave's DoG ``[5,h,w]``: ``(layer, r, c)`` arrays in layer then raster order."""
    out = []
    _, h, w = D.shape
    for i in range(1, N_LAYERS + 1):
        if h <= 2 * BORDER or w <= 2 * BORDER:
            continue
        v = D[i, BORDER:h - BORDER, BORDER:w - BORDER]
        mx = np.full(v.shape, -np.inf, f32)
        mn = np.full(v.shape, np.inf, f32)
        for l in (i - 1, i, i + 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if l == i and dy == 0 and dx == 0:
                        continue
                    n = D[l, BORDER + dy:h - BORDER + dy, BORDER + dx:w - BORDER + dx]
                    mx = np.maximum(mx, n)
                    mn = np.minimum(mn, n)
        keep = (np.abs(v) > THRESHOLD) & (((v > 0) & (v >= mx)) | ((v < 0) & (v <= mn)))
        rs, cs = np.nonzero(keep)
        out.append((np.full(len(rs), i), rs + BORDER, cs + BORDER))
    if not out:
        return np.zeros(0, int), np.zeros(0, int), np.zeros(0, int)
    return tuple(np.concatenate(a) for a in zip(*out))


def _fms(a, b, c, d):
    """``a b - c d`` as the compiler contracts it: ``fma(a, b, -(c d))``."""
    return fma32(a, b, -(f32(c) * f32(d)))


def solve3(H, b):
    """Matx33f::solve(b, DECOMP_LU)'s fast path: Cramer's rule in float32 with OpenCV's build's contractions (each
    ``p q - r s`` is ``fma(p, q, -(r s))``, each ``u v - w x + y z`` is ``fma(y, z, fma(u, v, -(w x)))``); 0 when the
    determinant is 0."""
    a = [[f32(v) for v in row] for row in H]
    b0, b1, b2 = (f32(v) for v in b)

    def cof3(u, p, w, q, y, r):
        return fma32(y, r, fma32(u, p, -(w * q)))
    det = cof3(a[0][0], _fms(a[1][1], a[2][2], a[2][1], a[1][2]), a[0][1], _fms(a[1][0], a[2][2], a[2][0], a[1][2]),
               a[0][2], _fms(a[1][0], a[2][1], a[2][0], a[1][1]))
    if det == 0:
        return f32(0), f32(0), f32(0)
    d = f32(1) / det
    x0 = d * cof3(b0, _fms(a[1][1], a[2][2], a[1][2], a[2][1]), a[0][1], _fms(b1, a[2][2], a[1][2], b2),
                  a[0][2], _fms(b1, a[2][1], a[1][1], b2))
    x1 = d * cof3(a[0][0], _fms(b1, a[2][2], a[1][2], b2), b0, _fms(a[1][0], a[2][2], a[1][2], a[2][0]),
                  a[0][2], _fms(a[1][0], b2, b1, a[2][0]))
    x2 = d * cof3(a[0][0], _fms(a[1][1], b2, b1, a[2][1]), a[0][1], _fms(a[1][0], b2, b1, a[2][0]),
                  b0, _fms(a[1][0], a[2][1], a[1][1], a[2][0]))
    return f32(x0), f32(x1), f32(x2)


IMG_SCALE = f32(1) / f32(255)
DERIV_SCALE = IMG_SCALE * f32(0.5)
CROSS_SCALE = IMG_SCALE * f32(0.25)


def _derivs(D, layer, r, c):
    img, prv, nxt = D[layer], D[layer - 1], D[layer + 1]
    dD = ((img[r, c + 1] - img[r, c - 1]) * DERIV_SCALE, (img[r + 1, c] - img[r - 1, c]) * DERIV_SCALE,
          (nxt[r, c] - prv[r, c]) * DERIV_SCALE)
    v2 = img[r, c] * f32(2)
    dxx = (img[r, c + 1] + img[r, c - 1] - v2) * IMG_SCALE
    dyy = (img[r + 1, c] + img[r - 1, c] - v2) * IMG_SCALE
    dss = (nxt[r, c] + prv[r, c] - v2) * IMG_SCALE
    dxy = (img[r + 1, c + 1] - img[r + 1, c - 1] - img[r - 1, c + 1] + img[r - 1, c - 1]) * CROSS_SCALE
    dxs = (nxt[r, c + 1] - nxt[r, c - 1] - prv[r, c + 1] + prv[r, c - 1]) * CROSS_SCALE
    dys = (nxt[r + 1, c] - nxt[r - 1, c] - prv[r + 1, c] + prv[r - 1, c]) * CROSS_SCALE
    return dD, dxx, dyy, dss, dxy, dxs, dys


def refine(D, o, layer, r, c):
    """adjustLocalExtrema of a candidate of octave o: None when rejected, else a dict of the final ``layer``, ``r``,
    ``c``, the offsets ``xc, xr, xi`` and the keypoint's ``pt`` (x, y), packed ``octave``, ``size`` and
    ``response`` in the input image's coordinates (firstOctave = -1 undone)."""
    _, h, w = D.shape
    xi = xr = xc = f32(0)
    i = 0
    while i < MAX_STEPS:
        dD, dxx, dyy, dss, dxy, dxs, dys = _derivs(D, layer, r, c)
        X = solve3(((dxx, dxy, dxs), (dxy, dyy, dys), (dxs, dys, dss)), dD)
        xi, xr, xc = -X[2], -X[1], -X[0]
        if abs(xi) < f32(0.5) and abs(xr) < f32(0.5) and abs(xc) < f32(0.5):
            break
        big = f32(2147483647 // 3)
        if abs(xi) > big or abs(xr) > big or abs(xc) > big:
            return None
        c += cv_round(xc)
        r += cv_round(xr)
        layer += cv_round(xi)
        if layer < 1 or layer > N_LAYERS or c < BORDER or c >= w - BORDER or r < BORDER or r >= h - BORDER:
            return None
        i += 1
    if i >= MAX_STEPS:
        return None
    dD, dxx, dyy, _, dxy, _, _ = _derivs(D, layer, r, c)
    t = fma32(dD[2], xi, fma32(dD[1], xr, dD[0] * xc))
    contr = fma32(D[layer][r, c], IMG_SCALE, t * f32(0.5))
    if abs(contr) * f32(N_LAYERS) < CONTRAST:
        return None
    tr = dxx + dyy
    det = _fms(dxx, dyy, dxy, dxy)
    if det <= 0 or tr * tr * EDGE >= (EDGE + f32(1)) * (EDGE + f32(1)) * det:
        return None
    sc = f32(1 << o) * f32(0.5)
    q = cv_round((float(xi) + 0.5) * 255)
    packed = (o + (layer << 8) + (q << 16)) & ~255 | ((o - 1) & 255)
    size = f32(SIGMA) * _pow2(f32(f32(layer) + xi) / f32(N_LAYERS)) * f32(1 << o) * f32(2)
    return dict(layer=layer, r=r, c=c, xc=xc, xr=xr, xi=xi,
                pt=(f32(f32(c) + xc) * sc, f32(f32(r) + xr) * sc), octave=packed,
                size=f32(size * f32(0.5)), response=f32(abs(contr)), scl=f32(size * f32(0.5) / f32(1 << o)))


def _pow2(x):
    """powf(2, x) as a correctly rounded float32 (through float64 exp2)."""
    return f32(np.exp2(f64(x)))


# ---------------------------------------------------------------------------------- the orientation histogram's math

_A0 = .9670371139572337719125840413672004409288e-2
EXP_TAB = np.array([math.pow(2.0, i / 64.0) * _A0 for i in range(64)]).astype(f32)
EXP_A4 = f32(1.000000000000002438532970795181890933776 / _A0)
EXP_A3 = f32(.6931471805521448196800669615864773144641 / _A0)
EXP_A2 = f32(.2402265109513301490103372422686535526573 / _A0)
EXP_A1 = f32(.5550339366753125211915322047004666939128e-1 / _A0)
EXP_PRE = f32(1.4426950408889634073599246810019 * 64)
EXP_POST = f32(1.0 / 64)
EXP_MAX = f32(3000.0)


def exp32(x):
    """exp of float32 x: OpenCV's classic table-and-polynomial exp32f in its vector form (64-entry table of
    ``2^(i/64)``, a degree-4 polynomial by fma)."""
    x = np.clip(np.asarray(x, f32), -EXP_MAX, EXP_MAX) * EXP_PRE
    xi = np.rint(x).astype(np.int64)
    x = ((x - xi.astype(f32)) * EXP_POST).astype(f32)
    t = np.clip((xi >> 6) + 127, 0, 255)
    y = EXP_TAB[xi & 63] * (t << 23).astype(np.uint32).view(f32)
    z = fma32(fma32(fma32(x + EXP_A1, x, EXP_A2), x, EXP_A3), x, EXP_A4)
    return (z * y).astype(f32)


ATAN_P1 = f32(0.9997878412794807 * (180 / math.pi))
ATAN_P3 = f32(-0.3258083974640975 * (180 / math.pi))
ATAN_P5 = f32(0.1555786518463281 * (180 / math.pi))
ATAN_P7 = f32(-0.04432655554792128 * (180 / math.pi))
ATAN_EPS = f32(np.finfo(np.float64).eps)


def atan32(y, x):
    """fastAtan2(y, x) in degrees, [0, 360): OpenCV's degree-7 polynomial in its vector form."""
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    ax, ay = np.abs(x), np.abs(y)
    c = (np.minimum(ax, ay) / (np.maximum(ax, ay) + ATAN_EPS)).astype(f32)
    cc = c * c
    a = (fma32(fma32(fma32(cc, ATAN_P7, ATAN_P5), cc, ATAN_P3), cc, ATAN_P1) * c).astype(f32)
    a = np.where(ax >= ay, a, f32(90) - a)
    a = np.where(x < 0, f32(180) - a, a)
    return np.where(y < 0, f32(360) - a, a).astype(f32)


def mag32(x, y):
    """Gradient magnitude ``sqrt(fma(x, x, y y))``."""
    x, y = np.asarray(x, f32), np.asarray(y, f32)
    return np.sqrt(fma32(x, x, (y * y).astype(f32))).astype(f32)


def orientation_hist(img, r0, c0, radius, sigma):
    """calcOrientationHist of the Gaussian layer ``img`` around (r0, c0): the 36 smoothed bins (float32)."""
    h, w = img.shape
    ii, jj, dxs, dys = [], [], [], []
    for i in range(-radius, radius + 1):
        y = r0 + i
        if y <= 0 or y >= h - 1:
            continue
        for j in range(-radius, radius + 1):
            x = c0 + j
            if x <= 0 or x >= w - 1:
                continue
            ii.append(i)
            jj.append(j)
    ii, jj = np.array(ii), np.array(jj)
    ys, xs = r0 + ii, c0 + jj
    dx = (img[ys, xs + 1] - img[ys, xs - 1]).astype(f32)
    dy = (img[ys - 1, xs] - img[ys + 1, xs]).astype(f32)
    expf_scale = f32(-1) / (f32(2) * sigma * sigma)
    W = exp32((ii * ii + jj * jj).astype(f32) * expf_scale)
    ori = atan32(dy, dx)
    mag = mag32(dx, dy)
    b = np.rint(f32(N_BINS / 360.0) * ori).astype(np.int64)
    b = np.where(b >= N_BINS, b - N_BINS, b)
    b = np.where(b < 0, b + N_BINS, b)
    n = len(ii)
    vec = n // HIST_LANES * HIST_LANES
    wm = (W * mag).astype(f32)
    hist = np.zeros(N_BINS, f32)
    for k in range(n):
        if k < vec:
            hist[b[k]] = hist[b[k]] + wm[k]
        else:
            hist[b[k]] = fma32(W[k], mag[k], hist[b[k]])
    t = np.concatenate([hist[-2:], hist, hist[:2]])
    out = np.empty(N_BINS, f32)
    for i in range(N_BINS):
        a = (t[i] + t[i + 4]).astype(f32)
        bb = (t[i + 1] + t[i + 3]).astype(f32)
        if i < N_BINS // HIST_LANES * HIST_LANES:
            out[i] = fma32(a, f32(1 / 16), fma32(bb, f32(4 / 16), t[i + 2] * f32(6 / 16)))
        else:
            out[i] = fma32(t[i + 2], f32(6 / 16), (a * f32(1 / 16) + bb * f32(4 / 16)).astype(f32))
    return out


def peaks(hist):
    """The histogram's orientations: angles (float32 degrees) of every strict local peak >= 0.8 max, in bin order."""
    thr = f32(hist.max() * f32(0.8))
    out = []
    for j in range(N_BINS):
        l, r = (j - 1) % N_BINS, (j + 1) % N_BINS
        if hist[j] > hist[l] and hist[j] > hist[r] and hist[j] >= thr:
            b = f32(j) + f32(0.5) * (hist[l] - hist[r]) / (hist[l] - f32(2) * hist[j] + hist[r])
            b = b + f32(N_BINS) if b < 0 else (b - f32(N_BINS) if b >= N_BINS else b)
            a = f32(360) - f32(f32(10) * f32(b))
            if abs(a - f32(360)) < np.finfo(f32).eps:
                a = f32(0)
            out.append(f32(a))
    return out


def dedup(kps):
    """removeDuplicatedSorted as a mask: keypoint i is dropped when another has equal (pt, size, angle) and a
    larger (response, octave), or equal ones and a smaller index."""
    key = {}
    keep = np.ones(len(kps), bool)
    for i, k in enumerate(kps):
        kk = (np.float32(k["pt"][0]).view(np.uint32).item(), np.float32(k["pt"][1]).view(np.uint32).item(),
              np.float32(k["size"]).view(np.uint32).item(), np.float32(k["angle"]).view(np.uint32).item())
        rank = (float(k["response"]), int(k["octave"]))
        if kk in key:
            j = key[kk]
            if rank > (float(kps[j]["response"]), int(kps[j]["octave"])):
                keep[j] = False
                key[kk] = i
            else:
                keep[i] = False
        else:
            key[kk] = i
    return keep


def detect(rgb):
    """SIFT keypoints of one RGB uint8 image ``[H,W,3]``: dict of ``pt [n,2]`` float32 (x, y), ``octave [n]``
    int32 (OpenCV's packing), ``size [n]``, ``angle [n]`` and ``response [n]`` float32, in canonical order."""
    gauss, dog = pyramids(rgb)
    kps = []
    for o, D in enumerate(dog):
        for layer, r, c in zip(*extrema(D)):
            k = refine(D, o, int(layer), int(r), int(c))
            if k is None:
                continue
            img = gauss[o][k["layer"]]
            hist = orientation_hist(img, k["r"], k["c"], cv_round(f32(4.5) * k["scl"]), f32(1.5) * k["scl"])
            for a in peaks(hist):
                kps.append(dict(k, angle=a))
    keep = dedup(kps)
    kps = [k for k, f in zip(kps, keep) if f]
    return dict(pt=np.array([k["pt"] for k in kps], f32).reshape(-1, 2),
                octave=np.array([k["octave"] for k in kps], np.int64).astype(np.int32),
                size=np.array([k["size"] for k in kps], f32), angle=np.array([k["angle"] for k in kps], f32),
                response=np.array([k["response"] for k in kps], f32))
