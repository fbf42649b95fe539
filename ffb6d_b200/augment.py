"""Host half of the datasets' synthetic-frame augmentation: the scalar draws of ``rgb_add_noise`` and
``add_real_back`` (datasets/ycb/ycb_dataset.py:79-163, datasets/linemod/linemod_dataset.py:114-186).

Plain numpy, no CUDA and no OpenCV, so a DataLoader worker can import it.  Each function consumes the scalar draws of
``rng`` (the datasets' ``self.rng``, which is ``np.random``) in exactly the reference's order and returns a
fixed-layout float64 *record* that :func:`ffb6d_b200.ops.rgb_add_noise` applies on the GPU.  The record carries the
sharpen 3x3 and motion-blur kernels built as the reference builds them, and the Gaussian blur's fixed-point taps
as OpenCV derives them from sigma.

The per-pixel normal draws (``rng.randn(*img.shape)`` in ``gaussian_noise``, ``np.random.normal`` in YCB's last step)
are NOT drawn here: the device draws them from a counter-based generator keyed by (seed, frame, stage, pixel,
channel).  They have numpy's distribution but not numpy's stream, and the positions of ``rng`` after a frame
therefore differ from the reference's, which would also have consumed 3*H*W normals per noise stage.

:func:`draw_color_jitter` draws the datasets' ``ColorJitter`` (``trancolor``) from torch's generator, as torchvision
does, and returns the plans that :func:`ffb6d_b200.ops.color_jitter` applies on the GPU.
"""
import math

import numpy as np

VERSION = 1
REC_LEN = 1024          # float64 per record
MAX_MOTION = 30         # a = int(max(|cos|,|sin|) * length * 2) with length <= 15

# record layout (float64 slots); include/ffb6d_b200.h FFB6D_AUG_* mirrors it
I_VERSION, I_DATASET, I_PASS = 0, 1, 2
I_HSV, I_S_FACTOR, I_V_FACTOR = 3, 4, 5
I_SHARPEN, I_SHARPEN_K = 6, 7                       # 9 slots: 7..15
I_MOTION_A, I_MOTION_ANGLE, I_MOTION_LEN = 16, 17, 18
I_GAUSS_K, I_GAUSS_SIGMA, I_GAUSS_TAPS = 19, 20, 21  # 5 slots: 21..25, integer taps of weight 1/256
I_NOISE, I_NOISE_SIGMA, I_FINAL = 26, 27, 28
I_MOTION_K = 32                                     # a*a slots, row-major
DATASETS = {"ycb": 0, "linemod": 1}


def identity_record(dataset, pass_=0):
    """A record under which every stage passes the frame through unchanged."""
    rec = np.zeros(REC_LEN, np.float64)
    rec[I_VERSION] = VERSION
    rec[I_DATASET] = DATASETS[dataset]
    rec[I_PASS] = pass_
    return rec


def _clip_line(w, h, x1, y1, x2, y2):
    """OpenCV's ``clipLine`` for integer end points (imgproc/src/drawing.cpp)."""
    right, bottom = w - 1, h - 1

    def code(x, y):
        return (x < 0) + (x > right) * 2 + (y < 0) * 4 + (y > bottom) * 8

    c1, c2 = code(x1, y1), code(x2, y2)
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, (x1, y1, x2, y2)


def _line8(img, p1, p2, value):
    """``cv2.line(img, p1, p2, value)``: thickness 1, 8-connected, integer points (OpenCV's LineIterator, drawn
    left to right)."""
    h, w = img.shape
    x1, y1 = p1
    x2, y2 = p2
    if not (0 <= x1 < w and 0 <= x2 < w and 0 <= y1 < h and 0 <= y2 < h):
        ok, (x1, y1, x2, y2) = _clip_line(w, h, x1, y1, x2, y2)
        if not ok:
            return
    if x2 < x1:
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy, sy = x2 - x1, y2 - y1, 1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
    err, x, y = dx - 2 * dy, x1, y1
    for _ in range(dx + 1):
        img[y, x] = value
        step = err < 0
        err += -2 * dy + (2 * dx if step else 0)
        if vert:
            y += sy
            x += 1 if step else 0
        else:
            x += 1
            y += sy if step else 0


def motion_kernel(angle, length):
    """The kernel of ``linear_motion_blur(img, angle, length)`` (ycb_dataset.py:88-105), or None where the
    reference returns the image unchanged (a <= 0)."""
    rad = np.deg2rad(angle)
    dx, dy = np.cos(rad), np.sin(rad)
    a = int(max(abs(dx), abs(dy)) * length * 2)
    if a <= 0:
        return None
    kern = np.zeros((a, a))
    cx, cy = a // 2, a // 2
    px, py = int(dx * length + cx), int(dy * length + cy)
    _line8(kern, (cx, cy), (px, py), 1.0)
    s = kern.sum()
    if s == 0:
        kern[cx, cy] = 1.0
    else:
        kern /= s
    return kern


def gaussian_taps(n, sigma):
    """The fixed-point taps (integers of weight 1/256, summing to 256) that ``cv2.GaussianBlur`` uses on 8-bit
    images for an n x n kernel (n = 3 or 5) and ``sigmaX = sigmaY = sigma``: OpenCV's bit-exact Gaussian kernel,
    rounded to 8 fractional bits with error diffusion from the outer taps inwards, the centre taking the rest."""
    if sigma <= 0:
        k = {3: [0.25, 0.5], 5: [0.0625, 0.25, 0.375]}[n][: n // 2]
    else:
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            scale = -0.125 / (sigma * sigma)
            vals = [math.exp((x * x) * scale) if np.isfinite(scale) else 0.0 for x in range(1 - n, -1, 2)]
        total = 2.0 * sum(vals) + 1.0 if vals else 1.0
        mul = 1.0 / total
        k = [v * mul for v in vals]
    taps, err, acc = [], 0.0, 0
    for v in k:
        adj = v * 256.0 + err
        v0 = int(np.rint(adj))
        err = adj - v0
        taps.append(v0)
        acc += v0
    taps = taps + [256 - 2 * acc] + taps[::-1]
    return np.array(taps, np.int64)


def draw_rgb_noise(rng, dataset, pass_=0):
    """The scalar draws of ``rgb_add_noise`` (ycb_dataset.py:107-143; linemod_dataset.py:142-164), in the
    reference's order, as a float64 record of length REC_LEN.  ``pass_`` (0 or 1) is the call's position in
    ``get_item``; it keys the device's per-pixel draws so that the two calls of a frame draw independent noise."""
    if dataset not in DATASETS:
        raise ValueError("dataset must be 'ycb' or 'linemod', got %r" % (dataset,))
    ycb = dataset == "ycb"
    rec = identity_record(dataset, pass_)
    if rng.rand() > 0:
        s_lo, s_hi, v_lo, v_hi = (1.25, 1.45, 1.15, 1.35) if ycb else (1 - 0.25, 1 + .25, 1 - .15, 1 + .15)
        rec[I_HSV] = 1
        rec[I_S_FACTOR] = rng.rand() * (s_hi - s_lo) + s_lo
        rec[I_V_FACTOR] = rng.rand() * (v_hi - v_lo) + v_lo
    if ycb and rng.rand() > .8:
        kernel = -np.ones((3, 3))
        kernel[1, 1] = rng.rand() * 3 + 9
        kernel /= kernel.sum()
        rec[I_SHARPEN] = 1
        rec[I_SHARPEN_K:I_SHARPEN_K + 9] = kernel.ravel()
    if rng.rand() > 0.8:
        r_angle = int(rng.rand() * 360)
        r_len = int(rng.rand() * 15) + 1
        kern = motion_kernel(r_angle, r_len)
        rec[I_MOTION_ANGLE], rec[I_MOTION_LEN] = r_angle, r_len
        if kern is not None:
            a = kern.shape[0]
            rec[I_MOTION_A] = a
            rec[I_MOTION_K:I_MOTION_K + a * a] = kern.ravel()
    if rng.rand() > 0.8:
        n = 3 if rng.rand() > 0.2 else 5
        sigma = rng.rand()
        rec[I_GAUSS_K], rec[I_GAUSS_SIGMA] = n, sigma
        rec[I_GAUSS_TAPS:I_GAUSS_TAPS + n] = gaussian_taps(n, sigma)
    if ycb:
        rec[I_NOISE] = 1
        rec[I_NOISE_SIGMA] = rng.randint(15) if rng.rand() > 0.2 else rng.randint(25)
        # (the reference draws rng.randn(H, W, 3) here)
        if rng.rand() > 0.8:
            rec[I_FINAL] = 1          # (and np.random.normal(0, 7, (H, W, 3)) here)
    return rec


JITTER_PLAN_LEN = 8     # include/ffb6d_b200.h FFB6D_JITTER_PLAN_LEN
# torchvision's ColorJitter(0.2, 0.2, 0.2, 0.05) ranges, formed as its _check_input forms them
JITTER_RANGES = ((1 - 0.2, 1 + 0.2), (1 - 0.2, 1 + 0.2), (1 - 0.2, 1 + 0.2), (-0.05, 0.05))


def draw_color_jitter(n, generator=None):
    """The draws of the datasets' ``self.trancolor = transforms.ColorJitter(0.2, 0.2, 0.2, 0.05)``
    (ycb_dataset.py:34, 190-193; linemod_dataset.py:35, 220-223) for ``n`` frames, frame after frame.

    Consumes ``generator`` (default: torch's default CPU generator) exactly as ``ColorJitter.get_params`` does:
    ``randperm(4)``, then four ``torch.empty(1).uniform_(lo, hi)``.  Plain torch on the CPU, no torchvision.

    :return: ``[n, JITTER_PLAN_LEN]`` float64 plans for :func:`ffb6d_b200.ops.color_jitter`: slots 0-3 the order of
      the ops (0 brightness, 1 contrast, 2 saturation, 3 hue), slots 4-7 the brightness, contrast, saturation and hue
      factors as torchvision holds them (float32 draws widened to float64)
    """
    import torch
    plan = np.zeros((int(n), JITTER_PLAN_LEN), np.float64)
    for i in range(int(n)):
        plan[i, :4] = torch.randperm(4, generator=generator).numpy()
        for k, (lo, hi) in enumerate(JITTER_RANGES):
            plan[i, 4 + k] = float(torch.empty(1).uniform_(lo, hi, generator=generator))
    return plan


def draw_frame_augmentation(rng, dataset, n_real, rnd_typ="syn"):
    """The scalar draws of ``get_item``'s augmentation block for one synthetic frame, in the reference's order
    (ycb_dataset.py:198-202; linemod_dataset.py:242-249).

    :param n_real: length of the dataset's ``real_lst`` (``real_gen`` draws the background frame from it)
    :param rnd_typ: LineMOD only: ``'render'`` or ``'fuse'`` (a fused frame is augmented with probability 0.8)
    :return: dict with ``plans`` ([2, REC_LEN] float64: the first and second ``rgb_add_noise``, an identity record
      where the reference skips the call), ``augment`` (False where nothing is applied), ``back_index`` (the
      ``real_lst`` index of the background frame, or -1) and ``apply_rgb`` (whether ``add_real_back`` composes the
      colour image; it always composes the depth)
    """
    if dataset not in DATASETS:
        raise ValueError("dataset must be 'ycb' or 'linemod', got %r" % (dataset,))
    plans = np.stack([identity_record(dataset, 0), identity_record(dataset, 1)])
    out = dict(plans=plans, augment=False, back_index=-1, apply_rgb=False)
    if dataset == "linemod":
        if rnd_typ not in ("render", "fuse"):
            raise ValueError("rnd_typ must be 'render' or 'fuse', got %r" % (rnd_typ,))
        if not (rnd_typ == "render" or rng.rand() < 0.8):
            return out
    plans[0] = draw_rgb_noise(rng, dataset, 0)
    out["back_index"] = int(rng.randint(0, n_real))
    out["apply_rgb"] = True if dataset == "ycb" else bool(rng.rand() < 0.6)
    if rng.rand() > 0.8:
        plans[1] = draw_rgb_noise(rng, dataset, 1)
    out["augment"] = True
    return out
