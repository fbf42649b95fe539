#!/usr/bin/env python
"""Generate tests/golden/jitter_cases.npz by running torchvision's colour jitter on PIL images in this container.

Source of truth: ``torchvision.transforms.ColorJitter(0.2, 0.2, 0.2, 0.05)`` as the datasets hold it
(datasets/ycb/ycb_dataset.py:34, 190-193; datasets/linemod/linemod_dataset.py:35, 220-223) and its
``F.adjust_brightness / adjust_contrast / adjust_saturation / adjust_hue`` on PIL images, with the installed
torchvision 0.26 and Pillow 12.2 (the versions the restatement is pinned to).

Every case is a plan ([8] float64: the order of the four ops, then the brightness, contrast, saturation and hue
factors) applied to one frame: the four ``F.adjust_*`` calls in the plan's order, which is the body of
``ColorJitter.forward``.  An op is tested alone by setting the other blend factors to 1.0 (Image.blend with factor 1.0
returns its second image) and running the hue op first with factor 0.0 (its HSV round trip is not the identity, so
it cannot be switched off).  Inputs are ``ffb6d_b200.synthetic.make_aug_frame`` frames, regenerated from
``meta = (seed, h, w)``, or stored as ``rgb`` where they are tiny or hand-made.  Outputs are stored as ``out`` (a
sha256 for the 480x640 case).

Also stored: whole ``ColorJitter`` calls under ``torch.manual_seed`` with the plans ``get_params`` drew for them
(``seed_*``), runs of ``get_params`` over several frames (``draws_*``), and RGBA inputs whose first three bands the
transform must leave as it leaves the RGB input (``rgba_*``, the alpha in ``alpha``).

Run:  python tests/golden/make_jitter_golden.py      (needs torchvision and Pillow; rewrites jitter_cases.npz)
"""
import hashlib
import io
import itertools
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ffb6d_b200.synthetic import make_aug_frame                     # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "jitter_cases.npz")
B_, C_, S_, H_ = 0, 1, 2, 3


def plan(order, b=1.0, c=1.0, s=1.0, h=0.0):
    return np.array(list(order) + [b, c, s, h], np.float64)


def alone(op, factor):
    """The blend op `op` alone after a hue round trip; hue alone with neutral blends."""
    if op == H_:
        return plan((B_, C_, S_, H_), h=factor)
    f = [1.0, 1.0, 1.0]
    f[op] = factor
    return plan([H_, op] + [o for o in (B_, C_, S_) if o != op], *f, h=0.0)


def apply_plan(img, p):
    """The body of ColorJitter.forward with the plan's draws, on a PIL image."""
    import torchvision.transforms.functional as TF
    fns = (TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue)
    for op in p[:4].astype(int):
        img = fns[op](img, float(p[4 + op]))
    return img


def run(rgb, p, mode="RGB", alpha=None):
    from PIL import Image
    a = rgb if alpha is None else np.concatenate([rgb, alpha[..., None]], -1)
    out = np.asarray(apply_plan(Image.fromarray(np.ascontiguousarray(a), mode), p))
    return np.ascontiguousarray(out[..., :3])


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def special_pixels():
    """Saturated, grey, black, white and near-extreme pixels, one row."""
    v = [0, 1, 127, 128, 254, 255]
    px = [(r, g, b) for r in v for g in v for b in v]
    return np.array(px, np.uint8).reshape(1, -1, 3)


def half_mean_frame(h, w, seed, grey):
    """A frame whose mean of L is k + 0.5 exactly (h * w even): the contrast mean rounds up on the boundary."""
    rs = np.random.RandomState(seed)
    if grey:
        x = np.repeat(rs.randint(0, 255, (h, w))[..., None], 3, -1).astype(np.uint8)
    else:
        x = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    n = h * w
    for v in range(256):                             # pixel 0 grey (L = v) tunes the sum to n/2 mod n
        x[0, 0] = v
        a = x.astype(np.int64)
        if ((19595 * a[..., 0] + 38470 * a[..., 1] + 7471 * a[..., 2] + 0x8000) >> 16).sum() % n == n // 2:
            return x
    raise AssertionError("no grey value puts the mean on .5")


def cases():
    import torch
    import torchvision.transforms as T
    c = {}
    # each op alone: both ends of its range, in between, and the neutral factor; extrapolation beyond the range too
    for op, name in ((B_, "brightness"), (C_, "contrast"), (S_, "saturation")):
        for f in (0.0, 0.5, 0.8, 0.9137, 1.0, 1.0731, 1.2, 1.9):
            c["alone_%s_%g" % (name, f)] = (dict(meta=(100 + op, 24, 32)), alone(op, f))
    for f in (-0.05, -0.0213, 0.0, 0.0371, 0.05, -0.5, 0.5):
        c["alone_hue_%g" % f] = (dict(meta=(104, 24, 32)), alone(H_, f))
    # every hue shift from -12 to 12 (int32(hue * 255) truncates toward zero), and |hue| just around 1/255
    for s in range(-12, 13):
        hue = 0.0 if s == 0 else (s + 0.5 * np.sign(s)) / 255.0
        c["shift_%+03d" % s] = (dict(meta=(200 + s, 16, 20)), alone(H_, hue))
    for k, hue in enumerate((1 / 255 * (1 - 1e-9), 1 / 255 * (1 + 1e-9), -1 / 255 * (1 - 1e-9), -1 / 255 * (1 + 1e-9))):
        c["shift_near_one_%d" % k] = (dict(meta=(230 + k, 16, 20)), alone(H_, hue))
    # all 24 orders
    for k, order in enumerate(itertools.permutations(range(4))):
        c["order_%s" % "".join(map(str, order))] = (dict(meta=(300 + k, 20, 28)), plan(order, 1.13, 0.87, 1.19, -0.037))
    # contrast on a constant frame and with the mean of L on a .5 boundary (contrast first, and after the round trip)
    const = np.empty((6, 7, 3), np.uint8)
    const[:] = (200, 30, 90)
    for f in (0.8, 1.2):
        c["contrast_const_%g" % f] = (dict(rgb=const), plan((C_, B_, S_, H_), c=f))
    for k, (grey, order) in enumerate(((True, (C_, B_, S_, H_)), (False, (C_, B_, S_, H_)), (True, (H_, C_, B_, S_)))):
        for f in (0.8, 1.2):
            c["contrast_half_%d_%g" % (k, f)] = (dict(rgb=half_mean_frame(6, 8, 400 + k, grey)), plan(order, c=f))
    # saturated, grey, black and white pixels
    sp = special_pixels()
    for k, order in enumerate(((0, 1, 2, 3), (3, 2, 1, 0), (2, 3, 0, 1))):
        for f, hue in ((0.8, -0.05), (1.2, 0.05)):
            c["special_%d_%g" % (k, f)] = (dict(rgb=sp), plan(order, f, 2.0 - f, f, hue))
    # sizes: 1x1, a row, a column, odd H and W
    rs = np.random.RandomState(500)
    for h, w in ((1, 1), (1, 13), (13, 1), (7, 5), (33, 47)):
        x = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        c["size_%dx%d" % (h, w)] = (dict(rgb=x), plan(rs.permutation(4), 1.17, 0.83, 1.08, 0.042))
    # whole ColorJitter calls under torch.manual_seed, with the plans get_params drew; one at 480x640
    cj = T.ColorJitter(0.2, 0.2, 0.2, 0.05)
    extra = {}
    for seed, (h, w) in ((0, (24, 32)), (1, (24, 32)), (7, (40, 48)), (42, (33, 47)), (1234, (480, 640))):
        torch.manual_seed(seed)
        fn_idx, b, co, s, hu = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        p = plan(fn_idx.tolist(), b, co, s, hu)
        fr = make_aug_frame(600 + seed, h, w)["rgb"]
        from PIL import Image
        torch.manual_seed(seed)
        whole = np.asarray(cj(Image.fromarray(fr)))
        assert np.array_equal(whole, run(fr, p)), seed
        c["seed_%d" % seed] = (dict(meta=(600 + seed, h, w)), p)
        extra["seed_%d/torch_seed" % seed] = np.array(seed)
    # get_params over several frames: the plans draw_color_jitter must reproduce
    for seed in (0, 3, 2024):
        torch.manual_seed(seed)
        ps = []
        for _ in range(6):
            fn_idx, b, co, s, hu = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
            ps.append(plan(fn_idx.tolist(), b, co, s, hu))
        extra["draws_%d/plans" % seed] = np.stack(ps)
        extra["draws_%d/torch_seed" % seed] = np.array(seed)
    # RGBA: the first three bands equal those of the RGB input, over several seeds
    for seed in range(6):
        torch.manual_seed(50 + seed)
        fn_idx, b, co, s, hu = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        p = plan(fn_idx.tolist(), b, co, s, hu)
        fr = make_aug_frame(700 + seed, 20, 24)["rgb"]
        alpha = np.random.RandomState(700 + seed).randint(0, 256, fr.shape[:2]).astype(np.uint8)
        alpha[0, 0], alpha[0, 1] = 0, 255
        out4 = run(fr, p, "RGBA", alpha)
        assert np.array_equal(out4, run(fr, p)), seed
        c["rgba_%d" % seed] = (dict(meta=(700 + seed, 20, 24), alpha=alpha), p)

    data = dict(extra)
    for name, (inp, p) in sorted(c.items()):
        if "rgb" in inp:
            rgb = inp["rgb"]
            data[name + "/rgb"] = rgb
        else:
            seed, h, w = inp["meta"]
            rgb = make_aug_frame(seed, h, w)["rgb"]
            data[name + "/meta"] = np.array(inp["meta"])
        data[name + "/plan"] = p
        if "alpha" in inp:
            data[name + "/alpha"] = inp["alpha"]
            out = run(rgb, p, "RGBA", inp["alpha"])
        else:
            out = run(rgb, p)
        if out.size >= 480 * 640 * 3:
            data[name + "/sha256_out"] = np.array(sha(out))
        else:
            data[name + "/out"] = out
    return data


def main():
    data = cases()
    # fixed member order and timestamps, so the file is reproducible byte for byte
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(data):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(data[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
