#!/usr/bin/env python
"""Generate tests/golden/aug_cases.npz by running THE REFERENCE'S OWN augmentation code in this container.

Source of truth: ``rand_range``, ``gaussian_noise``, ``linear_motion_blur``, ``rgb_add_noise`` and ``add_real_back`` of
both datasets (datasets/ycb/ycb_dataset.py:79-163, datasets/linemod/linemod_dataset.py:114-186), executed from the
reference's source text with OpenCV (the dataset modules import normalSpeed, so the methods are taken out of the files
with ``ast``).  ``self.rng`` is a replay RNG that returns scripted scalars and serves ``randn`` / ``np.random.normal``
from given float64 fields; ``Image.open`` hands out the synthetic background frame.  The inputs are
``ffb6d_b200.synthetic.make_aug_frame`` frames; the tests regenerate them from their seeds.

Stored per case: the record that ``ffb6d_b200.augment`` draws from the same scalars, the normal fields (seeded numpy
draws) where a noise stage has a nonzero sigma, and the reference's outputs (a sha256 for the 480x640 case).  Also
stored: the reference's sequence of ``rng`` calls for whole frames of both datasets at several seeds.

Run:  python tests/golden/make_aug_golden.py      (needs /root/reference; rewrites aug_cases.npz)
"""
import hashlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader as R                                  # noqa: E402
from ffb6d_b200 import augment as A                                 # noqa: E402
from ffb6d_b200.synthetic import make_aug_frame                     # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "aug_cases.npz")
METHODS = ["rand_range", "gaussian_noise", "linear_motion_blur", "rgb_add_noise", "add_real_back"]
N_REAL = 7


class ScriptRNG:
    """Serves scripted rand() / randint() values; randn / normal from fields (in order); logs every call."""

    def __init__(self, script, fields=()):
        self.script, self.fields, self.log = list(script), list(fields), []

    def rand(self):
        self.log.append("rand")
        return float(self.script.pop(0))

    def randint(self, *a):
        self.log.append("randint%r" % (a,))
        return int(self.script.pop(0))

    def randn(self, *shape):
        self.log.append("randn")
        return self.fields.pop(0)

    def normal(self, loc=0.0, scale=1.0, size=None):
        self.log.append("normal")
        return loc + scale * self.fields.pop(0)


class RecordingRNG:
    """A RandomState whose scalar draws are logged (and whose per-pixel draws are logged and made)."""

    def __init__(self, seed):
        self.rs, self.log, self.values = np.random.RandomState(seed), [], []

    def rand(self):
        self.log.append("rand")
        v = self.rs.rand()
        self.values.append(v)
        return v

    def randint(self, *a):
        self.log.append("randint%r" % (a,))
        v = self.rs.randint(*a)
        self.values.append(v)
        return v

    def randn(self, *shape):
        self.log.append("randn")
        return self.rs.randn(*shape)

    def normal(self, loc=0.0, scale=1.0, size=None):
        self.log.append("normal")
        return self.rs.normal(loc, scale, size)


def reference_self(dataset, rng, frame):
    """``self`` of the dataset's Dataset with the reference's augmentation methods bound to it."""
    import cv2
    path = os.path.join(R.REF_ROOT, "ffb6d", "datasets", dataset,
                        "%s_dataset.py" % ("ycb" if dataset == "ycb" else "linemod"))
    fns = R._extract(path, "Dataset", METHODS)

    class _Img:
        def __init__(self, a):
            self.a = a

        def __enter__(self):
            return self

        def __exit__(self, *e):
            return False

        def __array__(self, dtype=None, copy=None):
            return self.a

    def _open(p):
        if "depth" in p:
            return _Img(frame["back_dpt"])
        if "label" in p or "mask" in p:
            return _Img(frame["back_labels"])
        return _Img(frame["back_rgb"])

    np_proxy = types.SimpleNamespace(**{k: getattr(np, k) for k in dir(np) if not k.startswith("__")})
    np_proxy.random = types.SimpleNamespace(normal=rng.normal)
    for f in fns.values():
        f.__globals__.update(np=np_proxy, cv2=cv2, os=os, Image=types.SimpleNamespace(open=_open))
    self = types.SimpleNamespace(rng=rng, root="/r", cls_root="/r")
    for name, f in fns.items():
        setattr(self, name, f.__get__(self))
    self.real_gen = lambda: "bg"
    return self


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def script(dataset, hsv=(0.5, 0.5), sharpen=None, motion=None, gauss=None, noise=(0.5, 0), final=False):
    """Scalars that force the given stages, in rgb_add_noise's order.  noise = (rand, sigma)."""
    s = [0.5 if hsv else 0.0] + (list(hsv) if hsv else [])
    if dataset == "ycb":
        s += [0.9, sharpen] if sharpen is not None else [0.1]
    if motion:
        s += [0.9, (motion[0] + 0.5) / 360.0, (motion[1] - 0.5) / 15.0]
    else:
        s += [0.1]
    if gauss:
        s += [0.9, 0.9 if gauss[0] == 3 else 0.1, gauss[1]]
    else:
        s += [0.1]
    if dataset == "ycb":
        s += [noise[0], noise[1], 0.9 if final else 0.1]
    return s


def cases():
    out = {}
    c = {}
    for d in ("ycb", "linemod"):
        c[d + "_hsv_max"] = (d, 1, 40, 48, 1, script(d, hsv=(0.9999, 0.9999)))
        c[d + "_hsv_min"] = (d, 2, 40, 48, 1, script(d, hsv=(0.0, 0.0)))
        c[d + "_hsv_off"] = (d, 3, 40, 48, 1, script(d, hsv=None, gauss=(3, 0.6)))
        for ang in (0, 45, 90, 137, 359):
            for ln in (1, 7, 15):
                c["%s_motion_%d_%d" % (d, ang, ln)] = (d, 10 + ang + ln, 40, 48, 1,
                                                       script(d, hsv=None, motion=(ang, ln)))
        for k, sg in ((3, 0.0), (3, 1e-7), (3, 0.37), (5, 0.0), (5, 1e-4), (5, 0.999)):
            c["%s_gauss_%d_%g" % (d, k, sg)] = (d, 20 + k, 40, 48, 1, script(d, hsv=None, gauss=(k, sg)))
    c["ycb_sharpen_lo"] = ("ycb", 4, 40, 48, 1, script("ycb", hsv=None, sharpen=0.0))
    c["ycb_sharpen_hi"] = ("ycb", 5, 40, 48, 1, script("ycb", hsv=None, sharpen=0.9999))
    c["ycb_noise_max"] = ("ycb", 6, 40, 48, 1, script("ycb", hsv=None, noise=(0.1, 24)))
    c["ycb_noise_14"] = ("ycb", 7, 40, 48, 1, script("ycb", hsv=None, noise=(0.9, 14)))
    c["ycb_final"] = ("ycb", 8, 40, 48, 1, script("ycb", hsv=None, noise=(0.9, 9), final=True))
    c["ycb_all_odd"] = ("ycb", 9, 33, 47, 1, script("ycb", sharpen=0.5, motion=(137, 7), gauss=(5, 0.8),
                                                   noise=(0.9, 11), final=True))
    c["linemod_all_odd"] = ("linemod", 9, 35, 41, 1, script("linemod", motion=(200, 15), gauss=(3, 0.3)))
    c["ycb_full_480"] = ("ycb", 11, 480, 640, 1, script("ycb", sharpen=0.2, motion=(45, 7), gauss=(5, 0.7)))
    for name, (d, seed, h, w, ch, sc) in sorted(c.items()):
        fr = make_aug_frame(seed, h, w, d, ch)
        rec = A.draw_rgb_noise(ScriptRNG(sc), d)
        fz = np.random.RandomState(seed + 1000)
        fields = [fz.randn(h, w, 3), fz.randn(h, w, 3)]
        rng = ScriptRNG(sc, fields)
        ref = reference_self(d, rng, fr).rgb_add_noise(fr["rgb"])
        assert not rng.script, name
        out[name + "/meta"] = np.array([0 if d == "ycb" else 1, seed, h, w, ch])
        out[name + "/record"] = rec
        if rec[A.I_NOISE] and rec[A.I_NOISE_SIGMA] or rec[A.I_FINAL]:
            out[name + "/fields"] = np.stack(fields)
        if h * w >= 480 * 640:
            out[name + "/sha256_out"] = np.array(sha(ref))
        else:
            out[name + "/out"] = ref
    # add_real_back
    for name, d, ch, flag in (("back_ycb", "ycb", 1, 0.5), ("back_lm_rgb", "linemod", 1, 0.3),
                              ("back_lm_norgb", "linemod", 1, 0.7), ("back_lm_3ch", "linemod", 3, 0.1),
                              ("back_lm_3ch_odd", "linemod", 3, 0.1)):
        h, w = (37, 45) if name.endswith("odd") else (40, 48)
        fr = make_aug_frame(31 + len(name), h, w, d, ch)
        rng = ScriptRNG([flag] if d == "linemod" else [])
        rgb, dpt = reference_self(d, rng, fr).add_real_back(fr["rgb"], fr["labels"], fr["raw"], fr["raw"] > 1e-6)
        assert dpt.dtype == np.float32 and np.array_equal(dpt, dpt.astype(np.uint16))
        out[name + "/meta"] = np.array([0 if d == "ycb" else 1, 31 + len(name), h, w, ch, flag < 0.6])
        out[name + "/rgb"] = rgb
        out[name + "/dpt"] = dpt.astype(np.uint16)
    # the reference's sequence of rng calls for whole frames (get_item's augmentation block)
    for d in ("ycb", "linemod"):
        for seed in range(6):
            for typ in (("syn",) if d == "ycb" else ("render", "fuse")):
                rng = RecordingRNG(seed)
                fr = make_aug_frame(seed, 32, 32, d)
                me = reference_self(d, rng, fr)
                me.real_gen = lambda: (rng.randint(0, N_REAL), "bg")[1]
                rgb, dpt = fr["rgb"], fr["raw"]
                if d == "ycb" or typ == "render" or rng.rand() < 0.8:           # linemod_dataset.py:243
                    rgb = me.rgb_add_noise(rgb)
                    rgb, dpt = me.add_real_back(rgb, fr["labels"], dpt, dpt > 1e-6)
                    if rng.rand() > 0.8:
                        rgb = me.rgb_add_noise(rgb)
                out["calls_%s_%s_%d/log" % (d, typ, seed)] = np.array(rng.log)
    return out


def main():
    if not R.reference_sources_present():
        raise SystemExit("needs /root/reference")
    import zipfile
    data = cases()
    # fixed member order and timestamps, so the file is reproducible byte for byte
    with zipfile.ZipFile(OUT, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(data):
            import io
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(data[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
