"""CPU: the fuse oracle (DESIGN.md §4.34) against closed forms, the crop table's host side, and the host draws of
``draw_fuse_frame`` / ``draw_linemod_frame_kind``: ranges, one crop per class, a permutation of the slots, the label on
the target alone, and the principal-point shift that keeps the target's back-projection exact."""
import numpy as np
import pytest

from ffb6d_b200 import fuse_frames
from oracle import fuse_oracle as O

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1


def _crop(h, w, seed, full=False):
    rs = np.random.RandomState(seed)
    sil = np.ones((h, w), np.uint8) if full else (rs.rand(h, w) < 0.6).astype(np.uint8)
    return (rs.randint(0, 256, (h, w, 3)).astype(np.uint8), rs.randint(1, 5000, (h, w)).astype(np.uint16), sil)


def _one(crops, slots, H, W, **kw):
    crop = np.array([[s[0] for s in slots]], np.int64)
    offset = np.array([[s[1] for s in slots]], np.int64)
    label = np.array([[s[2] for s in slots]], np.uint8)
    d, c, l = O.fuse(crops, crop, offset, label, H, W, **kw)
    return d[0], c[0], l[0]


def test_one_crop_pixel_set():
    crops = [_crop(4, 5, 0)]
    d, c, l = _one(crops, [(0, (2, 3), 7)], 10, 12)
    rgb, dpt, sil = crops[0]
    want = {(2 + i, 3 + j) for i, j in zip(*np.nonzero(sil))}
    assert set(zip(*np.nonzero(l))) == want
    for i, j in zip(*np.nonzero(sil)):
        assert d[2 + i, 3 + j] == dpt[i, j] and (c[2 + i, 3 + j] == rgb[i, j]).all() and l[2 + i, 3 + j] == 7
    assert (d[l == 0] == 0).all() and (c[l == 0] == 0).all()


def test_later_slot_wins_and_empty_slots():
    crops = [_crop(4, 4, 1, full=True), _crop(4, 4, 2, full=True)]
    d, c, l = _one(crops, [(0, (0, 0), 1), (1, (2, 2), 2)], 8, 8)
    assert (l[2:6, 2:6] == 2).all() and (d[2:6, 2:6] == crops[1][1]).all()
    assert (l[0:2, 0:4] == 1).all() and (l[2:4, 0:2] == 1).all()
    # reversed order: the first crop now covers the overlap
    _, _, l2 = _one(crops, [(1, (2, 2), 2), (0, (0, 0), 1)], 8, 8)
    assert (l2[0:4, 0:4] == 1).all() and (l2[4:6, 2:6] == 2).all()
    # -1 and indices outside the table paste nothing
    for k in (-1, 2, 99, I32_MIN, I32_MAX):
        d, c, l = _one(crops, [(k, (0, 0), 5)], 8, 8)
        assert not l.any() and not d.any() and not c.any()


def test_silhouette_holes_let_earlier_slots_through():
    a = _crop(3, 3, 3, full=True)
    b = list(_crop(3, 3, 4, full=True))
    b[2] = np.array([[1, 0, 1], [0, 0, 0], [1, 0, 1]], np.uint8)
    d, c, l = _one([a, tuple(b)], [(0, (0, 0), 1), (1, (0, 0), 2)], 3, 3)
    assert (l == np.where(b[2] != 0, 2, 1)).all()
    assert (d == np.where(b[2] != 0, b[1], a[1])).all()


@pytest.mark.parametrize("off, box", [
    ((-2, -3), (0, 1, 0, 1)), ((6, 9), (6, 7, 9, 10)), ((-1, 8), (0, 2, 8, 10)),
    ((-4, 0), None), ((8, 0), None), ((0, 11), None), ((0, -5), None),
    ((I32_MIN, 0), None), ((0, I32_MIN), None), ((I32_MAX, I32_MAX), None), ((I32_MIN, I32_MAX), None),
])
def test_crops_partly_or_wholly_outside(off, box):
    crops = [_crop(4, 5, 5, full=True)]
    d, c, l = _one(crops, [(0, off, 1)], 8, 11)
    if box is None:
        assert not l.any() and not d.any()
        return
    r0, r1, c0, c1 = box
    want = np.zeros((8, 11), bool)
    want[r0:r1 + 1, c0:c1 + 1] = True
    assert (l.astype(bool) == want).all()
    assert d[r0, c0] == crops[0][1][r0 - off[0], c0 - off[1]]


def test_in_place_leaves_uncovered_pixels_alone():
    rs = np.random.RandomState(6)
    bg = (rs.randint(0, 65535, (2, 6, 7)).astype(np.uint16), rs.randint(0, 256, (2, 6, 7, 3)).astype(np.uint8),
          rs.randint(0, 3, (2, 6, 7)).astype(np.uint8))
    crops = [_crop(3, 3, 7)]
    crop = np.array([[0], [0]])
    offset = np.array([[[1, 1]], [[2, 2]]])
    d, c, l = O.fuse(crops, crop, offset, np.array([[9], [9]]), 6, 7, active=[True, False], out=bg)
    covered = l[0] == 9
    assert covered.sum() == crops[0][2].sum()
    assert (d[0][~covered] == bg[0][0][~covered]).all() and (c[0][~covered] == bg[1][0][~covered]).all()
    assert (d[1] == bg[0][1]).all() and (c[1] == bg[1][1]).all() and (l[1] == bg[2][1]).all()   # inactive


def test_inclusive_bounding_box():
    m = np.zeros((9, 10), np.uint8)
    m[2, 3] = 255
    m[6, 8] = 1
    assert O.crop_box(m) == (2, 6, 3, 8)
    m1 = np.zeros((5, 5), bool)
    m1[4, 4] = True
    assert O.crop_box(m1) == (4, 4, 4, 4)
    assert O.crop_box(np.zeros((3, 3))) is None
    rgb, dpt, sil, org = O.crop_frame(np.zeros((9, 10, 3), np.uint8), np.zeros((9, 10), np.uint16), m)
    assert sil.shape == (5, 6) == dpt.shape and rgb.shape == (5, 6, 3) and org == (2, 3)
    assert sil[0, 0] == 1 and sil[4, 5] == 1 and sil.sum() == 2


# ------------------------------------------------------------------------------------------------ the crop table
def _frames(n_per_class=(3, 2, 4), H=40, W=50, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for cls, n in zip((1, 5, 9), n_per_class):
        for _ in range(n):
            h, w = rs.randint(3, 15), rs.randint(3, 20)
            r, c = rs.randint(0, H - h), rs.randint(0, W - w)
            mask = np.zeros((H, W), np.uint8)
            mask[r:r + h, c:c + w] = (rs.rand(h, w) < 0.7) * 255
            mask[r, c] = mask[r + h - 1, c + w - 1] = 255
            out.append((rs.randint(0, 256, (H, W, 3)).astype(np.uint8),
                        rs.randint(300, 2000, (H, W)).astype(np.uint16), mask, cls))
    return out


def test_table_packs_the_oracle_crops():
    frames = _frames()
    t = fuse_frames.FuseCropTable(iter(frames), device="cpu")       # any iterable
    assert len(t) == len(frames) and t.classes == (1, 5, 9)
    assert t.nbytes == 6 * int((t.size[:, 0] * t.size[:, 1]).sum()) + 8 * len(t) + 8 * len(t)
    for k, (rgb, dpt, mask, cls) in enumerate(frames):
        c_rgb, c_dpt, c_sil, org = O.crop_frame(rgb, dpt, mask)
        h, w = c_sil.shape
        o = int(t.off[k])
        assert t.cls[k] == cls and tuple(t.origin[k]) == org and tuple(t.size[k]) == (h, w)
        assert tuple(t.hw[k].tolist()) == (h, w)
        assert np.array_equal(t.sil[o:o + h * w].numpy().reshape(h, w), c_sil)
        assert np.array_equal(t.dpt[o:o + h * w].numpy().reshape(h, w), c_dpt)
        assert np.array_equal(t.rgb[3 * o:3 * (o + h * w)].numpy().reshape(h, w, 3), c_rgb)


def test_table_refuses_bad_frames():
    good = _frames((1, 0, 0))[0]
    rgb, dpt, mask, cls = good
    cases = [((rgb, dpt, np.zeros_like(mask), cls), "frame 1: empty silhouette"),
             ((rgb.astype(np.int32), dpt, mask, cls), "frame 1: rgb"),
             ((rgb[..., :2], dpt, mask, cls), "frame 1: rgb"),
             ((rgb, dpt.astype(np.float32), mask, cls), "frame 1: dpt"),
             ((rgb, dpt[:-1], mask, cls), "frame 1: dpt"),
             ((rgb, dpt, mask[:, :-1], cls), "frame 1: mask"),
             ((rgb, dpt, mask.astype(object), cls), "frame 1: mask"),
             ((rgb, dpt, mask), "frame 1 must be")]
    for bad, what in cases:
        with pytest.raises(ValueError, match=what):
            fuse_frames.FuseCropTable([good, bad], device="cpu")
    with pytest.raises(ValueError, match="no frames"):
        fuse_frames.FuseCropTable([], device="cpu")


# ------------------------------------------------------------------------------------------------------ the draws
K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])


def test_draw_ranges_classes_order_and_label():
    frames = _frames()
    t = fuse_frames.FuseCropTable(frames, device="cpu")
    rs = np.random.RandomState(1)
    H, W = 30, 40
    seen_first = set()
    for i in range(300):
        target = (1, 5, 9)[i % 3]
        keys, K_f, tk = fuse_frames.draw_fuse_frame(rs, t if i % 2 else t.meta, target, K, H, W)
        crop, off, lab = keys["fuse_crop"], keys["fuse_offset"], keys["fuse_label"]
        assert keys["fused"] is True and crop.dtype == np.int32 and off.dtype == np.int32 and lab.dtype == np.uint8
        assert crop.shape == (3,) and off.shape == (3, 2) and lab.shape == (3,)
        assert sorted(t.cls[crop]) == [1, 5, 9]                                   # one crop of each class
        seen_first.add(int(t.cls[crop[0]]))
        for s, k in enumerate(crop):
            h, w = t.size[k]
            assert 0 <= off[s, 0] < max(H - h, 1) and 0 <= off[s, 1] < max(W - w, 1)
        assert lab.tolist() == [int(t.cls[k] == target) for k in crop] and lab.sum() == 1
        assert tk == crop[lab.argmax()] and t.cls[tk] == target
        assert K_f.dtype == np.float64 and np.array_equal(K_f[[0, 1, 2], [0, 1, 2]], K[[0, 1, 2], [0, 1, 2]])
    assert seen_first == {1, 5, 9}                                               # the paste order is drawn
    with pytest.raises(ValueError, match="no crops"):
        fuse_frames.draw_fuse_frame(rs, t, 2, K, H, W)


def test_draw_picks_each_crop_of_a_class():
    t = fuse_frames.FuseCropTable(_frames((4, 1, 1)), device="cpu")
    rs = np.random.RandomState(2)
    counts = np.zeros(len(t), int)
    for _ in range(800):
        keys, _, _ = fuse_frames.draw_fuse_frame(rs, t, 1, K, 30, 40)
        counts[keys["fuse_crop"]] += 1
    assert (counts[:4] > 120).all() and counts[4] == counts[5] == 800


def test_k_shift_keeps_the_target_back_projection():
    """Back-projecting the pasted target pixels with the drawn K gives the source pixels' points under the base K."""
    frames = _frames((2, 2, 2), H=120, W=160, seed=3)
    t = fuse_frames.FuseCropTable(frames, device="cpu")
    crops = [O.crop_frame(*f[:3])[:3] for f in frames]
    rs = np.random.RandomState(4)
    checked = 0
    for i in range(20):
        target = (1, 5, 9)[i % 3]
        keys, K_f, tk = fuse_frames.draw_fuse_frame(rs, t, target, K, 120, 160)
        d, _, l = O.fuse(crops, keys["fuse_crop"][None], keys["fuse_offset"][None], keys["fuse_label"][None], 120, 160)
        r, c = np.nonzero(l[0] == 1)
        z = d[0][r, c].astype(np.float64) / 1000.0
        x_f, y_f = (c - K_f[0, 2]) * z / K_f[0, 0], (r - K_f[1, 2]) * z / K_f[1, 1]
        s = int(np.flatnonzero(keys["fuse_label"])[0])
        rs_, cs_ = r - keys["fuse_offset"][s, 0] + t.origin[tk, 0], c - keys["fuse_offset"][s, 1] + t.origin[tk, 1]
        src = frames[tk]
        assert (src[2][rs_, cs_] != 0).all() and np.array_equal(src[1][rs_, cs_], d[0][r, c])
        z_s = src[1][rs_, cs_].astype(np.float64) / 1000.0
        x_s, y_s = (cs_ - K[0, 2]) * z_s / K[0, 0], (rs_ - K[1, 2]) * z_s / K[1, 1]
        assert np.abs(x_f - x_s).max() <= 1e-12 and np.abs(y_f - y_s).max() <= 1e-12
        checked += r.size
    assert checked > 500


def test_unfused_keys():
    t = fuse_frames.FuseCropTable(_frames(), device="cpu")
    k = fuse_frames.unfused_keys(t.meta)
    assert k["fused"] is False and k["fuse_crop"].tolist() == [-1, -1, -1] and k["fuse_offset"].shape == (3, 2)


def test_frame_kind_follows_real_syn_gen():
    class Rec:
        def __init__(self, vals):
            self.vals, self.n = list(vals), 0

        def rand(self):
            self.n += 1
            return self.vals.pop(0)

    for vals, kind, n in (([0.1], "real", 1), ([0.29], "real", 1), ([0.3, 0.1], "fuse", 2), ([0.9, 0.39], "fuse", 2),
                          ([0.5, 0.4], "render", 2), ([0.5, 0.99], "render", 2)):
        r = Rec(vals)
        assert fuse_frames.draw_linemod_frame_kind(r) == kind and r.n == n
    assert fuse_frames.draw_linemod_frame_kind(Rec([0.5, 0.5]), 0.6, 0.6) == "real"
    rs = np.random.RandomState(5)
    kinds = [fuse_frames.draw_linemod_frame_kind(rs) for _ in range(20000)]
    frac = {k: kinds.count(k) / len(kinds) for k in ("real", "fuse", "render")}
    assert abs(frac["real"] - 0.3) < 0.015 and abs(frac["fuse"] - 0.28) < 0.015 and abs(frac["render"] - 0.42) < 0.015
