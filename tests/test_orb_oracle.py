"""oracle/orb_oracle.py against OpenCV's keypoints (tests/golden/orb_cases.npz), closed forms and the reference's
sphere poses and lift.  CPU only."""
import os

import numpy as np
import pytest

from oracle import orb_oracle as O
import orb_cases as OC

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "orb_cases.npz"))


def as_set(octave, pt, response):
    pt = np.asarray(pt, np.float32).reshape(-1, 2)
    return set(zip(np.asarray(octave).astype(int).tolist(), pt[:, 0].view(np.uint32).tolist(),
                   pt[:, 1].view(np.uint32).tolist(), np.asarray(response, np.float32).view(np.uint32).tolist()))


def golden_set(name):
    k = GOLDEN["kp:" + name]
    return as_set(k[:, 0], k[:, 1:3], k[:, 3])


@pytest.mark.parametrize("i", range(len(OC.CASES)))
def test_detect_matches_opencv(i):
    d = O.detect(OC.image(*OC.CASES[i]))
    assert as_set(d["octave"], d["pt"], d["response"]) == golden_set(str(i))


@pytest.mark.parametrize("v", OC.APE_VIEWS)
def test_detect_matches_opencv_on_ape_renders(v):
    _, rgb = OC.ape_render(GOLDEN["ape_poses"][v])
    d = O.detect(rgb)
    assert len(d["octave"]) > 50
    assert as_set(d["octave"], d["pt"], d["response"]) == golden_set("ape%d" % v)


def test_canonical_order():
    d = O.detect(OC.image(0, 0, 480, 640))
    assert np.all(np.diff(d["octave"]) >= 0)
    for l in range(O.N_LEVELS):
        p = d["pt"][d["octave"] == l]
        assert np.array_equal(np.lexsort((p[:, 0], p[:, 1])), np.arange(len(p)))


def test_level_budgets():
    b = O.level_budgets()
    assert b == [109, 90, 75, 63, 52, 44, 36, 31] and sum(b) == 500


def test_ties_are_kept():
    """The checker tile repeats: far more points than the budget tie at both cuts, and every tie is kept."""
    d = O.detect(OC.image(2, 0, 200, 260))
    n0 = np.count_nonzero(d["octave"] == 0)
    assert n0 > O.level_budgets()[0]
    assert len(np.unique(d["response"][d["octave"] == 0])) < n0


def test_single_square_and_black_frame():
    assert len(O.detect(OC.image(5, 0, 100, 100))["octave"]) == 0
    d = O.detect(OC.image(4, 0, 120, 160))
    # one keypoint at each of the square's four corners (level 1: at level 0 the corner's neighbours tie with it)
    corners = np.array([(60, 40), (99, 40), (60, 79), (99, 79)], np.float32)
    dist = np.abs(d["pt"][:, None, :] - corners[None]).max(-1)
    assert len(d["pt"]) == 4 and np.all(dist.min(1) <= 2) and sorted(dist.argmin(1)) == [0, 1, 2, 3]


def test_resize_identity_and_constant():
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (37, 53), dtype=np.uint8)
    assert np.array_equal(O.resize_exact(img, 53, 37), img)
    c = np.full((41, 29), 77, np.uint8)
    assert np.all(O.resize_exact(c, 17, 23) == 77)


def test_fast_score_closed_form():
    img = np.zeros((9, 9), np.uint8)
    img[4, 4] = 100                      # a bright dot: every circle pixel is 100 darker
    s = O.fast_scores(img)
    assert s[4, 4] == 99 and np.count_nonzero(s) == 1


def test_sphere_poses_match_reference():
    from ffb6d_b200 import objinfo
    r = GOLDEN["ape_radius"]
    assert r.dtype == np.float32
    want = GOLDEN["ape_poses"]
    assert np.array_equal(O.sphere_poses(r[()]), want)
    assert np.array_equal(objinfo.sphere_poses(r[()]), want)
    _, _, _, _, radius = OC.ape_setup()
    assert radius == r


@pytest.mark.parametrize("v", OC.APE_VIEWS)
def test_lift_matches_reference(v):
    depth, _ = OC.ape_render(GOLDEN["ape_poses"][v])
    pts, ok = O.lift(GOLDEN["liftpt:ape%d" % v], depth, GOLDEN["ape_K"], GOLDEN["ape_poses"][v])
    want = GOLDEN["lift:ape%d" % v]
    assert pts.shape == want.shape and pts.dtype == want.dtype == np.float64
    # numpy's dot may fuse or reorder the 3-term sums; the oracle's order is fixed (no contraction)
    np.testing.assert_allclose(pts, want, rtol=0, atol=1e-15)
    assert np.array_equal(pts.astype(np.float32), want.astype(np.float32))
