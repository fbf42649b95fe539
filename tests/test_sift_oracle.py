"""oracle/sift_oracle.py against OpenCV's SIFT keypoints (tests/golden/sift_cases.npz) to the bound DESIGN.md §4.33
states, and closed forms of its steps.  CPU only."""
import collections
import os

import numpy as np
import pytest

from oracle import sift_oracle as S
import orb_cases as OC
import sift_cases as SC

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sift_cases.npz"))
SIZE_ULPS = 8          # OpenCV's sizes differ from the oracle's by up to 7 ulp for ~2% of keypoints
ANGLE_DEG = 1e-4       # OpenCV 4.13's exp / atan / magnitude differ from the oracle's in the last bits


def assert_matches_opencv(d, name):
    """The bound of DESIGN.md §4.33: the same number of keypoints, the same (packed octave, pt) multiset bit for bit
    (so the same int32 pixels, all the tool reads), and per (octave, pt) the same sizes to SIZE_ULPS and angles to
    ANGLE_DEG."""
    k, o = GOLDEN["kp:" + name], GOLDEN["oct:" + name]
    assert len(d["octave"]) == len(o)
    want = collections.defaultdict(list)
    for oc, row in zip(o.tolist(), k):
        want[(oc, row[0].view(np.uint32).item(), row[1].view(np.uint32).item())].append(row[2:4])
    got = collections.defaultdict(list)
    for oc, p, s, a in zip(d["octave"].tolist(), d["pt"], d["size"], d["angle"]):
        got[(oc, p[0].view(np.uint32).item(), p[1].view(np.uint32).item())].append(np.array([s, a], np.float32))
    assert {key: len(v) for key, v in got.items()} == {key: len(v) for key, v in want.items()}
    for key in got:
        g = np.array(sorted(map(tuple, got[key])), np.float32)
        w = np.array(sorted(map(tuple, want[key])), np.float32)
        assert np.all(np.abs(g[:, 0].view(np.int32) - w[:, 0].view(np.int32)) <= SIZE_ULPS), key
        assert np.all(np.abs(g[:, 1] - w[:, 1]) <= ANGLE_DEG), key


@pytest.mark.parametrize("i", [i for i, c in enumerate(SC.CASES) if c[2] * c[3] <= 240 * 320])
def test_detect_matches_opencv(i):
    assert_matches_opencv(S.detect(SC.image(*SC.CASES[i])), str(i))


@pytest.mark.parametrize("v", SC.APE_VIEWS)
def test_detect_matches_opencv_on_ape_renders(v):
    _, rgb = OC.ape_render(GOLDEN["ape_poses"][v])
    d = S.detect(rgb)
    assert len(d["octave"]) > 5
    assert_matches_opencv(d, "ape%d" % v)


def test_canonical_order_and_packing():
    d = S.detect(SC.image(6, 0, 120, 160))
    o = d["octave"].astype(np.int64)
    octv = ((o & 255) + 1) & 255                       # 255 is octave -1 (the upscaled image), 0 the input's scale
    layer = (o >> 8) & 255
    assert np.all(np.diff(octv) >= 0) and set(layer.tolist()) <= {1, 2, 3}
    assert np.all(d["size"] > 0) and np.all((d["angle"] >= 0) & (d["angle"] < 360))


def test_orientation_copies_share_a_point():
    """Each strict peak of the 36-bin histogram is its own keypoint at the same pt: fewer distinct points than
    keypoints on round blobs, and at most 18 copies of one."""
    d = S.detect(SC.image(6, 0, 120, 160))
    pts = collections.Counter(map(tuple, d["pt"].tolist()))
    assert len(pts) < len(d["pt"]) and max(pts.values()) <= S.MAX_COPIES


def test_octave_sizes():
    assert [hw for hw in S.octave_sizes(480, 640)] == [(960 >> o, 1280 >> o) for o in range(8)] + [(3, 5)]
    assert S.n_octaves(4, 4) == 2 and S.n_octaves(2048, 24) == 5


def test_blur_of_constant_and_taps():
    for s in [S.base_sigma()] + S.layer_sigmas():
        k = S.gaussian_taps(s)
        assert len(k) % 2 == 1 and np.array_equal(k, k[::-1]) and abs(float(k.astype(np.float64).sum()) - 1) < 1e-6
    c = np.full((7, 21), 64, np.float32)
    out = S.blur(c, S.gaussian_taps(S.layer_sigmas()[-1]))
    assert np.allclose(out, 64, rtol=1e-6, atol=0)


def test_column_modes():
    assert S.column_modes(5).tolist() == [1, 1, 1, 1, 2]
    assert S.column_modes(13).tolist() == [0] * 8 + [1] * 4 + [2]
    assert S.column_modes(16).tolist() == [0] * 16


def test_hal_closed_forms():
    assert S.exp32(np.float32(0)) == 1
    x = np.linspace(-36, 0, 3601).astype(np.float32)
    assert np.allclose(S.exp32(x), np.exp(x.astype(np.float64)), rtol=3e-6, atol=0)
    assert S.atan32(np.float32(0), np.float32(1)) == 0 and abs(S.atan32(np.float32(1), np.float32(0)) - 90) < 1e-3
    assert S.mag32(np.float32(3), np.float32(4)) == 5


def test_dedup_keeps_the_larger_response():
    kp = dict(pt=(np.float32(1), np.float32(2)), size=np.float32(3), angle=np.float32(4), octave=5)
    keep = S.dedup([dict(kp, response=np.float32(0.1)), dict(kp, response=np.float32(0.2)),
                    dict(kp, response=np.float32(0.2)), dict(kp, pt=(np.float32(1), np.float32(3)), response=0.0)])
    assert keep.tolist() == [False, True, False, True]
