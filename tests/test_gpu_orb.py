"""GPU: ``orb_detect`` (``ffb6d_orb_detect``, DESIGN.md §4.32) equals oracle/orb_oracle.py bit for bit (the same
keypoint sets, bitwise equal ``pt`` and responses, canonical order) and OpenCV's keypoints of tests/golden/orb_cases.npz
as sets: mixed batches, empty frames, odd and small sizes, tie-heavy frames; repeatability; a call at the frame and
side limits."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib
from oracle import orb_oracle as O
import orb_cases as OC
from test_orb_oracle import GOLDEN, as_set, golden_set

pytestmark = pytest.mark.gpu


def detect(imgs):
    x = torch.from_numpy(np.stack(imgs)).cuda()
    count, pt, octave, response = (t.cpu().numpy() for t in F.orb_detect(x))
    return [dict(pt=pt[b, :count[b]], octave=octave[b, :count[b]], response=response[b, :count[b]])
            for b in range(len(imgs))], (count, pt, octave, response)


def assert_equal_to_oracle(got, img):
    want = O.detect(img)
    assert np.array_equal(got["octave"], want["octave"])
    assert np.array_equal(got["pt"].view(np.uint32), want["pt"].view(np.uint32))
    assert np.array_equal(got["response"].view(np.uint32), want["response"].view(np.uint32))


@pytest.mark.parametrize("shape", [(480, 640), (240, 320), (200, 260), (77, 179), (301, 167)])
def test_batches_match_oracle_and_opencv(shape):
    idx = [i for i, c in enumerate(OC.CASES) if tuple(c[2:]) == shape]
    imgs = [OC.image(*OC.CASES[i]) for i in idx]
    got, _ = detect(imgs)
    for i, g, img in zip(idx, got, imgs):
        assert_equal_to_oracle(g, img)
        assert as_set(g["octave"], g["pt"], g["response"]) == golden_set(str(i))


def test_mixed_batch_with_empty_frames():
    imgs = [OC.image(5, 0, 100, 100), OC.image(0, 3, 100, 100), OC.image(5, 0, 100, 100), OC.image(2, 1, 100, 100)]
    got, (count, _, _, _) = detect(imgs)
    assert count[0] == 0 and count[2] == 0 and count[1] > 0 and count[3] > 0
    for g, img in zip(got, imgs):
        assert_equal_to_oracle(g, img)


@pytest.mark.parametrize("hw", [(2, 2), (3, 70), (63, 63), (64, 64), (65, 70), (97, 131), (141, 391), (391, 141),
                                (33, 500)])
def test_small_and_odd_sizes(hw):
    i = [k for k, c in enumerate(OC.CASES) if c[0] == 0 and c[1] >= 10 and tuple(c[2:]) == hw]
    img = OC.image(*OC.CASES[i[0]]) if i else OC.image(0, 10, *hw)
    got, _ = detect([img])
    assert_equal_to_oracle(got[0], img)
    if i:
        assert as_set(got[0]["octave"], got[0]["pt"], got[0]["response"]) == golden_set(str(i[0]))


def test_ties_kept_at_both_cuts():
    img = OC.image(2, 0, 200, 260)
    got, _ = detect([img])
    g = got[0]
    n0 = np.count_nonzero(g["octave"] == 0)
    assert n0 > O.level_budgets()[0]
    assert_equal_to_oracle(g, img)


def test_repeatable():
    x = torch.from_numpy(np.stack([OC.image(3, s, 480, 640) for s in range(3)])).cuda()
    a = [t.clone() for t in F.orb_detect(x)]
    for _ in range(2):
        b = F.orb_detect(x)
        assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_at_limits():
    # the frame limit at the smallest side, and the side limit in both directions
    n = _lib.ORB_MAX_FRAMES
    x = torch.zeros((n, 2, 2, 3), dtype=torch.uint8, device="cuda")
    count = F.orb_detect(x)[0]
    assert int(count.sum()) == 0
    for hw in ((_lib.ORB_MAX_SIDE, 64), (64, _lib.ORB_MAX_SIDE)):
        img = OC.image(0, 21, *hw)
        got, _ = detect([img])
        assert_equal_to_oracle(got[0], img)
