"""GPU: ``sift_detect`` (``ffb6d_sift_detect``, DESIGN.md §4.33) equals oracle/sift_oracle.py bit for bit (the same
keypoints in the same canonical order, bitwise ``pt``, ``octave``, ``size`` and ``angle``) and OpenCV's keypoints of
tests/golden/sift_cases.npz to the bound DESIGN states: ape views, generated images, odd sizes, the smallest and
largest accepted sides, ``B = 0``, a cap too small (reported, then rerun), and repeatability."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib, objinfo
from ffb6d_b200.render import RenderMeshTable
from oracle import sift_oracle as S
import orb_cases as OC
import sift_cases as SC
from test_sift_oracle import assert_matches_opencv

pytestmark = pytest.mark.gpu


def detect(imgs, **kw):
    x = torch.from_numpy(np.stack(imgs)).cuda()
    count, pt, octave, size, angle = (t.cpu().numpy() for t in F.sift_detect(x, **kw))
    return [dict(pt=pt[b, :count[b]], octave=octave[b, :count[b]], size=size[b, :count[b]],
                 angle=angle[b, :count[b]]) for b in range(len(imgs))], count


def assert_equal_to_oracle(got, img):
    want = S.detect(img)
    assert np.array_equal(got["octave"], want["octave"])
    for k in ("pt", "size", "angle"):
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    return want


def test_ape_views_match_oracle():
    xyz, faces, rgb = OC.ape_mesh()
    table = RenderMeshTable([(xyz, faces, rgb)])
    poses = objinfo.sphere_poses(objinfo.get_r(objinfo.get_3D_bbox(xyz)))
    _, img, _ = F.render_rgbd(table, np.zeros((9, 1), np.int32), poses[:, None, :3, :].astype(np.float32),
                              np.ones((9, 1), np.uint8), objinfo.TOOL_K, 480, 640)
    img = img.cpu().numpy()
    got, count = detect(list(img))
    assert count.sum() > 50
    for g, im in zip(got, img):
        assert_equal_to_oracle(g, im)


@pytest.mark.parametrize("shape", [(120, 160), (480, 640)])
def test_generated_batches_match_oracle_and_opencv(shape):
    idx = [i for i, c in enumerate(SC.CASES) if tuple(c[2:]) == shape]
    imgs = [SC.image(*SC.CASES[i]) for i in idx]
    got, _ = detect(imgs)
    for i, g, img in zip(idx, got, imgs):
        assert_equal_to_oracle(g, img)
        assert_matches_opencv(g, str(i))


@pytest.mark.parametrize("hw", [(4, 4), (9, 13), (33, 251), (77, 179), (97, 131), (301, 167), (240, 320), (64, 80),
                                (100, 100)])
def test_odd_and_small_sizes(hw):
    idx = [i for i, c in enumerate(SC.CASES) if tuple(c[2:]) == hw]
    img = SC.image(*SC.CASES[idx[0]])
    got, _ = detect([img])
    assert_equal_to_oracle(got[0], img)
    assert_matches_opencv(got[0], str(idx[0]))


@pytest.mark.parametrize("hw", [(_lib.SIFT_MIN_SIDE, 37), (_lib.SIFT_MAX_SIDE, 24), (24, _lib.SIFT_MAX_SIDE)])
def test_side_limits(hw):
    img = SC.image(6, 21, *hw)
    got, _ = detect([img])
    assert_equal_to_oracle(got[0], img)


def test_empty_batch_and_black_frame():
    count, pt, octave, size, angle = F.sift_detect(torch.zeros((0, 64, 64, 3), dtype=torch.uint8, device="cuda"))
    assert count.shape == (0,) and pt.shape[0] == 0
    got, count = detect([SC.image(5, 0, 100, 100)])
    assert count[0] == 0


def test_small_cap_is_reported_then_rerun():
    imgs = [SC.image(6, s, 120, 160) for s in range(3)]
    want, wc = detect(imgs)
    x = torch.from_numpy(np.stack(imgs)).cuda()
    count = F.sift_detect(x, cap=5, check=False)[0].cpu().numpy()
    assert np.all(count > 5)                                   # did not fit: the count before deduplication
    got, gc = detect(imgs, cap=5)                              # check=True reruns with a cap that fits
    assert np.array_equal(gc, wc)
    for g, w in zip(got, want):
        for k in g:
            assert np.array_equal(g[k], w[k]), k


def test_repeatable():
    x = torch.from_numpy(np.stack([SC.image(6, s, 240, 320) for s in range(3)])).cuda()
    a = [t.clone() for t in F.sift_detect(x)]
    for _ in range(2):
        b = F.sift_detect(x)
        assert all(torch.equal(u, v) for u, v in zip(a, b))
