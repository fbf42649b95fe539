"""CPU: the numpy restatement of the drawing (oracle/vis_oracle.py) equals the reference's own outputs in
tests/golden/vis_cases.npz bitwise, and ``vis.get_label_color`` / ``label_color_list`` equal the reference's tables."""
import os
from fractions import Fraction

import numpy as np
import pytest

from conftest import GOLDEN
import vis_cases as VC
from oracle import vis_oracle as O


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "vis_cases.npz"))
    return {k: z[k] for k in z.files}


def test_fma_is_correctly_rounded():
    rs = np.random.RandomState(5)
    n = 4000
    a, b, c = (rs.normal(size=n) * 10.0 ** rs.uniform(-8, 8, n) for _ in range(3))
    c[::4] = -(a[::4] * b[::4])                    # cancellation: the result is the product's rounding error
    got = O.fma(a, b, c)
    want = [float(Fraction(x) * Fraction(y) + Fraction(z)) for x, y, z in zip(a, b, c)]
    assert np.array_equal(got, np.array(want))
    nan = O.fma(np.array([np.nan, np.inf, np.inf, 1.0]), np.array([1.0, 0.0, 1.0, 1.0]),
                np.array([0.0, 0.0, -np.inf, np.inf]))
    assert np.isnan(nan[:3]).all() and nan[3] == np.inf


def test_to_int32_is_numpys_cast():
    q = np.array([np.nan, np.inf, -np.inf, 2.0 ** 31, 2.0 ** 31 - 1, -2.0 ** 31, -2.0 ** 31 - 1, 1e20, -7.0, 0.0])
    with np.errstate(invalid="ignore"):
        assert np.array_equal(O.to_int32(q), q.astype(np.int32))


def test_projection_matches_golden(golden):
    for name, (p, cs, K, pose) in VC.proj_cases().items():
        got = O.project_p3d(p, cs, K, pose)
        key = "proj:" + name
        if key + ":sha256" in golden:
            assert VC.sha(got) == str(golden[key + ":sha256"]), name
        else:
            assert np.array_equal(got, golden[key]), name


def test_ties_round_half_to_even(golden):
    p = VC.proj_cases()["ties_f64"][0]
    u = 2.0 * p[:, 0] / p[:, 2] + 3.0
    assert (u % 1 == 0.5).sum() > 300                # the case really holds ties
    assert np.array_equal(golden["proj:ties_f64"][:, 0], np.rint(u).astype(np.int32))


def test_edges_give_int32_min(golden):
    g = golden["proj:edge_f64"]
    assert (g == np.iinfo(np.int32).min).any() and (g != np.iinfo(np.int32).min).any()


def test_drawing_matches_golden(golden):
    for name, (bg, sets) in VC.draw_cases().items():
        img = bg.copy()
        for p2ds, r, cols in sets:
            O.draw_p2ds(img, p2ds, r, list(cols))
        assert np.array_equal(img, golden["draw:" + name]), name


def test_circle_sizes():
    assert [len(O.circle_offsets(r)[0]) for r in (0, 1, 2, 3, 5)] == [1, 5, 13, 29, 81]
    dy, dx = O.circle_offsets(3)
    widths = {k: int((dy == k).sum()) for k in range(-3, 4)}
    assert widths == {-3: 1, -2: 5, -1: 5, 0: 7, 1: 5, 2: 5, 3: 1}


def test_demo_and_view_labels_match_golden(golden):
    for ds, f in VC.demo_frames().items():
        bgr = O.demo_draw(f["rgb"], f["cls_ids"], f["pred_cls_ids"], f["pred_pose_lst"], f["mesh_pts"], f["K"], ds,
                          f["obj_id"])
        assert VC.sha(bgr) == str(golden["demo:%s:sha256" % ds]), ds
    cld, labels = VC.view_labels_frame()
    assert VC.sha(O.view_labels(480, 640, cld.T, labels, VC.K_YCB)) == str(golden["view_labels:sha256"])


def test_label_colors(golden):
    from ffb6d_b200 import vis
    for mode in (0, 1):
        assert [vis.get_label_color(c, mode=mode) for c in range(22)] == [tuple(r) for r in
                                                                           golden["color:mode%d" % mode].tolist()]
    for n in (2, 13, 22):
        want = [tuple(r) for r in golden["color:mode2:%d" % n].tolist()]
        assert [vis.get_label_color(c, n_obj=n, mode=2) for c in range(n + 3)] == want
        assert [O.label_color_mode2(c, n) for c in range(n + 3)] == want
    for n in (2, 22):
        want = [tuple(r) for r in golden["color_lst:%d" % n].tolist()]
        assert vis.label_color_list(n) == want and O.color_lst(n) == want
    with pytest.raises(IndexError):
        vis.get_label_color(22, mode=0)
