"""CPU: the numpy restatement of the per-point item arrays (oracle/item_oracle.py) and the host half of
get_pose_gt_info (ffb6d_b200.item.pose_gt_objects) reproduce, bit for bit, what the reference's own code wrote into
tests/golden/item_cases.npz on the same frames and the same ``choose``."""
import hashlib
import os

import numpy as np
import pytest

from conftest import GOLDEN, _npz_groups
from oracle import item_oracle as O
from ffb6d_b200.item import pose_gt_objects
from ffb6d_b200.synthetic import item_test_frames, make_item_frame

FRAMES = sorted(item_test_frames())
POINT_KEYS = ("cld_rgb_nrm", "labels", "kp_targ_ofst", "ctr_targ_ofst")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]) if a.dtype.kind == "f" else a


def assert_bitwise(got, want, what=""):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    assert np.array_equal(bits(got), bits(want)), what


def assert_point_outputs(got, g, what=""):
    """``got``: dict of POINT_KEYS for one frame, against the golden arrays or their digests."""
    for k in POINT_KEYS:
        if k in g:
            assert_bitwise(got[k], g[k], "%s %s" % (what, k))
        else:
            assert sha(got[k]) == str(g["sha256_" + k]), "%s %s" % (what, k)


def objects_of(frame, dataset, n_objects):
    return pose_gt_objects(frame["poses"], frame["cls_ids"], frame["kps"], frame["ctrs"], n_objects,
                           frame["kps"][0].shape[0], dataset=dataset)


def dpt_m_of(frame):
    return frame["raw"].astype(np.float32) / np.float32(frame["cam_scale"])


@pytest.fixture(scope="module")
def golden():
    return _npz_groups(os.path.join(GOLDEN, "item_cases.npz"))


@pytest.mark.parametrize("name", FRAMES)
def test_inputs_unchanged(golden, name):
    frame = item_test_frames()[name][0]
    for k in ("raw", "rgb", "nrm", "labels", "poses"):
        assert sha(frame[k]) == str(golden[name]["sha256_in_" + k]), "input generator changed: " + k
    assert sha(dpt_m_of(frame)) == str(golden[name]["sha256_dpt_map_m"])


@pytest.mark.parametrize("name", FRAMES)
def test_pose_gt_objects_match_reference(golden, name):
    frame, dataset, _, n_objects = item_test_frames()[name]
    g, obj = golden[name], objects_of(frame, dataset, n_objects)
    for k in ("RTs", "kp_3ds", "ctr_3ds", "cls_ids"):
        assert_bitwise(obj[k], g[k], k)
    assert_bitwise(obj["obj_kps"], g["kp3ds64"], "obj_kps")
    assert_bitwise(obj["obj_ctr"], g["ctr3ds64"], "obj_ctr")
    n = len(frame["cls_ids"])
    assert obj["obj_cls"].dtype == np.int32 and obj["obj_cls"].shape == (n_objects,)
    assert np.array_equal(obj["obj_cls"][:n], frame["cls_ids"].astype(np.int32))
    assert (obj["obj_cls"][n:] == -1).all() and (g["cls_ids"][n:] == 0).all()


@pytest.mark.parametrize("name", FRAMES)
def test_oracle_matches_reference(golden, name):
    frame, dataset, n_points, n_objects = item_test_frames()[name]
    g, obj = golden[name], objects_of(frame, dataset, n_objects)
    assert g["choose"].shape == (n_points,)
    out = O.point_item(dpt_m_of(frame), frame["K"], g["choose"], frame["rgb"], frame["labels"], frame["nrm"],
                       obj["obj_cls"], obj["obj_kps"], obj["obj_ctr"])
    assert_point_outputs(dict(zip(POINT_KEYS, out)), g, name)


def test_golden_frames_cover_the_cases(golden):
    """The frames exercise what item_test_frames says they do."""
    frames = item_test_frames()
    ys = frames["ycb_small"][0]
    msk = ys["raw"] > 0
    assert 400 <= msk.sum() < frames["ycb_small"][2]                                  # 'wrap' padding
    lab = golden["ycb_small"]["labels"]
    cls = list(ys["cls_ids"])
    assert 9 in lab and 9 not in cls                                                 # a label absent from the list
    assert 20 in cls and 20 not in ys["labels"]                                      # an object without points
    assert cls.count(3) == 2 and 3 in lab                                            # a duplicated class id
    assert (lab == 0).any()                                                          # background, padding slots
    for name in ("ycb_small", "lm_small"):
        assert frames[name][2] % 64 != 0                                             # not a multiple of the tile
    assert frames["lm_small"][0]["nrm"].dtype == np.float64
    assert {f[0]["kps"][0].shape[0] for f in frames.values()} == {8, 16}


def test_offsets_need_the_float64_point(golden):
    """Subtracting the keypoints from the float32 point instead of the float64 one changes many offsets: the
    restatement's float64 path is what the golden data pins."""
    frame, dataset, _, n_objects = item_test_frames()["ycb_small"]
    g, obj = golden["ycb_small"], objects_of(frame, dataset, n_objects)
    cld32 = g["cld_rgb_nrm"][:3].T.astype(np.float64)
    hit = (g["kp_targ_ofst"] != 0).any(axis=(1, 2))
    slot = {int(c): i for i, c in enumerate(obj["obj_cls"]) if c >= 0}
    s = np.array([slot[int(v)] for v in g["labels"][hit]])
    alt = (cld32[hit][:, None, :] - obj["obj_kps"][s]).astype(np.float32)
    assert (alt != g["kp_targ_ofst"][hit]).mean() > 0.05


def test_pose_gt_objects_rejects():
    fr = make_item_frame(5, h=16, w=16, cls_ids=(1, 2, 3), blobs=(1,))
    with pytest.raises(ValueError):
        pose_gt_objects(fr["poses"], fr["cls_ids"], fr["kps"], fr["ctrs"], 2, 8)              # 3 objects > 2 slots
    with pytest.raises(ValueError):
        pose_gt_objects(fr["poses"], fr["cls_ids"], fr["kps"], fr["ctrs"], 22, 16)             # kps are [8,3]
    with pytest.raises(ValueError):
        pose_gt_objects(fr["poses"], fr["cls_ids"], fr["kps"][:2], fr["ctrs"], 22, 8)          # one set per object
    with pytest.raises(ValueError):
        pose_gt_objects(fr["poses"], fr["cls_ids"], fr["kps"], fr["ctrs"], 22, 8, dataset="bop")
    lm = make_item_frame(6, h=16, w=16, dataset="linemod", cls_ids=(1,), blobs=(1,))
    with pytest.raises(ValueError):
        pose_gt_objects(lm["poses"], [2], lm["kps"], lm["ctrs"], 2, 8, dataset="linemod")
