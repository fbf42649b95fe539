"""oracle/item_oracle.py -- TEST INFRASTRUCTURE ONLY.  A numpy restatement of the part of the datasets' get_item
that reads ``choose``, for checking ``ffb6d_point_item`` where the reference's sources are absent.

Reference: datasets/ycb/ycb_dataset.py:165-176 (dpt_2_pcld), 218-247 (sampling, per-point arrays) and 348-386
(get_pose_gt_info); datasets/linemod/linemod_dataset.py:188-199, 264-293, 398-436.  Where the reference loops over
the frame's objects and writes the offsets of the points of each (a later object overwriting an earlier one), this
restatement looks up each point's object in a label -> last-slot table, and forms all offsets in one broadcast
subtraction.  The arithmetic is the reference's: a float64 cloud (integer pixel grid minus float64 intrinsics),
float64 offsets, one rounding to float32 at the end.  tests/test_item_oracle.py holds it to tests/golden/item_cases.npz,
made from the reference's own code.
"""
import numpy as np


def dpt_2_pcld(dpt_m, K):
    """Organised float64 cloud ``[H,W,3]`` of a metres depth map: x from the column, y from the row."""
    H, W = dpt_m.shape
    K = np.asarray(K)
    d = dpt_m.astype(np.float32)
    rows, cols = np.indices((H, W))
    x = (cols - np.float64(K[0][2])) * d / np.float64(K[0][0])
    y = (rows - np.float64(K[1][2])) * d / np.float64(K[1][1])
    cld = np.stack((x, y, d.astype(np.float64)), axis=2)
    return cld * (d > 1e-8)[:, :, None]


def sample_choose(msk_dp, n_points):
    """The reference's draw of ``choose`` from ``msk_dp`` with numpy's global random stream (ycb_dataset.py:218-235):
    a random subset of ``n_points`` valid pixels, or all of them padded cyclically ('wrap'), then shuffled."""
    valid = msk_dp.reshape(-1).nonzero()[0].astype(np.uint32)
    picks = np.arange(len(valid))
    if len(picks) > n_points:
        keep = np.zeros(len(picks), dtype=int)
        keep[:n_points] = 1
        np.random.shuffle(keep)
        picks = picks[keep.nonzero()]
    else:
        picks = np.pad(picks, (0, n_points - len(picks)), 'wrap')
    choose = valid[picks]
    order = np.arange(choose.shape[0])
    np.random.shuffle(order)
    return choose[order]


def point_item(dpt_m, K, choose, rgb, labels, nrm, obj_cls, obj_kps, obj_ctr):
    """One frame: ``dpt_m [H,W]`` metres, ``choose [N]`` flat pixels, ``rgb [H,W,3]``, ``labels [H,W]``, ``nrm
    [H,W,3]``, and the object tables of ``ffb6d_b200.item.pose_gt_objects`` (``obj_cls [n_obj]``, ``obj_kps
    [n_obj,n_kps,3]``, ``obj_ctr [n_obj,3]``).  Returns what ``ffb6d_point_item`` writes for the frame:
    ``cld_rgb_nrm [9,N]`` f32, ``labels [N]`` i32, ``kp_targ_ofst [N,n_kps,3]`` f32, ``ctr_targ_ofst [N,3]`` f32."""
    choose = np.asarray(choose).reshape(-1).astype(np.int64)
    cld = dpt_2_pcld(dpt_m, K).reshape(-1, 3)[choose]                       # float64 [N,3]
    feats = np.empty((choose.size, 9), np.float32)
    feats[:, :3] = cld                                                    # one rounding
    feats[:, 3:6] = rgb.reshape(-1, 3)[choose]
    feats[:, 6:] = nrm.reshape(-1, 3)[choose]
    lab = labels.reshape(-1)[choose].astype(np.int64)
    slot_of = np.full(256, -1, np.int64)
    for i, c in enumerate(np.asarray(obj_cls).tolist()):
        if 0 <= c < 256:
            slot_of[c] = i                                                # the last slot of a class wins
    slot = slot_of[lab]
    hit = slot >= 0
    n_kps = obj_kps.shape[1]
    kp = np.zeros((choose.size, n_kps, 3), np.float32)
    ctr = np.zeros((choose.size, 3), np.float32)
    kp[hit] = cld[hit][:, None, :] - np.asarray(obj_kps, np.float64)[slot[hit]]
    ctr[hit] = cld[hit] - np.asarray(obj_ctr, np.float64)[slot[hit]]
    return feats.T.copy(), lab.astype(np.int32), kp, ctr
