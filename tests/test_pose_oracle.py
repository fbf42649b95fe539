"""CPU: the pose-voting oracle (oracle/pose_oracle.py) against the outputs of the reference's own
MeanShiftTorch.fit / best_fit_transform (tests/golden/pose_cases.npz, made by make_golden.py)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import pose_oracle as PO

CASES = ["small", "mid", "wide", "capped", "single"]


@pytest.fixture(scope="module")
def pose_golden():
    return np.load(os.path.join(GOLDEN, "pose_cases.npz"))


@pytest.mark.parametrize("case", CASES)
def test_mean_shift_oracle_matches_reference(pose_golden, case):
    votes = pose_golden[case + "_votes"]
    bw, max_iter = pose_golden[case + "_params"]
    for g in range(votes.shape[0]):
        c, lab, it = PO.mean_shift_fit(votes[g], bw, int(max_iter))
        assert np.abs(c - pose_golden[case + "_centres"][g]).max() < 2e-4      # metres: see oracle/pose_oracle.py on ties
        want = pose_golden[case + "_labels"][g].astype(bool)
        assert (lab != want).sum() <= max(1, votes.shape[1] // 200)            # points on the bandwidth boundary
        if case == "capped":
            assert it == int(max_iter) + 1                                      # `it > max_iter` stops AFTER max_iter + 1


def test_best_fit_oracle_catalogue():
    """The rigid-fit contract of tests/test_gpu_pose_contract.py holds for numpy's SVD route itself: on every
    degenerate problem of the catalogue a proper rotation at the least-squares minimum, so the contract can be met."""
    for name, A, B in PO.fit_catalogue():
        for g in range(A.shape[0]):
            T = PO.best_fit_transform(A[g], B[g])
            orth, det, excess, t_err = PO.fit_errors(T, A[g], B[g])
            assert orth <= 1e-12 and det <= 1e-12 and excess <= 1e-12, (name, g, orth, det, excess)
            assert t_err is None or t_err <= 1e-9, (name, g, t_err)


def test_frame_oracle_matches_reference():
    """The restatement of cal_frame_poses / cal_frame_poses_lm against the reference's own functions
    (tests/golden/pose_frame_cases.npz), on the frame the fixture was made from."""
    from ffb6d_b200.synthetic import make_pose_frame
    gold = PO.load_frame_golden(os.path.join(GOLDEN, "pose_frame_cases.npz"))
    fr = make_pose_frame(int(gold["seed"]))
    assert PO.frame_input_sha256(fr) == str(gold["input_sha256"])
    args = [fr[k] for k in ("pcld", "mask", "ctr_of", "kp_of")]
    n_kps = fr["kp_of"].shape[0]
    for name, use_ctr, flt in PO.FRAME_VARIANTS:
        ids, poses, kps = PO.cal_frame_poses(*args, use_ctr, flt, fr["mesh"], fr["cls_radius"])
        PO.check_frame_poses(ids, poses, kps, gold[name], fr["mesh"], n_kps, use_ctr)
    # the fixture exercises what it is meant to: refinement empties class 4 only when it runs
    assert not gold["TT"]["kps_4"].any() and gold["TF"]["kps_4"].any() and gold["FF"]["kps_4"].any()
    lm = PO.cal_frame_poses_lm(*args, True, True, fr["mesh"][1])[0]
    w = gold["lm"]["poses"]
    m = fr["mesh"][1]
    assert np.linalg.norm((m @ lm[:, :3].T + lm[:, 3]) - (m @ w[0][:, :3].T + w[0][:, 3]), axis=1).mean() < 2e-4
    empty = PO.cal_frame_poses_lm(args[0], np.zeros_like(args[1]), *args[2:], True, True, fr["mesh"][1])[0]
    assert np.array_equal(empty, w[1]) and np.array_equal(w[1], np.identity(4)[:3])


def _refine_with(mistake):
    """``PO.refine_mask`` carrying one plausible mistake."""
    def refine(pred_ctr, mask, ids, cls_radius, radius):
        ctrs = np.stack([PO.mean_shift_fit(pred_ctr[mask == c], radius, 300)[0] for c in ids])
        d = np.sqrt(((pred_ctr[:, None, :] - ctrs[None]) ** 2).sum(2, dtype=np.float32))
        j = d.argmin(1)
        near = ids[j]
        rad = np.asarray(cls_radius, np.float64)
        r = rad[near] if mistake == "radius_by_cls" else rad[near - 1]
        r = r * (1.6 if mistake == "radius_1.6" else 0.1 if mistake == "radius_0.1" else 0.8)
        upd = d[np.arange(len(j)), j] < r.astype(np.float32)
        if mistake != "background_too":
            upd &= mask > 0
        if mistake == "only_ties":                          # relabel only the duplicated class, not mislabelled points
            upd &= mask == ids[-1]
        return np.where(upd, near, mask)
    return refine


FRAME_MISTAKES = ["background_too", "radius_1.6", "radius_0.1", "radius_by_cls", "only_ties", "no_refinement",
                  "no_centre_filter"]


@pytest.mark.parametrize("mistake", FRAME_MISTAKES)
def test_frame_fixture_catches_mistake(monkeypatch, mistake):
    """The frame fixture is sensitive to every rule of the refinement and the centre-label filter: a restatement
    carrying one mistake fails the frame-voting contract against it (use_ctr and use_ctr_clus_flter on)."""
    from ffb6d_b200.synthetic import make_pose_frame
    gold = PO.load_frame_golden(os.path.join(GOLDEN, "pose_frame_cases.npz"))
    fr = make_pose_frame(int(gold["seed"]))
    if mistake == "no_refinement":
        monkeypatch.setattr(PO, "refine_mask", lambda pred_ctr, mask, *a: mask)
    elif mistake == "no_centre_filter":
        vote = PO._vote_object
        monkeypatch.setattr(PO, "_vote_object", lambda c, k, m, r, use_ctr, flt: vote(c, k, m, r, use_ctr, False))
    else:
        monkeypatch.setattr(PO, "refine_mask", _refine_with(mistake))
    args = [fr[k] for k in ("pcld", "mask", "ctr_of", "kp_of")]
    ids, poses, kps = PO.cal_frame_poses(*args, True, True, fr["mesh"], fr["cls_radius"])
    with pytest.raises(AssertionError):
        PO.check_frame_poses(ids, poses, kps, gold["TT"], fr["mesh"], fr["kp_of"].shape[0], True)


def test_best_fit_oracle_matches_reference(pose_golden):
    A, B, T = pose_golden["fit_A"], pose_golden["fit_B"], pose_golden["fit_T"]
    for k in range(A.shape[0]):
        got = PO.best_fit_transform(A[k], B[k])
        assert np.abs(got - T[k]).max() < 1e-9
        R = got[:, :3]
        assert abs(np.linalg.det(R) - 1.0) < 1e-9 and np.abs(R @ R.T - np.eye(3)).max() < 1e-9
