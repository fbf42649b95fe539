"""GPU: pose estimation from decoded RGB-D frames (:mod:`ffb6d_b200.estimate`, DESIGN.md §4.27).

``build_ffb6d_inputs`` against the same keys of ``build_ffb6d_item`` and ``ops.point_input`` against
``ops.point_item(...)[0]``, bit for bit; ``estimate_poses`` against its hand composition (the forward, the argmax and
``cal_batch_poses`` / ``pose._vote``) and, at B = 1, against ``cal_frame_poses(_lm)``; ``GraphedPoseStep`` against
``estimate_poses`` over several batches, after new weights, a switched path flag and a frame without depth; and the
rejected frames.  Frames are ``synthetic.make_item_frame``'s at 480x640, sampled at the reference's 12800 points."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib, pose
from ffb6d_b200.item import pose_gt_objects
from ffb6d_b200.model import FFB6D
from ffb6d_b200.synthetic import INTRINSICS, make_item_frame

pytestmark = pytest.mark.gpu

N = 480 * 640 // 24
N_KPS = 8
CAM_SCALE = {"ycb": 10000.0, "linemod": 1000.0}
N_CLS = {"ycb": 22, "linemod": 2}
K_OF = {"ycb": INTRINSICS["ycb_K1"], "linemod": INTRINSICS["linemod"]}
OUT_KEYS = ("present", "count", "kps", "poses", "valid")


def _frame(seed, dataset, nrm_dtype=np.float32):
    if dataset == "ycb":
        return make_item_frame(seed, n_kps=N_KPS, cls_ids=(1 + seed % 7, 9, 14, 21), blobs=(1 + seed % 7, 9, 14, 3),
                               nrm_dtype=nrm_dtype)
    return make_item_frame(seed, dataset="linemod", n_kps=N_KPS, cls_ids=(1,), blobs=(1,), nrm_dtype=nrm_dtype)


def _batch(seeds, dataset, cuda, nrm_dtype=np.float32, per_frame_K=False):
    """Frames as estimate_poses takes them, plus the labels and object tables build_ffb6d_item needs."""
    fr = [_frame(s, dataset, nrm_dtype) for s in seeds]
    frames = {"dpt": torch.from_numpy(np.stack([f["raw"] for f in fr])).to(cuda),
              "rgb": torch.from_numpy(np.stack([f["rgb"] for f in fr])).to(cuda),
              "nrm_map": torch.from_numpy(np.stack([f["nrm"] for f in fr])).to(cuda)}
    if per_frame_K:
        Ks = np.stack([INTRINSICS[("linemod", "ycb_K2")[i % 2] if dataset == "linemod" else ("ycb_K1", "ycb_K2")[i % 2]]
                       for i in range(len(seeds))])
        frames["K"] = torch.from_numpy(Ks).to(cuda)
    labels = torch.from_numpy(np.stack([f["labels"] for f in fr])).to(cuda)
    objs = [pose_gt_objects(f["poses"], f["cls_ids"] if dataset == "ycb" else [1], f["kps"], f["ctrs"], N_CLS[dataset],
                            N_KPS, dataset=dataset) for f in fr]
    return frames, labels, objs


def _mesh(dataset, seed=7):
    """Mesh keypoints (8 + centre) for every class 1..21 (YCB) or the object (LineMOD), and YCB radii."""
    rs = np.random.RandomState(seed)
    if dataset == "linemod":
        return rs.uniform(-0.08, 0.08, (N_KPS + 1, 3)).astype(np.float32), None
    return ({c: rs.uniform(-0.08, 0.08, (N_KPS + 1, 3)).astype(np.float32) for c in range(1, 22)},
            list(rs.uniform(0.04, 0.12, 21)))


@pytest.fixture(scope="module")
def models(cuda):
    torch.manual_seed(0)
    return {ds: FFB6D(n_classes=N_CLS[ds], n_pts=N, n_kps=N_KPS).to(cuda).eval() for ds in ("ycb", "linemod")}


def _kw(dataset):
    mesh, radius = _mesh(dataset)
    return dict(dataset=dataset, cam_scale=CAM_SCALE[dataset], K=K_OF[dataset], mesh_kps=mesh, cls_radius=radius)


def _assert_out_equal(got, want, when):
    for k in OUT_KEYS:
        g, w = got[k], want[k]
        assert g.dtype == w.dtype and g.shape == w.shape, (when, k)
        assert torch.equal(g.view(torch.uint8) if g.dtype == torch.bool else g.contiguous().view(torch.uint8),
                           w.view(torch.uint8) if w.dtype == torch.bool else w.contiguous().view(torch.uint8)), \
            "%s: %s differs" % (when, k)


def _clone(out):
    return {k: v.clone() for k, v in out.items()}


# ------------------------------------------------------------------------------------------ inputs
@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_build_inputs_equals_item(cuda, dataset):
    """The same keys as build_ffb6d_item, bitwise, on a batch with a full frame, one with fewer than N valid pixels
    (LineMOD: 5000, 'wrap'; YCB: a small block before depth completion), one with fewer than 400 (LineMOD: 399) and
    one without depth."""
    frames, labels, objs = _batch((11, 12, 13, 14), dataset, cuda)
    raw = frames["dpt"].cpu().numpy()
    rs = np.random.RandomState(0)
    if dataset == "linemod":
        for b, n_keep in ((1, 5000), (2, 399)):
            keep = rs.choice(np.flatnonzero(raw[b]), n_keep, replace=False)
            sparse = np.zeros(raw[b].size, raw.dtype)
            sparse[keep] = raw[b].reshape(-1)[keep]
            raw[b] = sparse.reshape(raw[b].shape)
    else:
        block = raw[1, 200:210, 300:310].copy()
        raw[1] = 0
        raw[1, 200:210, 300:310] = block
        raw[2] = 0
    raw[3] = 0
    frames["dpt"] = torch.from_numpy(raw).to(cuda)
    args = (frames["dpt"], CAM_SCALE[dataset], K_OF[dataset], frames["rgb"])
    got = F.build_ffb6d_inputs(*args, frames["nrm_map"], N, seed=3, fill=dataset == "ycb")
    want = F.build_ffb6d_item(*args, labels, frames["nrm_map"], objs, N, seed=3, fill=dataset == "ycb")
    assert "labels" not in got and "kp_targ_ofst" not in got and "RTs" not in got
    assert {"rgb", "cld_rgb_nrm", "choose", "dpt_map_m", "valid", "cld_xyz0", "cld_nei_idx0", "p2r_up_nei_idx2"} <= set(got)
    for key, g in got.items():
        w = want[key]
        assert g.dtype == w.dtype and g.shape == w.shape and torch.equal(g, w), key
    choose = got["choose"][:, 0].cpu().numpy()
    if dataset == "linemod":
        assert got["valid"].tolist() == [True, True, False, False]
        assert len(np.unique(choose[1])) == 5000 < N                                   # every valid pixel, 'wrap'
    else:
        assert got["valid"].tolist()[2:] == [False, False]
    assert (choose[3] == 0).all()


@pytest.mark.parametrize("nrm_dtype", [np.float32, np.float64])
@pytest.mark.parametrize("per_frame_K", [False, True])
def test_point_input_equals_point_item(cuda, nrm_dtype, per_frame_K):
    frames, labels, objs = _batch((21, 22), "ycb", cuda, nrm_dtype)
    from ffb6d_b200.ops import _fill_depth
    _, depth_m = _fill_depth(frames["dpt"], CAM_SCALE["ycb"])
    choose = F.sample_valid_pixels(depth_m, N, seed=1)
    K = np.stack([INTRINSICS["ycb_K1"], INTRINSICS["ycb_K2"]]) if per_frame_K else INTRINSICS["ycb_K1"]
    o = {k: torch.from_numpy(np.stack([ob[k] for ob in objs])).to(cuda) for k in ("obj_cls", "obj_kps", "obj_ctr")}
    got = F.point_input(depth_m, K, choose, frames["rgb"], frames["nrm_map"])
    want = F.point_item(depth_m, K, choose, frames["rgb"], labels, frames["nrm_map"], o["obj_cls"], o["obj_kps"],
                        o["obj_ctr"])[0]
    assert got.shape == (2, 9, N) and got.dtype == torch.float32
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert torch.equal(got[:, :3].permute(0, 2, 1), F.backproject(depth_m, K, choose)[0])


# ------------------------------------------------------------------------------------------ eager
def _by_hand(model, frames, dataset, seed=0):
    mesh, radius = _mesh(dataset)
    item = F.build_ffb6d_inputs(frames["dpt"], CAM_SCALE[dataset], K_OF[dataset], frames["rgb"], frames["nrm_map"], N,
                                seed=seed, fill=dataset == "ycb")
    item["rgb"] = item["rgb"].float()
    with torch.no_grad():
        ep = model(item)
    mask = torch.max(ep["pred_rgbd_segs"], 1)[1]
    pcld = item["cld_rgb_nrm"][:, :3, :].permute(0, 2, 1).contiguous()
    if dataset == "ycb":
        votes = pose.cal_batch_poses(pcld, mask, ep["pred_ctr_ofs"], ep["pred_kp_ofs"], True, 22, True, mesh_kps=mesh,
                                     cls_radius=radius)
    else:
        votes = pose._vote(pose._lm_table(mesh, pcld.device), pcld, mask == 1, ep["pred_ctr_ofs"], ep["pred_kp_ofs"],
                           True, False, False)
    return dict(zip(OUT_KEYS, tuple(votes) + (item["valid"],))), (pcld, mask, ep)


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_estimate_equals_composition(cuda, models, dataset):
    model = models[dataset]
    frames, _, _ = _batch((31, 32), dataset, cuda)
    got = F.estimate_poses(model, frames, **_kw(dataset))
    want, _ = _by_hand(model, frames, dataset)
    _assert_out_equal(got, want, dataset)
    assert got["present"].shape == (2, N_CLS[dataset]) and got["poses"].dtype == torch.float64
    assert got["kps"].shape == (2, N_CLS[dataset], N_KPS + 1, 3)
    assert got["valid"].tolist() == [True, True]
    assert not torch.isnan(got["poses"]).any()


@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_estimate_b1_equals_frame_lists(cuda, models, dataset):
    model = models[dataset]
    frames, _, _ = _batch((41,), dataset, cuda)
    got = F.estimate_poses(model, frames, **_kw(dataset))
    _, (pcld, mask, ep) = _by_hand(model, frames, dataset)
    mesh, radius = _mesh(dataset)
    present, count = got["present"][0].cpu().numpy(), got["count"][0].cpu().numpy()
    poses, kps = got["poses"][0].cpu().numpy(), got["kps"][0].cpu().numpy()
    if dataset == "ycb":
        ids, pose_lst, kps_lst = pose.cal_frame_poses(pcld[0], mask[0], ep["pred_ctr_ofs"][0], ep["pred_kp_ofs"][0],
                                                      True, 22, True, mesh_kps=mesh, cls_radius=radius)
        assert ids.tolist() == np.flatnonzero(present).tolist()
        for c, p, k in zip(ids, pose_lst, kps_lst):
            empty = count[c] == 0
            assert np.array_equal(p, np.identity(4)[:3] if empty else poses[c]), c
            assert np.array_equal(k, np.zeros((N_KPS + 1, 3)) if empty else kps[c]), c
    else:
        lst = pose.cal_frame_poses_lm(pcld[0], mask[0], ep["pred_ctr_ofs"][0], ep["pred_kp_ofs"][0], True, 2, False, 1,
                                      mesh_kps=mesh)
        assert np.array_equal(lst[0], poses[1] if present[1] else np.identity(4)[:3])


# ------------------------------------------------------------------------------------------ graphed
@pytest.mark.parametrize("dataset", ["ycb", "linemod"])
def test_graphed_equals_eager(cuda, models, dataset):
    """Three batches replayed in turn, against estimate_poses; LineMOD with one camera matrix per frame."""
    model = models[dataset]
    per_frame = dataset == "linemod"
    seq = [_batch(s, dataset, cuda, per_frame_K=per_frame)[0] for s in ((51, 52), (53, 54), (55, 56))]
    kw = _kw(dataset)
    step = F.GraphedPoseStep(model, seq[0], seed=4, **kw)
    for i in (0, 1, 2, 1):
        n0 = _lib.launch_count()
        got = _clone(step(seq[i]))
        assert _lib.launch_count() == n0, "a replay called the library"
        want = F.estimate_poses(model, seq[i], seed=4, **kw)
        _assert_out_equal(got, want, "%s batch %d" % (dataset, i))
    assert step.captures == 1


def test_new_weights_and_switches(cuda, models):
    """load_state_dict of other weights: the next replay equals eager with them, from the same capture; switching
    fused_image_head captures again."""
    model = FFB6D(n_classes=22, n_pts=N, n_kps=N_KPS).to(cuda).eval()
    model.load_state_dict(models["ycb"].state_dict())
    seq = [_batch(s, "ycb", cuda)[0] for s in ((61, 62), (63, 64))]
    kw = _kw("ycb")
    step = F.GraphedPoseStep(model, seq[0], warmup=1, **kw)
    _assert_out_equal(step(seq[0]), F.estimate_poses(model, seq[0], **kw), "before")
    torch.manual_seed(1)
    other = FFB6D(n_classes=22, n_pts=N, n_kps=N_KPS).eval()
    with torch.no_grad():
        for m in other.modules():
            if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
                m.running_mean.uniform_(-0.1, 0.1)
                m.running_var.uniform_(0.5, 1.5)
    model.load_state_dict(other.state_dict())
    got = _clone(step(seq[1]))
    want = F.estimate_poses(model, seq[1], **kw)
    _assert_out_equal(got, want, "after load_state_dict")
    assert step.captures == 1
    model.fused_image_head = True
    _assert_out_equal(_clone(step(seq[0])), F.estimate_poses(model, seq[0], **kw), "fused_image_head")
    assert step.captures == 2


def test_frame_without_depth(cuda, models):
    model = models["ycb"]
    frames = _batch((71, 72), "ycb", cuda)[0]
    kw = _kw("ycb")
    step = F.GraphedPoseStep(model, frames, warmup=1, **kw)
    before = _clone(step(frames))
    assert before["valid"].tolist() == [True, True]
    holed = dict(frames, dpt=frames["dpt"].clone())
    holed["dpt"][1] = 0
    after = _clone(step(holed))
    torch.cuda.synchronize()
    assert after["valid"].tolist() == [True, False]
    for k in OUT_KEYS:
        assert torch.equal(after[k][0], before[k][0]), k
    _assert_out_equal(after, F.estimate_poses(model, holed, **kw), "frame 1 without depth")
    assert step.captures == 1


def test_rejected_frames(cuda, models):
    model = models["linemod"]
    frames = _batch((81, 82), "linemod", cuda)[0]
    kw = _kw("linemod")
    step = F.GraphedPoseStep(model, frames, warmup=1, **kw)
    bad = [({k: v for k, v in frames.items() if k != "rgb"}, "keys"),
           (dict(frames, K=torch.from_numpy(np.stack([K_OF["linemod"]] * 2)).to(cuda)), "keys"),
           (dict(frames, dpt=frames["dpt"][:1]), "captured for"),
           (dict(frames, nrm_map=frames["nrm_map"].double()), "captured for"),
           (dict(frames, rgb=frames["rgb"][:, :240]), "captured for"),
           (dict(frames, dpt=frames["dpt"].cpu()), "captured for")]
    for f, what in bad:
        with pytest.raises(ValueError, match="GraphedPoseStep: .*" + what):
            step(f)
    assert step.captures == 1
    _assert_out_equal(_clone(step(frames)), F.estimate_poses(model, frames, **kw), "after the rejections")
    model.train()
    with pytest.raises(ValueError, match="training mode"):
        step(frames)
    with pytest.raises(ValueError, match="training mode"):
        F.GraphedPoseStep(model, frames, **kw)
    model.eval()
    torch.cuda.synchronize()
