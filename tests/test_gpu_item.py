"""GPU: the sampled points' input features and pose targets (ffb6d_point_item / ops.point_item) bitwise against the
reference's outputs in tests/golden/item_cases.npz and against the numpy oracle on seeded frames; the batch get_item
(schedule.build_ffb6d_item) against its explicit composition, with the frames it must flag invalid; determinism,
CUDA-graph replay, and the item feeding FFB6DFusionNet."""
import os

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from conftest import GOLDEN, _npz_groups
from oracle import item_oracle as O
from ffb6d_b200.item import pose_gt_objects
from ffb6d_b200.synthetic import INTRINSICS, item_test_frames, make_item_frame
from test_item_oracle import POINT_KEYS, assert_bitwise, assert_point_outputs, dpt_m_of, objects_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return _npz_groups(os.path.join(GOLDEN, "item_cases.npz"))


def to_dev(a, cuda):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def device_args(frames, objs, chooses, cuda, choose_dtype=torch.int32, choose_2d=False):
    """Stack per-frame numpy inputs into the CUDA tensors ops.point_item takes (K per frame)."""
    ch = to_dev(np.stack(chooses).astype(np.int64), cuda).to(choose_dtype)
    if not choose_2d:
        ch = ch[:, None, :]
    return dict(depth_m=to_dev(np.stack([dpt_m_of(f) for f in frames]), cuda),
                K=np.stack([np.asarray(f["K"], np.float64) for f in frames]), choose=ch,
                rgb=to_dev(np.stack([f["rgb"] for f in frames]), cuda),
                labels=to_dev(np.stack([f["labels"] for f in frames]), cuda),
                nrm_map=to_dev(np.stack([f["nrm"] for f in frames]), cuda),
                obj_cls=to_dev(np.stack([o["obj_cls"] for o in objs]), cuda),
                obj_kps=to_dev(np.stack([o["obj_kps"] for o in objs]), cuda),
                obj_ctr=to_dev(np.stack([o["obj_ctr"] for o in objs]), cuda))


def host(outs):
    return [o.cpu().numpy() for o in outs]


def assert_matches_oracle(got, frames, objs, chooses):
    for b, (f, o, ch) in enumerate(zip(frames, objs, chooses)):
        want = O.point_item(dpt_m_of(f), f["K"], ch, f["rgb"], f["labels"], f["nrm"], o["obj_cls"], o["obj_kps"],
                            o["obj_ctr"])
        for k, g, w in zip(POINT_KEYS, got, want):
            assert_bitwise(g[b], w, "frame %d %s" % (b, k))


@pytest.mark.parametrize("name", sorted(item_test_frames()))
@pytest.mark.parametrize("choose_dtype,choose_2d", [(torch.int32, False), (torch.int64, True)])
def test_golden_frames_bitwise(cuda, golden, name, choose_dtype, choose_2d):
    frame, dataset, n_points, n_objects = item_test_frames()[name]
    g, obj = golden[name], objects_of(frame, dataset, n_objects)
    args = device_args([frame], [obj], [g["choose"]], cuda, choose_dtype, choose_2d)
    got = host(F.point_item(**args))
    assert_point_outputs({k: v[0] for k, v in zip(POINT_KEYS, got)}, g, name)


def _seeded_batch(B, h, w, n_points, n_kps, seed, dataset="ycb", nrm_dtype=np.float32):
    frames, objs, chooses = [], [], []
    for b in range(B):
        if dataset == "ycb":
            f = make_item_frame(seed + b, h=h, w=w, n_kps=n_kps, cls_ids=(1 + b % 5, 6, 1 + b % 5, 21),
                                blobs=(1 + b % 5, 6, 12), hole_frac=0.1 + 0.3 * (b % 2), nrm_dtype=nrm_dtype,
                                intrinsics=("ycb_K1", "ycb_K2")[b % 2])
            o = pose_gt_objects(f["poses"], f["cls_ids"], f["kps"], f["ctrs"], 22, n_kps)
        else:
            f = make_item_frame(seed + b, h=h, w=w, dataset="linemod", n_kps=n_kps, cls_ids=(1,), blobs=(1,),
                                nrm_dtype=nrm_dtype)
            o = pose_gt_objects(f["poses"], [1], f["kps"], f["ctrs"], 2, n_kps, dataset="linemod")
        np.random.seed(seed + b)
        frames.append(f)
        objs.append(o)
        chooses.append(O.sample_choose(f["raw"] > 0, n_points))
    return frames, objs, chooses


@pytest.mark.parametrize("B,h,w,n_points,n_kps,dataset,nrm_dtype", [
    (3, 480, 640, 12288, 8, "ycb", np.float32),
    (2, 480, 640, 12288, 16, "linemod", np.float64),
    (4, 37, 53, 1500, 16, "ycb", np.float64),          # n_valid < N on the odd frames: 'wrap' padding
    (2, 24, 24, 129, 1, "linemod", np.float32),
    (32, 480, 640, 12288, 8, "ycb", np.float32),
])
def test_seeded_batches_match_oracle(cuda, B, h, w, n_points, n_kps, dataset, nrm_dtype):
    frames, objs, chooses = _seeded_batch(B, h, w, n_points, n_kps, 50 * B + n_kps, dataset, nrm_dtype)
    args = device_args(frames, objs, chooses, cuda)
    got = host(F.point_item(**args))
    assert_matches_oracle(got, frames, objs, chooses)
    # channels 0-2 are ops.backproject's cloud, bitwise
    if h % 8 == 0 and w % 8 == 0:
        cld, _ = F.backproject(args["depth_m"], args["K"], args["choose"])
        assert torch.equal(torch.from_numpy(got[0][:, :3]).view(torch.int32),
                           cld.transpose(1, 2).cpu().view(torch.int32))


def test_background_and_padding_never_match(cuda):
    """Background label 0 with padding slots (-1), and an obj_cls of 0 in a slot: only the latter matches 0."""
    frames, objs, chooses = _seeded_batch(2, 24, 32, 300, 8, 7)
    args = device_args(frames, objs, chooses, cuda)
    kp = F.point_item(**args)[2].cpu().numpy()
    lab = args["labels"].cpu().numpy().reshape(2, -1)[np.arange(2)[:, None], np.stack(chooses)]
    assert (lab == 0).any() and (kp[lab == 0] == 0).all()
    assert not np.signbit(kp[lab == 0]).any()                                        # +0.0
    objs[1]["obj_cls"][5] = 0
    args = device_args(frames, objs, chooses, cuda)
    got = host(F.point_item(**args))
    assert_matches_oracle(got, frames, objs, chooses)
    assert (got[2][1][lab[1] == 0] != 0).any()


def test_runs_and_graph_replays_bitwise(cuda):
    from ffb6d_b200.ops import intrinsics_to_device
    frames, objs, chooses = _seeded_batch(4, 480, 640, 12288, 16, 3)
    args = device_args(frames, objs, chooses, cuda)
    args["K"] = intrinsics_to_device(args["K"], cuda)
    a = F.point_item(**args)
    b = F.point_item(**args)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    side = torch.cuda.Stream(device=cuda)
    side.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(side):
        F.point_item(**args)
    torch.cuda.current_stream(cuda).wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = F.point_item(**args)
    for _ in range(2):
        for t in got:
            t.fill_(-7)
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(got, a):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def _item_inputs(frames, objs, cuda):
    return dict(dpt=to_dev(np.stack([f["raw"] for f in frames]), cuda),
                rgb=to_dev(np.stack([f["rgb"] for f in frames]), cuda),
                labels=to_dev(np.stack([f["labels"] for f in frames]), cuda),
                nrm_map=to_dev(np.stack([f["nrm"] for f in frames]), cuda), objects=objs)


ITEM_KEYS = {"rgb", "cld_rgb_nrm", "choose", "labels", "rgb_labels", "dpt_map_m", "RTs", "kp_targ_ofst",
             "ctr_targ_ofst", "cls_ids", "ctr_3ds", "kp_3ds", "valid"}


def test_build_item_ycb_equals_composition(cuda):
    from ffb6d_b200.ops import _fill_depth
    frames, objs, _ = _seeded_batch(3, 480, 640, 12288, 8, 11)
    frames[2]["raw"][:] = 0                                                          # n_valid = 0
    K = INTRINSICS["ycb_K1"]
    x = _item_inputs(frames, objs, cuda)
    item = F.build_ffb6d_item(x["dpt"], 10000.0, K, x["rgb"], x["labels"], x["nrm_map"], objs, 12288, seed=5)
    assert ITEM_KEYS <= set(item) and "cld_nei_idx0" in item and "p2r_up_nei_idx2" in item
    filled, depth_m = _fill_depth(x["dpt"], 10000.0)
    choose, count = F.sample_valid_pixels(filled, 12288, seed=5, min_depth=1e-6, return_count=True)
    want = F.build_ffb6d_indices_from_depth(depth_m, K, choose)
    o = {k: torch.from_numpy(np.stack([ob[k] for ob in objs])).to(cuda) for k in ("obj_cls", "obj_kps", "obj_ctr")}
    pts = F.point_item(depth_m, K, choose, x["rgb"], x["labels"], x["nrm_map"], o["obj_cls"], o["obj_kps"], o["obj_ctr"])
    want.update(dict(zip(POINT_KEYS, pts)), choose=choose, dpt_map_m=depth_m)
    for key, w in want.items():
        assert item[key].dtype == w.dtype and torch.equal(item[key], w), key
    assert item["valid"].tolist() == [True, True, False] and count[2].item() == 0
    assert torch.equal(item["rgb"], x["rgb"].permute(0, 3, 1, 2))
    assert item["rgb"].shape == (3, 3, 480, 640) and item["rgb"].dtype == torch.uint8
    assert torch.equal(item["rgb_labels"], x["labels"].to(torch.int32))
    for k in ("RTs", "kp_3ds", "ctr_3ds", "cls_ids"):
        assert np.array_equal(item[k].cpu().numpy(), np.stack([ob[k] for ob in objs])), k


def test_build_item_linemod_against_oracle(cuda):
    """fill=False: dpt_m = dpt_mm / 1000 in float32, msk_dp = dpt_mm > 0; frames with n_valid < N ('wrap'),
    n_valid < 400 and n_valid = 0."""
    frames, objs, _ = _seeded_batch(4, 480, 640, 12288, 16, 21, dataset="linemod")
    rs = np.random.RandomState(0)
    for b, n_keep in ((1, 5000), (2, 399), (3, 0)):
        raw = frames[b]["raw"]
        keep = rs.choice(np.flatnonzero(raw), n_keep, replace=False)
        sparse = np.zeros_like(raw).reshape(-1)
        sparse[keep] = raw.reshape(-1)[keep]
        frames[b]["raw"] = sparse.reshape(raw.shape)
    x = _item_inputs(frames, objs, cuda)
    K = INTRINSICS["linemod"]
    item = F.build_ffb6d_item(x["dpt"], 1000.0, K, x["rgb"], x["labels"], x["nrm_map"], objs, 12288, seed=2,
                              fill=False)
    assert item["valid"].tolist() == [True, True, False, False]
    for b, f in enumerate(frames):
        want_m = f["raw"].astype(np.float32) / 1000.0
        assert_bitwise(item["dpt_map_m"][b].cpu().numpy(), want_m, "dpt_map_m")
    choose = item["choose"][:, 0].cpu().numpy()
    for b in (1, 2):                                                                 # every valid pixel, 'wrap'
        assert set(choose[b].tolist()) == set(np.flatnonzero(frames[b]["raw"]).tolist())
    assert (choose[3] == 0).all()
    got = host([item[k] for k in POINT_KEYS])
    assert_matches_oracle(got, frames, objs, list(choose))


@pytest.mark.parametrize("n_classes", [22, 2])
def test_item_feeds_the_network(cuda, n_classes):
    from ffb6d_b200.model import FFB6DFusionNet
    dataset = "ycb" if n_classes == 22 else "linemod"
    frames, objs, _ = _seeded_batch(2, 480, 640, 12288, 8, 31, dataset=dataset)
    x = _item_inputs(frames, objs, cuda)
    K = INTRINSICS["ycb_K1" if dataset == "ycb" else "linemod"]
    item = F.build_ffb6d_item(x["dpt"], 10000.0 if dataset == "ycb" else 1000.0, K, x["rgb"], x["labels"],
                              x["nrm_map"], objs, 12288, fill=dataset == "ycb")
    torch.manual_seed(0)
    model = FFB6DFusionNet(n_classes=n_classes).to(cuda).eval()
    g = torch.Generator(device=cuda).manual_seed(0)
    feats = [torch.randn(s, generator=g, device=cuda) for s in FFB6DFusionNet.rgb_feature_shapes(2)]
    with torch.no_grad():
        out = model(item, rgb_feats=feats)
    assert out["pred_rgbd_segs"].shape == (2, n_classes, 12288)
    assert out["pred_kp_ofs"].shape == (2, 8) + tuple(item["kp_targ_ofst"].shape[1:2]) + (3,)
    assert out["pred_kp_ofs"].transpose(1, 2).shape == item["kp_targ_ofst"].shape
    assert out["pred_ctr_ofs"].shape[2:] == item["ctr_targ_ofst"].shape[1:]
    for v in (out["pred_rgbd_segs"], out["pred_kp_ofs"], out["pred_ctr_ofs"]):
        assert torch.isfinite(v).all()
