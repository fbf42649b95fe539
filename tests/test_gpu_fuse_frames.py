"""GPU: LineMOD training batches with fused frames (DESIGN.md §4.34).  ``build_ffb6d_train_item(..., crops=)`` equals
``fuse_rgbd(out=...)`` into copies of the images followed by today's call without the fuse keys, and leaves the
caller's tensors as they were; a batch mixing real, rendered and fused frames equals render, then fuse, then the plain
call; a ``GraphedFrameTrainStep(..., crops=)`` replay equals that eager composition plus a training step, bit for
bit, with no host synchronisation, reading new draws at every call without capturing again; on a fused frame the
sampled target points have their source pixels' camera-frame points; and the refusals."""
import copy

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200.fuse_frames import FUSE_KEYS, FuseCropTable, draw_fuse_frame, unfused_keys
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.render import RENDER_KEYS, RenderMeshTable
from frame_batches import CAM_SCALE, make_train_batch
from test_fuse_abi import _mesh_table, _table, refusal_cases
from test_gpu_render import K_SMALL, ape, pose

pytestmark = pytest.mark.gpu

B, H, W, N, N_KPS = 4, 120, 160, 4096, 8
KW = dict(dataset="linemod", cam_scale=CAM_SCALE["linemod"], K=K_SMALL, n_points=N, normals="device")


def _bits(t):
    return t.contiguous().view(torch.uint8)


def source_frames(n=6, seed=0):
    """Decoded-frame stand-ins at the batch's size: the ape rendered at seeded poses over a random background, two
    classes."""
    rs = np.random.RandomState(seed)
    mesh = RenderMeshTable([ape()])
    RTs = np.stack([pose(rs, rs.uniform(0.35, 0.6), 0.03) for _ in range(n)])[:, None]
    out = tuple(torch.zeros(s, dtype=d, device="cuda") for s, d in (((n, H, W), torch.uint16),
                                                                      ((n, H, W, 3), torch.uint8),
                                                                      ((n, H, W), torch.uint8)))
    F.render_rgbd(mesh, np.zeros((n, 1), np.int32), RTs, np.full((n, 1), 255, np.uint8), K_SMALL, H, W, out=out)
    dpt, rgb, lab = (t.cpu().numpy() for t in out)
    rgb = np.where(lab[..., None] > 0, rgb, rs.randint(0, 256, (n, H, W, 3)).astype(np.uint8))
    dpt = np.where(lab > 0, dpt, rs.randint(400, 900, (n, H, W)).astype(np.uint16))
    return [(rgb[k], dpt[k], lab[k], 1 + k % 2) for k in range(n)]


@pytest.fixture(scope="module")
def crops(cuda):
    frames = source_frames()
    return FuseCropTable(frames), frames


def fuse_batch(seed, table, kinds, on_device=False, meshes=False):
    """make_train_batch's LineMOD frames without a normal map, a per-frame K and the fuse keys: frame b is
    ``kinds[b]`` ('real', 'render' or 'fuse'); a fused frame's K is its draw's.  Returns the batch and, per fused
    frame, the target's crop index."""
    batch = make_train_batch(seed, "linemod", B, H, W, 2)
    del batch["nrm_map"]
    rs = np.random.RandomState(seed)
    rows, Ks, targets = [], [], {}
    for b, kind in enumerate(kinds):
        if kind == "fuse":
            keys, K_f, targets[b] = draw_fuse_frame(rs, table.meta, 1 + b % 2, K_SMALL, H, W)
        else:
            keys, K_f = unfused_keys(table.meta), K_SMALL
        rows.append(keys)
        Ks.append(K_f)
    keys = {k: torch.from_numpy(np.stack([np.asarray(r[k]) for r in rows])) for k in FUSE_KEYS}
    keys["K"] = torch.from_numpy(np.stack(Ks).astype(np.float64))
    if meshes:
        keys.update(rendered=torch.tensor([k == "render" for k in kinds]),
                    render_mesh=torch.zeros((B, 1), dtype=torch.int32),
                    render_RTs=torch.from_numpy(np.stack([pose(rs, rs.uniform(0.35, 0.6), 0.03)
                                                          for _ in range(B)])[:, None]),
                    render_label=torch.ones((B, 1), dtype=torch.uint8))
    batch.update({k: v.cuda() if on_device else v for k, v in keys.items()})
    return batch, targets


def composed(batch, table, seed, meshes=None):
    """The eager composition: render (with meshes), then fuse into copies, then today's build_ffb6d_train_item on a
    batch without the render and fuse keys."""
    out = tuple(batch[k].clone() for k in ("dpt", "rgb", "labels"))
    Kd = batch["K"].cpu().numpy()
    if meshes is not None:
        F.render_rgbd(meshes, batch["render_mesh"], batch["render_RTs"], batch["render_label"], Kd, H, W,
                      active=batch["rendered"], out=out)
    F.fuse_rgbd(table, batch["fuse_crop"], batch["fuse_offset"], batch["fuse_label"], H, W, active=batch["fused"],
                out=out)
    plain = {k: v for k, v in batch.items() if k not in FUSE_KEYS + RENDER_KEYS}
    plain.update(dpt=out[0], rgb=out[1], labels=out[2])
    return F.build_ffb6d_train_item(plain, seed=seed, **KW), out


@pytest.mark.parametrize("on_device", [False, True])
def test_train_item_equals_fuse_then_train_item(crops, on_device):
    table = crops[0]
    batch, _ = fuse_batch(3, table, ("real", "fuse", "fuse", "real"), on_device)
    before = {k: batch[k].clone() for k in ("dpt", "rgb", "labels")}
    want, out = composed(batch, table, 11)
    for b in range(B):
        assert torch.equal(out[0][b], before["dpt"][b]) != bool(batch["fused"][b]), b
    for seed in (11, torch.tensor([11], device="cuda")):
        got = F.build_ffb6d_train_item(batch, seed=seed, crops=table, **KW)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and torch.equal(_bits(got[k]), _bits(want[k])), k
    assert all(torch.equal(batch[k], before[k]) for k in before)        # the caller's tensors are not written


def test_mixed_batch_equals_render_then_fuse_then_plain(crops):
    table = crops[0]
    meshes = RenderMeshTable([ape()])
    batch, _ = fuse_batch(4, table, ("render", "fuse", "real", "fuse"), meshes=True)
    before = {k: batch[k].clone() for k in ("dpt", "rgb", "labels")}
    want, out = composed(batch, table, 12, meshes)
    assert (out[2][0] == 1).sum() > 200                                  # the render drew the ape
    got = F.build_ffb6d_train_item(batch, seed=12, crops=table, meshes=meshes, **KW)
    for k in want:
        assert got[k].dtype == want[k].dtype and torch.equal(_bits(got[k]), _bits(want[k])), k
    assert all(torch.equal(batch[k], before[k]) for k in before)


def test_fused_target_points_are_their_source_points(crops):
    """No augmentation: every sampled point labelled 1 on a fused frame is its source pixel's camera-frame point (to
    float32 rounding), so its offset targets are those of the source frame's pose."""
    table, frames = crops
    batch, targets = fuse_batch(5, table, ("fuse", "fuse", "fuse", "real"))
    batch.update(jittered=torch.zeros(B, dtype=torch.bool), augment=torch.zeros(B, dtype=torch.bool))
    batch["labels"][:3] = 0          # a worker sends no labels for a fused frame: the crops bring them
    item = F.build_ffb6d_train_item(batch, seed=3, crops=table, **KW)
    choose = item["choose"].reshape(B, -1).cpu().numpy()
    xyz = item["cld_rgb_nrm"][:, :3].cpu().numpy()
    lab = item["labels"].cpu().numpy()
    ctr_ofst = item["ctr_targ_ofst"].cpu().numpy()
    obj_ctr = batch["obj_ctr"].cpu().numpy()
    n_checked = 0
    for b, tk in targets.items():
        s = int(np.flatnonzero(batch["fuse_label"][b].numpy())[0])
        row, col = batch["fuse_offset"][b, s].tolist()
        r0, c0 = table.origin[tk]
        pts = np.flatnonzero(lab[b] == 1)
        assert pts.size > 50
        r, c = choose[b, pts] // W, choose[b, pts] % W
        rs_, cs_ = r - row + r0, c - col + c0
        src = frames[tk]
        assert (src[2][rs_, cs_] != 0).all()
        z = src[1][rs_, cs_].astype(np.float64) / 1000.0
        want = np.stack([(cs_ - K_SMALL[0, 2]) * z / K_SMALL[0, 0], (rs_ - K_SMALL[1, 2]) * z / K_SMALL[1, 1], z])
        assert np.abs(xyz[b][:, pts] - want).max() <= 4e-7 * max(1.0, np.abs(want).max()), b
        assert np.abs(ctr_ofst[b, pts] - (want.T - obj_ctr[b, 0])).max() <= 2e-6, b       # the cloud minus the centre
        n_checked += pts.size
    assert n_checked > 150


def deterministic(on):
    torch.use_deterministic_algorithms(on)
    torch.backends.cudnn.deterministic = on


def make_model():
    torch.manual_seed(3)
    model = F.model.FFB6D(n_classes=2, n_pts=N, n_kps=N_KPS, fused_image_head=True).cuda()
    for m in model.modules():
        if isinstance(m, torch.nn.modules.dropout._DropoutNd):
            m.p = 0.0
    return model.train()


def adam(model):
    return torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-3, device="cuda"), capturable=True)


def eager_step(model, opt, batch, table, seed, meshes):
    item, _ = composed(batch, table, seed, meshes)
    opt.zero_grad(set_to_none=True)
    loss, info = ffb6d_loss(model(item), item, valid=item["valid"])
    loss.backward()
    opt.step()
    return loss.detach(), info


def test_graphed_equals_eager_and_reads_new_draws(crops):
    table = crops[0]
    meshes = RenderMeshTable([ape()])
    kinds = (("render", "fuse", "real", "fuse"), ("fuse", "real", "fuse", "render"), ("fuse", "fuse", "render", "real"))
    seq = [fuse_batch(s, table, k, meshes=True)[0] for s, k in zip((21, 22, 23), kinds)]
    assert not torch.equal(seq[1]["fuse_offset"], seq[2]["fuse_offset"])
    seeds = (5, 6, 7)
    deterministic(True)
    try:
        model = make_model()
        twin = copy.deepcopy(model)
        opt, opt_e = adam(model), adam(twin)
        step = F.GraphedFrameTrainStep(model, opt, seq[0], warmup=2, meshes=meshes, crops=table, **KW)
        for i, (batch, seed) in enumerate(zip(seq, seeds)):
            before = {k: batch[k].clone() for k in ("dpt", "rgb", "labels")}
            if i:
                torch.cuda.set_sync_debug_mode("error")
            try:
                loss, info = step(batch, seed=seed)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            loss_e, info_e = eager_step(twin, opt_e, batch, table, seed, meshes)
            assert torch.equal(loss, loss_e), "step %d: loss" % i
            assert all(torch.equal(info[k], info_e[k]) for k in info_e), "step %d: info" % i
            diff = sum(not torch.equal(a, b) for a, b in zip(model.parameters(), twin.parameters()))
            assert diff == 0, "step %d: %d parameters differ" % (i, diff)
            assert all(torch.equal(batch[k], before[k]) for k in before)
            assert step.captures == 1
    finally:
        deterministic(False)


def test_refusals(crops):
    table = crops[0]
    seq = [fuse_batch(s, table, ("real", "fuse", "fuse", "real"))[0] for s in (31, 32)]
    model = make_model()
    step = F.GraphedFrameTrainStep(model, adam(model), seq[0], warmup=1, crops=table, **KW)
    for bad, what in ((dict(seq[1], fuse_crop=torch.full((B, 2), len(table), dtype=torch.int32)), "crop indices"),
                      (dict(seq[1], fuse_offset=torch.zeros((B, 2, 2), dtype=torch.int64)), "fuse_offset"),
                      (dict(seq[1], fused=torch.zeros(B, dtype=torch.uint8)), r"batch\['fused'\]")):
        with pytest.raises(ValueError, match=what):
            step(bad, seed=1)
    loss, _ = step(seq[1], seed=1)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item() and step.captures == 1
    # every refusal of the host checks, here with a CUDA device present
    for args, what in refusal_cases(_table(), _mesh_table()):
        batch, dataset, tab = args[:3]
        normals = args[3] if len(args) > 3 else "device"
        meshes = args[4] if len(args) > 4 else None
        with pytest.raises(ValueError, match=what):
            F.build_ffb6d_train_item(batch, dataset=dataset, cam_scale=1e3, K=np.eye(3), n_points=64, seed=0,
                                     crops=tab, normals=normals, meshes=meshes)
