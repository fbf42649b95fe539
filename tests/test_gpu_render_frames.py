"""GPU: LineMOD training batches that mix decoded and rendered frames (DESIGN.md §4.31).  ``build_ffb6d_train_item(...,
meshes=)`` equals ``render_rgbd(out=...)`` into copies of the images followed by today's ``build_ffb6d_train_item``,
and leaves the caller's tensors as they were; a ``GraphedFrameTrainStep(..., meshes=)`` replay equals that eager
composition plus a training step, bit for bit, with no host synchronisation, and reads new poses at every call
without capturing again."""
import copy

import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D
from ffb6d_b200.render import RENDER_KEYS, RenderMeshTable
from frame_batches import CAM_SCALE, make_train_batch
from test_gpu_render import K_SMALL, ape, pose

pytestmark = pytest.mark.gpu

B, H, W, N, N_KPS = 4, 120, 160, 4096, 8
# a rendered frame's normals come from its own depth, on the device (meshes= refuses normals="input")
KW = dict(dataset="linemod", cam_scale=CAM_SCALE["linemod"], K=K_SMALL, n_points=N, normals="device")


def _bits(t):
    return t.contiguous().view(torch.uint8)


def render_batch(seed, on_device=False):
    """make_train_batch's LineMOD frames without a normal map, frames 0 and 2 flagged as renders of the ape at a seeded
    pose."""
    batch = make_train_batch(seed, "linemod", B, H, W, 2)
    del batch["nrm_map"]
    rs = np.random.RandomState(seed)
    keys = dict(rendered=torch.tensor([True, False, True, False]),
                render_mesh=torch.zeros((B, 1), dtype=torch.int32),
                render_RTs=torch.from_numpy(np.stack([pose(rs, rs.uniform(0.35, 0.6), 0.03) for _ in range(B)])[:, None]),
                render_label=torch.ones((B, 1), dtype=torch.uint8))
    batch.update({k: v.cuda() if on_device else v for k, v in keys.items()})
    return batch


def composed(batch, table, seed):
    """The eager composition: render into copies, then today's build_ffb6d_train_item on a batch without the keys (its
    normals="device" computes every frame's normals from its composed depth, the rendered frames' from the render)."""
    out = tuple(batch[k].clone() for k in ("dpt", "rgb", "labels"))
    F.render_rgbd(table, batch["render_mesh"], batch["render_RTs"], batch["render_label"], K_SMALL, H, W,
                  active=batch["rendered"], out=out)
    plain = {k: v for k, v in batch.items() if k not in RENDER_KEYS}
    plain.update(dpt=out[0], rgb=out[1], labels=out[2])
    return F.build_ffb6d_train_item(plain, seed=seed, **KW), out


@pytest.mark.parametrize("on_device", [False, True])
def test_train_item_equals_render_then_train_item(cuda, on_device):
    table = RenderMeshTable([ape()])
    batch = render_batch(3, on_device)
    before = {k: batch[k].clone() for k in ("dpt", "rgb", "labels")}
    want, out = composed(batch, table, 11)
    # the flagged frames are renders (the ape is in view), the others the decoded frames
    for b in range(B):
        same = torch.equal(out[0][b], before["dpt"][b])
        assert same != bool(batch["rendered"][b]), b
        if batch["rendered"][b]:
            assert (out[2][b] == 1).sum() > 200 and torch.equal(out[2][b] == 1, out[0][b].to(torch.int32) > 0)
    for seed in (11, torch.tensor([11], device="cuda")):
        got = F.build_ffb6d_train_item(batch, seed=seed, meshes=table, **KW)
        assert sorted(got) == sorted(want)
        for k in want:
            assert got[k].dtype == want[k].dtype and torch.equal(_bits(got[k]), _bits(want[k])), k
    assert all(torch.equal(batch[k], before[k]) for k in before)        # the caller's tensors are not written


def deterministic(on):
    torch.use_deterministic_algorithms(on)
    torch.backends.cudnn.deterministic = on


def make_model():
    torch.manual_seed(3)
    model = FFB6D(n_classes=2, n_pts=N, n_kps=N_KPS, fused_image_head=True).cuda()
    for m in model.modules():
        if isinstance(m, torch.nn.modules.dropout._DropoutNd):
            m.p = 0.0
    return model.train()


def adam(model):
    return torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-3, device="cuda"), capturable=True)


def eager_step(model, opt, batch, table, seed):
    item, _ = composed(batch, table, seed)
    opt.zero_grad(set_to_none=True)
    loss, info = ffb6d_loss(model(item), item, valid=item["valid"])
    loss.backward()
    opt.step()
    return loss.detach(), info


def test_graphed_equals_eager_and_reads_new_poses(cuda):
    table = RenderMeshTable([ape()])
    seq = [render_batch(s) for s in (21, 22, 23)]
    assert not torch.equal(seq[1]["render_RTs"], seq[2]["render_RTs"])
    seeds = (5, 6, 7)
    deterministic(True)
    try:
        model = make_model()
        twin = copy.deepcopy(model)
        opt, opt_e = adam(model), adam(twin)
        step = F.GraphedFrameTrainStep(model, opt, seq[0], warmup=2, meshes=table, **KW)
        for i, (batch, seed) in enumerate(zip(seq, seeds)):
            before = {k: batch[k].clone() for k in ("dpt", "rgb", "labels")}
            if i:
                torch.cuda.set_sync_debug_mode("error")
            try:
                loss, info = step(batch, seed=seed)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            loss_e, info_e = eager_step(twin, opt_e, batch, table, seed)
            assert torch.equal(loss, loss_e), "step %d: loss" % i
            assert all(torch.equal(info[k], info_e[k]) for k in info_e), "step %d: info" % i
            diff = sum(not torch.equal(a, b) for a, b in zip(model.parameters(), twin.parameters()))
            assert diff == 0, "step %d: %d parameters differ" % (i, diff)
            assert all(torch.equal(batch[k], before[k]) for k in before)
            assert step.captures == 1
    finally:
        deterministic(False)


def test_graphed_step_refuses_bad_host_indices(cuda):
    table = RenderMeshTable([ape()])
    seq = [render_batch(s) for s in (31, 32)]
    model = make_model()
    step = F.GraphedFrameTrainStep(model, adam(model), seq[0], warmup=1, meshes=table, **KW)
    bad = dict(seq[1], render_mesh=torch.full((B, 1), 1, dtype=torch.int32))
    with pytest.raises(ValueError, match="mesh indices"):
        step(bad, seed=1)
    loss, _ = step(seq[1], seed=1)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item() and step.captures == 1
