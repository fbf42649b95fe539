"""GPU: ``fuse_rgbd`` (``ffb6d_fuse_rgbd``, DESIGN.md §4.34) equals oracle/fuse_oracle.py bit for bit: 13-slot
480x640 frames whose crops come from renders of the golden ape at seeded poses (stand-ins for decoded real frames),
overlapping, partly outside and empty slots, extreme offsets, device indices outside the table, inactive frames,
``out=`` over a background, 1x1 and odd sizes, ``B = 0``, and one call at each checked limit."""
import numpy as np
import pytest
import torch

import ffb6d_b200 as F
from ffb6d_b200 import _lib
from ffb6d_b200.fuse_frames import FuseCropTable, draw_fuse_frame
from ffb6d_b200.render import RenderMeshTable
from oracle import fuse_oracle as O
from test_gpu_render import ape, pose

pytestmark = pytest.mark.gpu

H, W = 480, 640
K_LM = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
N_CLS = 13


def ape_frames(n, seed):
    """n decoded-frame stand-ins: the ape rendered at seeded poses, its mask 255, class k % 13 + 1."""
    rs = np.random.RandomState(seed)
    mesh = RenderMeshTable([ape()])
    RTs = np.stack([pose(rs, rs.uniform(0.3, 0.9), 0.08) for _ in range(n)])[:, None]
    dpt = torch.zeros((n, H, W), dtype=torch.uint16, device="cuda")
    rgb = torch.zeros((n, H, W, 3), dtype=torch.uint8, device="cuda")
    lab = torch.zeros((n, H, W), dtype=torch.uint8, device="cuda")
    F.render_rgbd(mesh, np.zeros((n, 1), np.int32), RTs, np.full((n, 1), 255, np.uint8), K_LM, H, W,
                  out=(dpt, rgb, lab))
    dpt, rgb, lab = dpt.cpu().numpy(), rgb.cpu().numpy(), lab.cpu().numpy()
    # real frames have a background: give the stand-ins one, which the crops must leave behind
    bg = rs.randint(0, 256, (n, H, W, 3)).astype(np.uint8)
    rgb = np.where(lab[..., None] > 0, rgb, bg)
    dpt = np.where(lab > 0, dpt, rs.randint(500, 3000, (n, H, W)).astype(np.uint16))
    frames = [(rgb[k], dpt[k], lab[k], k % N_CLS + 1) for k in range(n)]
    assert all((f[2] > 0).sum() > 200 for f in frames)
    return frames


@pytest.fixture(scope="module")
def tables(cuda):
    frames = ape_frames(26, 0)
    return FuseCropTable(frames), [O.crop_frame(*f[:3])[:3] for f in frames], frames


def check(tables, crop, offset, label, h, w, active=None, out=None, device_args=False):
    table, crops, _ = tables
    crop, offset, label = (np.asarray(crop, np.int32), np.asarray(offset, np.int32), np.asarray(label, np.uint8))
    want = O.fuse(crops, crop, offset, label, h, w, active=active,
                  out=None if out is None else tuple(t.cpu().numpy() for t in out))
    args = (crop, offset, label)
    act = active
    if device_args:
        args = tuple(torch.from_numpy(a).cuda() for a in args)
        act = None if active is None else torch.as_tensor(np.asarray(active, bool)).cuda()
    got = F.fuse_rgbd(table, *args, h, w, active=act, out=out)
    if out is not None:
        assert all(g is o for g, o in zip(got, out))
    for g, wnt, name in zip(got, want, ("dpt_mm", "rgb", "labels")):
        g = g.cpu().numpy()
        assert g.dtype == wnt.dtype and g.shape == wnt.shape and np.array_equal(g, wnt), name
    return want


def test_drawn_13_slot_frames(tables):
    table = tables[0]
    rs = np.random.RandomState(1)
    keys = [draw_fuse_frame(rs, table, (b % N_CLS) + 1, K_LM, H, W)[0] for b in range(6)]
    crop = np.stack([k["fuse_crop"] for k in keys])
    offset = np.stack([k["fuse_offset"] for k in keys])
    label = np.stack([k["fuse_label"] for k in keys])
    assert crop.shape == (6, N_CLS)
    for dev in (False, True):
        d, _, l = check(tables, crop, offset, label, H, W, device_args=dev)
    assert all((l[b] == 1).sum() > 0 for b in range(6)) and (d > 0).sum() > 13 * 200


def test_overlap_outside_and_empty_slots(tables):
    rs = np.random.RandomState(2)
    B, M = 5, 16
    crop = rs.randint(-1, 26, (B, M))
    crop[:, 3] = -1
    offset = np.stack([rs.randint(-200, 500, (B, M)), rs.randint(-200, 700, (B, M))], -1)
    offset[0, :4] = [[I32_MIN, 0], [0, I32_MIN], [I32_MAX, I32_MAX], [I32_MIN, I32_MAX]]
    offset[1, :] = [100, 200]                       # every slot at the same corner: the last non-empty one shows
    label = rs.randint(0, 256, (B, M))
    for dev in (False, True):
        check(tables, crop, offset, label, H, W, device_args=dev)


def test_device_indices_outside_the_table_paste_nothing(tables):
    crop = np.array([[26, 9999, I32_MIN, I32_MAX, -5, -1, 0]], np.int32)
    offset = np.zeros((1, 7, 2), np.int32)
    d, _, l = check(tables, crop, offset, np.full((1, 7), 3), H, W, device_args=True)
    assert (l > 0).sum() == tables[1][0][2].sum()            # only slot 6's crop
    with pytest.raises(ValueError, match="crop indices"):
        F.fuse_rgbd(tables[0], crop, offset, np.zeros((1, 7), np.uint8), H, W)      # host values are checked


def test_inactive_frames_and_background(tables):
    rs = np.random.RandomState(3)
    B, M = 4, 13
    crop = rs.randint(0, 26, (B, M))
    offset = np.stack([rs.randint(-50, 400, (B, M)), rs.randint(-50, 560, (B, M))], -1)
    label = rs.randint(1, 4, (B, M))
    for dev in (False, True):
        bg = (torch.from_numpy(rs.randint(0, 65536, (B, H, W)).astype(np.uint16)).cuda(),
              torch.from_numpy(rs.randint(0, 256, (B, H, W, 3)).astype(np.uint8)).cuda(),
              torch.from_numpy(rs.randint(0, 256, (B, H, W)).astype(np.uint8)).cuda())
        before = tuple(t.clone() for t in bg)
        active = [True, False, True, False]
        check(tables, crop, offset, label, H, W, active=active, out=bg, device_args=dev)
        for b in (1, 3):
            assert all(torch.equal(t[b], u[b]) for t, u in zip(bg, before))
        assert not torch.equal(bg[2][0], before[2][0])
    # new outputs start from zeros, inactive frames stay zero
    d, c, l = check(tables, crop, offset, label, H, W, active=[False, True, False, False])
    assert not d[0].any() and not c[2].any() and l[1].any()


@pytest.mark.parametrize("h, w", [(1, 1), (37, 53), (1, 641), (481, 1), (7, 3)])
def test_small_and_odd_sizes(tables, h, w):
    rs = np.random.RandomState(h * 1000 + w)
    B, M = 3, 5
    crop = rs.randint(-1, 26, (B, M))
    offset = np.stack([rs.randint(-300, h + 1, (B, M)), rs.randint(-300, w + 1, (B, M))], -1)
    # one slot per frame whose crop is known to cover pixel (0, 0): its silhouette's first set pixel there
    t0 = tables[1][0][2]
    i, j = np.argwhere(t0)[0]
    crop[:, 0] = 0
    offset[:, 0] = [-i, -j]
    d, _, l = check(tables, crop, offset, rs.randint(1, 9, (B, M)), h, w, device_args=bool(h % 2))
    assert (l[:, 0, 0] > 0).all()


def test_empty_batch(tables):
    d, c, l = F.fuse_rgbd(tables[0], np.zeros((0, 3), np.int32), np.zeros((0, 3, 2), np.int32),
                          np.zeros((0, 3), np.uint8), H, W)
    assert d.shape == (0, H, W) and c.shape == (0, H, W, 3) and l.shape == (0, H, W)


def test_repeatable(tables):
    rs = np.random.RandomState(4)
    crop = torch.from_numpy(rs.randint(0, 26, (8, 13)).astype(np.int32)).cuda()
    offset = torch.from_numpy(rs.randint(-100, 500, (8, 13, 2)).astype(np.int32)).cuda()
    label = torch.from_numpy(rs.randint(0, 5, (8, 13)).astype(np.uint8)).cuda()
    a = F.fuse_rgbd(tables[0], crop, offset, label, H, W)
    b = F.fuse_rgbd(tables[0], crop, offset, label, H, W)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_each_checked_limit_is_admitted(cuda):
    # a 2 x 3 crop with its centre column empty
    sil = np.array([[255, 0, 255], [255, 0, 255]], np.uint8)
    rgb = np.full((2, 3, 3), 7, np.uint8)
    dpt = np.full((2, 3), 1234, np.uint16)
    table = FuseCropTable([(rgb, dpt, sil, 1)])

    def run(B, M, h, w, crop, offset):
        out = (torch.zeros((B, h, w), dtype=torch.uint16, device="cuda"),
               torch.zeros((B, h, w, 3), dtype=torch.uint8, device="cuda"),
               torch.zeros((B, h, w), dtype=torch.uint8, device="cuda"))
        F.fuse_rgbd(table, crop, offset, torch.full((B, M), 9, dtype=torch.uint8, device="cuda"), h, w, out=out)
        return out

    B = _lib.FUSE_MAX_FRAMES
    off = torch.zeros((B, 1, 2), dtype=torch.int32, device="cuda")
    off[1::2, 0, 1] = -1                                  # odd frames see the crop's empty centre column
    d, c, l = run(B, 1, 1, 1, torch.zeros((B, 1), dtype=torch.int32, device="cuda"), off)
    assert (l[0::2] == 9).all() and (d[0::2].to(torch.int32) == 1234).all() and not l[1::2].any()
    del d, c, l
    # the most slots: only the first pastes; every later slot is empty or outside the frame
    M = _lib.FUSE_MAX_SLOTS
    crop = torch.full((1, M), -1, dtype=torch.int32, device="cuda")
    crop[0, 0] = 0
    crop[0, 1::2] = 0
    off = torch.zeros((1, M, 2), dtype=torch.int32, device="cuda")
    off[0, 1::2] = torch.tensor([50, 50], dtype=torch.int32, device="cuda")
    d, c, l = run(1, M, 4, 4, crop, off)
    want = np.zeros((4, 4), np.uint8)
    want[:2, [0, 2]] = 9
    assert np.array_equal(l[0].cpu().numpy(), want) and (c[0][l[0] > 0] == 7).all()
    del d, c, l
    # the most pixels in a frame: the crop pasted at the last three columns
    P = _lib.FUSE_MAX_FRAME_PIXELS
    off = torch.tensor([[[0, P - 3]]], dtype=torch.int32, device="cuda")
    d, c, l = run(1, 1, 1, P, torch.zeros((1, 1), dtype=torch.int32, device="cuda"), off)
    assert l[0, 0, -3:].tolist() == [9, 0, 9] and (l[0, 0, :-3] == 0).all()
    assert d[0, 0, -1].item() == 1234 and c[0, 0, -3].tolist() == [7, 7, 7]
    del d, c, l
    torch.cuda.empty_cache()
