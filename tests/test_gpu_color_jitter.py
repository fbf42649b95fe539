"""GPU: ffb6d_color_jitter / ops.color_jitter against torchvision and Pillow's outputs (tests/golden/jitter_cases.npz)
and the numpy restatement (oracle/jitter_oracle.py)."""
import hashlib
import itertools
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, _npz_groups
import ffb6d_b200 as F
from ffb6d_b200 import augment as A, _lib
from ffb6d_b200.synthetic import make_aug_frame
from oracle import jitter_oracle as JO

pytestmark = pytest.mark.gpu
G = _npz_groups(os.path.join(GOLDEN, "jitter_cases.npz"))
CASES = sorted(k for k, v in G.items() if "plan" in v)


def case_input(c):
    if "rgb" in c:
        return c["rgb"]
    seed, h, w = (int(x) for x in c["meta"])
    return make_aug_frame(seed, h, w)["rgb"]


def random_plans(B, seed):
    """B plans: the 24 orders first, then random ones; blend factors in [0, 2] (both of Image.blend's branches),
    hue anywhere in [-0.5, 0.5]; a few of them exactly as ColorJitter draws them."""
    rs = np.random.RandomState(seed)
    orders = list(itertools.permutations(range(4)))
    p = np.zeros((B, A.JITTER_PLAN_LEN))
    for b in range(B):
        p[b, :4] = orders[b] if b < len(orders) else rs.permutation(4)
        p[b, 4:7] = rs.uniform(0.0, 2.0, 3)
        p[b, 7] = rs.uniform(-0.5, 0.5)
    torch.manual_seed(seed)
    k = min(3, B)
    p[B - k:] = A.draw_color_jitter(k)
    return p


def oracle(frames, plans, active=None):
    return np.stack([JO.color_jitter(f, p) if active is None or active[b] else f
                     for b, (f, p) in enumerate(zip(frames, plans))])


def c_call(rgb, plan, plan_d, active, out, work, stream=None):
    B, H, W, _ = rgb.shape
    return _lib.lib.ffb6d_color_jitter(rgb.data_ptr(), B, H, W, plan.ctypes.data, plan_d.data_ptr(),
                                       active.data_ptr(), out.data_ptr(), work.data_ptr(), stream)


@pytest.mark.parametrize("name", CASES)
def test_matches_torchvision(cuda, name):
    c = G[name]
    got = F.color_jitter(torch.from_numpy(case_input(c)[None]).to(cuda), c["plan"][None])[0].cpu().numpy()
    if "sha256_out" in c:
        assert hashlib.sha256(got.tobytes()).hexdigest() == str(c["sha256_out"])
    else:
        assert np.array_equal(got, c["out"]), (name, np.count_nonzero(got != c["out"]))


def test_fixture_cases_as_one_batch(cuda):
    """The fixture's 24 x 20 order cases in one call: frames do not leak into each other's means."""
    names = [n for n in CASES if n.startswith("order_")]
    x = np.stack([case_input(G[n]) for n in names])
    got = F.color_jitter(torch.from_numpy(x).to(cuda), np.stack([G[n]["plan"] for n in names])).cpu().numpy()
    assert np.array_equal(got, np.stack([G[n]["out"] for n in names]))


def test_batch_480x640_matches_oracle(cuda):
    B = 32
    frames = [make_aug_frame(900 + b, 480, 640)["rgb"] for b in range(B)]
    plans = random_plans(B, 17)
    rgb = torch.from_numpy(np.stack(frames)).to(cuda)
    got = F.color_jitter(rgb, plans)
    assert np.array_equal(got.cpu().numpy(), oracle(frames, plans))
    assert torch.equal(got, F.color_jitter(rgb, plans))                  # bitwise the same on a second run


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (5, 1), (3, 5), (2, 2), (37, 41), (61, 641)])
def test_odd_sizes_match_oracle(cuda, h, w):
    """Frames whose pixel count is not a multiple of 4 start at bytes that are not 4-byte aligned."""
    B = 5
    rs = np.random.RandomState(h * 1000 + w)
    frames = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for _ in range(B)]
    plans = random_plans(B, h + w)
    got = F.color_jitter(torch.from_numpy(np.stack(frames)).to(cuda), plans).cpu().numpy()
    assert np.array_equal(got, oracle(frames, plans))


def test_in_place_and_active_mask(cuda):
    B, h, w = 6, 45, 77
    frames = [make_aug_frame(950 + b, h, w)["rgb"] for b in range(B)]
    plans = random_plans(B, 3)
    act = np.array([1, 0, 1, 1, 0, 1], bool)
    want = oracle(frames, plans, act)
    x = torch.from_numpy(np.stack(frames)).to(cuda)
    assert np.array_equal(F.color_jitter(x, plans, active=act).cpu().numpy(), want)
    assert np.array_equal(F.color_jitter(x, plans, active=torch.from_numpy(act).to(cuda)).cpu().numpy(), want)
    got = F.color_jitter(x, plans, active=act).cpu().numpy()
    assert np.array_equal(got[~act], np.stack(frames)[~act])           # inactive frames byte-identical
    # in place through the C ABI (out == rgb), odd frame size and a batch with every frame active
    y = x.clone()
    plan_d = torch.from_numpy(plans).to(cuda)
    a_d = torch.from_numpy(act.astype(np.uint8)).to(cuda)
    work = torch.empty(B, dtype=torch.int64, device=cuda)
    _lib.check(c_call(y, plans, plan_d, a_d, y, work))
    assert np.array_equal(y.cpu().numpy(), want)
    z = x.clone()
    _lib.check(c_call(z, plans, plan_d, torch.ones_like(a_d), z, work))
    assert np.array_equal(z.cpu().numpy(), oracle(frames, plans))


def test_cuda_graph_replay(cuda):
    B, h, w = 8, 96, 128
    frames = [make_aug_frame(970 + b, h, w)["rgb"] for b in range(B)]
    plans = random_plans(B, 9)
    rgb = torch.from_numpy(np.stack(frames)).to(cuda)
    want = F.color_jitter(rgb, plans)
    assert np.array_equal(want.cpu().numpy(), oracle(frames, plans))
    plan_d = torch.from_numpy(plans).to(cuda)
    act = torch.ones(B, dtype=torch.uint8, device=cuda)
    out, work = torch.empty_like(rgb), torch.full((B,), 12345, dtype=torch.int64, device=cuda)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _lib.check(c_call(rgb, plans, plan_d, act, out, work, s.cuda_stream))
    for _ in range(3):
        out.zero_()
        work.fill_(-7)                      # the call zeroes its sums itself
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)


def test_ops_validation(cuda):
    rgb = torch.zeros(2, 4, 6, 3, dtype=torch.uint8, device=cuda)
    p = random_plans(2, 1)
    with pytest.raises(ValueError, match="plan"):
        F.color_jitter(rgb, p[:1])
    with pytest.raises(ValueError, match="rgb"):
        F.color_jitter(rgb.float(), p)
    with pytest.raises(ValueError, match="rgb"):
        F.color_jitter(rgb[..., :2], p)
    with pytest.raises(ValueError, match="active"):
        F.color_jitter(rgb, p, active=[True])
    bad = p.copy()
    bad[1, 7] = 0.6
    with pytest.raises(_lib.FFB6DError, match="hue"):
        F.color_jitter(rgb, bad)
    assert F.color_jitter(rgb[:0], p[:0]).shape == (0, 4, 6, 3)


def test_chain_into_build_item(cuda):
    """color_jitter -> rgb_add_noise -> add_real_back -> build_ffb6d_item(fill=True) on the device equals the same
    chain through the oracles."""
    from oracle import aug_oracle as AO
    from ffb6d_b200.schedule import build_ffb6d_item
    from ffb6d_b200.item import pose_gt_objects
    from ffb6d_b200.synthetic import make_item_frame
    B, h, w = 2, 480, 640
    frames = [make_aug_frame(40 + b, h, w, "ycb") for b in range(B)]
    torch.manual_seed(8)
    jit = A.draw_color_jitter(B)
    noise = np.stack([A.draw_rgb_noise(np.random.RandomState(3 + b), "ycb") for b in range(B)])
    noise[:, A.I_HSV], noise[:, A.I_S_FACTOR], noise[:, A.I_V_FACTOR] = 1, 1.3, 1.2
    noise[:, A.I_NOISE], noise[:, A.I_NOISE_SIGMA] = 1, 9
    t = lambda k: torch.from_numpy(np.stack([f[k] for f in frames])).to(cuda)      # noqa: E731
    rgb = F.color_jitter(t("rgb"), jit)
    rgb = F.rgb_add_noise(rgb, noise, 3)
    rgb, dpt = F.add_real_back(rgb, t("labels"), t("raw"), t("back_rgb"), t("back_labels"), t("back_dpt"))
    z = [F.aug_noise_field(3, B, h, w, st, cuda).cpu().numpy() for st in (0, 1)]
    want_rgb, want_dpt = [], []
    for b, f in enumerate(frames):
        x = AO.rgb_add_noise(JO.color_jitter(f["rgb"], jit[b]), noise[b], z[0][b], z[1][b])
        r, d = AO.add_real_back(x, f["labels"], f["raw"], f["back_rgb"], f["back_labels"], f["back_dpt"], True, "ycb")
        want_rgb.append(r)
        want_dpt.append(d)
    want_rgb, want_dpt = np.stack(want_rgb), np.stack(want_dpt)
    assert np.array_equal(rgb.cpu().numpy(), want_rgb) and np.array_equal(dpt.cpu().numpy(), want_dpt)
    it = make_item_frame(9, h=h, w=w, cls_ids=(2, 5, 2), blobs=(2, 5, 7))
    obj = [pose_gt_objects(it["poses"], it["cls_ids"], it["kps"], it["ctrs"], 22, 8)] * B
    nrm = torch.from_numpy(np.stack([it["nrm"]] * B)).to(cuda)
    args = dict(cam_scale=float(it["cam_scale"]), K=it["K"], nrm_map=nrm, objects=obj, n_points=2048, seed=5,
                fill=True)
    got = build_ffb6d_item(dpt, rgb=rgb, labels=t("labels"), **args)
    want = build_ffb6d_item(torch.from_numpy(want_dpt).to(cuda), rgb=torch.from_numpy(want_rgb).to(cuda),
                            labels=t("labels"), **args)
    assert set(got) == set(want)
    for k in got:
        if isinstance(got[k], torch.Tensor):
            assert torch.equal(got[k], want[k]), k
