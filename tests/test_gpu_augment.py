"""GPU: ffb6d_rgb_add_noise / ffb6d_add_real_back / ffb6d_aug_noise_field against the reference's outputs
(tests/golden/aug_cases.npz) and the numpy restatement (oracle/aug_oracle.py)."""
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, _npz_groups
import ffb6d_b200 as F
from ffb6d_b200 import augment as A, _lib
from ffb6d_b200.synthetic import make_aug_frame
from oracle import aug_oracle as O

pytestmark = pytest.mark.gpu
G = _npz_groups(os.path.join(GOLDEN, "aug_cases.npz"))
NOISE_CASES = sorted(k for k, v in G.items() if "record" in v)
BACK_CASES = sorted(k for k in G if k.startswith("back_"))
DS = ("ycb", "linemod")


def case_frame(c):
    d, seed, h, w, ch = (int(x) for x in c["meta"][:5])
    return DS[d], make_aug_frame(seed, h, w, DS[d], ch)


@pytest.mark.parametrize("name", NOISE_CASES)
def test_rgb_add_noise_matches_reference(cuda, name):
    c = G[name]
    _, fr = case_frame(c)
    noise = None
    if "fields" in c:
        noise = torch.from_numpy(c["fields"][:, None]).to(cuda)
    got = F.rgb_add_noise(torch.from_numpy(fr["rgb"][None]).to(cuda), c["record"][None], 5, noise=noise)
    got = got[0].cpu().numpy()
    if "sha256_out" in c:
        assert hashlib.sha256(got.tobytes()).hexdigest() == str(c["sha256_out"])
        return
    d = np.abs(got.astype(int) - c["out"])
    if c["record"][A.I_MOTION_A] >= 12:            # OpenCV's DFT path (DESIGN §4.14): measured 0 differing values
        assert d.max() <= 1 and np.count_nonzero(d) == 0
    else:
        assert np.array_equal(got, c["out"]), np.count_nonzero(d)


@pytest.mark.parametrize("name", BACK_CASES)
def test_add_real_back_matches_reference(cuda, name):
    c = G[name]
    d, fr = case_frame(c)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)[None]).to(cuda)       # noqa: E731
    rgb, dpt = F.add_real_back(t(fr["rgb"]), t(fr["labels"]), t(fr["raw"]), t(fr["back_rgb"]), t(fr["back_labels"]),
                               t(fr["back_dpt"]), [bool(c["meta"][5])], d)
    assert np.array_equal(rgb[0].cpu().numpy(), c["rgb"]) and np.array_equal(dpt[0].cpu().numpy(), c["dpt"])


def mixed_batch(B, h, w, seed):
    rs = np.random.RandomState(seed)
    frames = [make_aug_frame(seed + b, h, w, DS[b % 2], 1 + 2 * (b % 3 == 1)) for b in range(B)]
    plans = np.stack([A.draw_rgb_noise(rs, DS[b % 2], b % 2) for b in range(B)])
    plans[0] = A.draw_rgb_noise(np.random.RandomState(3), "ycb")     # plus forced stages on a few frames
    for b, (a, k) in enumerate([(30, 5), (13, 3), (2, 0)][:B - 1], start=1):
        p = plans[b]
        p[A.I_HSV], p[A.I_S_FACTOR], p[A.I_V_FACTOR] = 1, 1.45, 1.3
        kern = A.motion_kernel(*{30: (0, 15), 13: (137, 7), 2: (359, 1)}[a])
        p[A.I_MOTION_A] = kern.shape[0]
        p[A.I_MOTION_K:A.I_MOTION_K + kern.size] = kern.ravel()
        p[A.I_GAUSS_K] = k
        if k:
            p[A.I_GAUSS_TAPS:A.I_GAUSS_TAPS + k] = A.gaussian_taps(k, 0.77)
    plans[-1][A.I_NOISE], plans[-1][A.I_NOISE_SIGMA], plans[-1][A.I_FINAL] = 1, 24, 1
    return frames, plans


def oracle_batch(frames, plans, seed, dev):
    B, (h, w) = len(frames), frames[0]["labels"].shape
    fields = {}
    want = []
    for b in range(B):
        p = int(plans[b][A.I_PASS])
        z = []
        for st in (2 * p, 2 * p + 1):
            if st not in fields:                     # each stage's [B,H,W,3] field once
                fields[st] = F.aug_noise_field(seed, B, h, w, st, dev).cpu().numpy()
            z.append(fields[st][b])
        want.append(O.rgb_add_noise(frames[b]["rgb"], plans[b], z[0], z[1]))
    return np.stack(want)


def test_batch_480x640_matches_oracle(cuda):
    frames, plans = mixed_batch(32, 480, 640, 11)
    rgb = torch.from_numpy(np.stack([f["rgb"] for f in frames])).to(cuda)
    got = F.rgb_add_noise(rgb, plans, 1234).cpu().numpy()
    assert np.array_equal(got, oracle_batch(frames, plans, 1234, cuda))
    again = F.rgb_add_noise(rgb, plans, 1234).cpu().numpy()
    assert np.array_equal(got, again)
    assert not np.array_equal(got, F.rgb_add_noise(rgb, plans, 1235).cpu().numpy())


def test_odd_batch_matches_oracle(cuda):
    frames, plans = mixed_batch(6, 45, 77, 5)
    rgb = torch.from_numpy(np.stack([f["rgb"] for f in frames])).to(cuda)
    assert np.array_equal(F.rgb_add_noise(rgb, plans, 9).cpu().numpy(), oracle_batch(frames, plans, 9, cuda))


@pytest.mark.parametrize("h,w", [(33, 33), (32, 39), (45, 33)])
def test_narrow_frames_match_oracle(cuda, h, w):
    """Widths and heights just above 32, where the last tile's halo reaches furthest past the frame: the 30x30 motion
    blur (angle 0, length 15), the 5x5 Gaussian and the sharpen 3x3, on single frames and on a batch of two."""
    frames = [make_aug_frame(60 + i, h, w) for i in range(2)]
    plans = []
    for i, (ang, ln) in enumerate(((0, 15), (90, 15))):
        p = A.identity_record("ycb")
        k = A.motion_kernel(ang, ln)
        p[A.I_MOTION_A], p[A.I_MOTION_K:A.I_MOTION_K + k.size] = k.shape[0], k.ravel()
        p[A.I_GAUSS_K], p[A.I_GAUSS_TAPS:A.I_GAUSS_TAPS + 5] = 5, A.gaussian_taps(5, 0.9)
        p[A.I_SHARPEN] = i
        sh = -np.ones((3, 3))
        sh[1, 1] = 10.5
        p[A.I_SHARPEN_K:A.I_SHARPEN_K + 9] = (sh / sh.sum()).ravel()
        plans.append(p)
    plans = np.stack(plans)
    rgb = torch.from_numpy(np.stack([f["rgb"] for f in frames])).to(cuda)
    want = oracle_batch(frames, plans, 2, cuda)
    assert np.array_equal(F.rgb_add_noise(rgb[:1], plans[:1], 2).cpu().numpy(), want[:1])
    assert np.array_equal(F.rgb_add_noise(rgb, plans, 2).cpu().numpy(), want)


def test_noise_field_statistics(cuda):
    z = {(s, st): F.aug_noise_field(s, 2, 480, 640, st, cuda).cpu().numpy() for s in (1, 2) for st in (0, 1)}
    for v in z.values():
        for f in v:                                  # 921 600 samples per field
            assert abs(f.mean()) < 5 / np.sqrt(f.size) and abs(f.var() - 1) < 5 * np.sqrt(2 / f.size)
    flat = [v[b].ravel() for v in z.values() for b in range(2)]
    c = np.corrcoef(np.stack(flat))
    assert np.abs(c[~np.eye(len(flat), dtype=bool)]).max() < 5 / np.sqrt(flat[0].size)
    assert np.array_equal(z[(1, 0)], F.aug_noise_field(1, 2, 480, 640, 0, cuda).cpu().numpy())


def test_cuda_graph_replay(cuda):
    frames, plans = mixed_batch(4, 64, 96, 21)
    rgb = torch.from_numpy(np.stack([f["rgb"] for f in frames])).to(cuda)
    want = F.rgb_add_noise(rgb, plans, 77)
    plan_d = torch.from_numpy(plans).to(cuda)
    out, work = torch.empty_like(rgb), torch.empty_like(rgb)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _lib.check(_lib.lib.ffb6d_rgb_add_noise(rgb.data_ptr(), 4, 64, 96, plans.ctypes.data, plan_d.data_ptr(),
                                                    77, None, out.data_ptr(), work.data_ptr(), s.cuda_stream))
    for _ in range(2):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)


def test_composition_with_build_item(cuda):
    """Device-augmented rgb / depth into build_ffb6d_item(fill=True) equals build_ffb6d_item on the oracle's."""
    from ffb6d_b200.schedule import build_ffb6d_item
    B, h, w = 2, 480, 640
    frames, plans = mixed_batch(B, h, w, 40)
    for b in range(B):
        frames[b] = make_aug_frame(40 + b, h, w, "ycb")
    t = lambda k: torch.from_numpy(np.stack([f[k] for f in frames])).to(cuda)      # noqa: E731
    rgb = F.rgb_add_noise(t("rgb"), plans, 3)
    rgb, dpt = F.add_real_back(rgb, t("labels"), t("raw"), t("back_rgb"), t("back_labels"), t("back_dpt"))
    want_rgb = oracle_batch(frames, plans, 3, cuda)
    wd = []
    for b in range(B):
        r, d = O.add_real_back(want_rgb[b], frames[b]["labels"], frames[b]["raw"], frames[b]["back_rgb"],
                               frames[b]["back_labels"], frames[b]["back_dpt"], True, "ycb")
        want_rgb[b], _ = r, wd.append(d)
    assert np.array_equal(rgb.cpu().numpy(), want_rgb) and np.array_equal(dpt.cpu().numpy(), np.stack(wd))
    from ffb6d_b200.item import pose_gt_objects
    from ffb6d_b200.synthetic import make_item_frame
    it = make_item_frame(9, h=h, w=w, cls_ids=(2, 5, 2), blobs=(2, 5, 7))
    obj = [pose_gt_objects(it["poses"], it["cls_ids"], it["kps"], it["ctrs"], 22, 8)] * B
    nrm = torch.from_numpy(np.stack([it["nrm"]] * B)).to(cuda)
    args = dict(cam_scale=float(it["cam_scale"]), K=it["K"], nrm_map=nrm, objects=obj, n_points=2048, seed=5,
                fill=True)
    got = build_ffb6d_item(dpt, rgb=rgb, labels=t("labels"), **args)
    want = build_ffb6d_item(torch.from_numpy(np.stack(wd)).to(cuda), rgb=torch.from_numpy(want_rgb).to(cuda),
                            labels=t("labels"), **args)
    assert set(got) == set(want)
    for k in got:
        if isinstance(got[k], torch.Tensor):
            assert torch.equal(got[k], want[k]), k
