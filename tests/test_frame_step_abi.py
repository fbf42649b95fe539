"""CPU: the entry points of training from decoded frames (DESIGN.md §4.28) are declared and exported; the record and
plan checks reject, without a launch, every bad record and plan that test_aug_abi / test_jitter_abi feed to the
launching calls, with the launching calls' message; the ``_dseed`` entry points check their arguments, and their
size limits, as the by-value ones do."""
import ctypes as C

import numpy as np
import pytest

from ffb6d_b200 import _lib, augment as A
from test_abi import declared_symbols

NEW = ("ffb6d_sample_pixels_dseed", "ffb6d_rgb_add_noise_dseed", "ffb6d_rgb_noise_check_records",
       "ffb6d_color_jitter_check_plans")
B, H, W = 2, 32, 40
_buf = (C.c_double * (1 << 14))()
P = C.addressof(_buf)                 # a fake "device" address; no call below reaches a launch
FAR = P + 8 * 8192


def test_new_symbols_declared_and_exported():
    raw = C.CDLL(_lib.LIB_PATH)
    for s in NEW:
        assert s in declared_symbols() and s in _lib.SYMBOLS and hasattr(raw, s), s


def records(**slots):
    p = np.stack([A.identity_record("ycb")] * B)
    for k, v in slots.items():
        p[:, getattr(A, k)] = v
    return p


def noise(plan, dseed=False):
    args = (P, B, H, W, plan.ctypes.data, P, P + 64 if dseed else 1, None, P + 8, P + 16, None)
    return (_lib.lib.ffb6d_rgb_add_noise_dseed if dseed else _lib.lib.ffb6d_rgb_add_noise)(*args)


BAD_RECORDS = [dict(I_VERSION=2), dict(I_MOTION_A=31), dict(I_MOTION_A=2.5), dict(I_GAUSS_K=4), dict(I_GAUSS_K=3),
               dict(I_HSV=2), dict(I_NOISE_SIGMA=-1), dict(I_S_FACTOR=np.nan), dict(I_PASS=2),
               dict(I_SHARPEN_K=np.inf)]


@pytest.mark.parametrize("slots", BAD_RECORDS)
def test_record_check_matches_the_launching_call(slots):
    plan = records(**slots)
    plan[0] = A.identity_record("ycb")             # the bad record is frame 1's
    n0 = _lib.launch_count()
    messages = []
    for rc in (noise(plan), noise(plan, dseed=True), _lib.lib.ffb6d_rgb_noise_check_records(plan.ctypes.data, B)):
        assert rc == _lib.ERR_INVALID
        messages.append(_lib.last_error())
    assert messages[0].startswith("rgb_add_noise: frame 1: bad record") and len(set(messages)) == 1, messages
    assert _lib.launch_count() == n0
    with pytest.raises(_lib.FFB6DError) as e:
        from ffb6d_b200 import ops
        ops.rgb_noise_check_records(plan)
    assert messages[0] in str(e.value)


def test_record_check_accepts_good_records():
    rs = np.random.RandomState(3)
    plan = np.stack([A.draw_rgb_noise(rs, ds, p) for ds in ("ycb", "linemod") for p in (0, 1)])
    assert _lib.lib.ffb6d_rgb_noise_check_records(plan.ctypes.data, len(plan)) == _lib.OK
    assert _lib.lib.ffb6d_rgb_noise_check_records(None, 0) == _lib.OK


def test_record_check_arguments():
    plan = records()
    for b in (-1, 65536):
        assert _lib.lib.ffb6d_rgb_noise_check_records(plan.ctypes.data, b) == _lib.ERR_INVALID
        assert "bad size" in _lib.last_error()
    assert _lib.lib.ffb6d_rgb_noise_check_records(None, B) == _lib.ERR_INVALID and "null" in _lib.last_error()
    raw = np.zeros(B * A.REC_LEN + 1)
    assert _lib.lib.ffb6d_rgb_noise_check_records(raw.ctypes.data + 4, B) == _lib.ERR_INVALID
    assert "misaligned" in _lib.last_error()


def plans(order=(0, 1, 2, 3), factors=(1.1, 0.9, 1.0, 0.01)):
    return np.tile(np.array(list(order) + list(factors), np.float64), (B, 1))


BAD_PLANS = [plans(order=o) for o in [(0, 1, 2, 2), (0, 0, 0, 0), (1, 2, 3, 4), (-1, 1, 2, 3), (0.5, 1, 2, 3),
                                      (np.nan, 1, 2, 3), (3, 2, 1, np.inf)]] + \
            [plans(factors=f) for f in [(np.nan, 1, 1, 0), (1, np.inf, 1, 0), (1, 1, -1e-9, 0), (1e39, 1, 1, 0),
                                        (1, 1, 1, 0.5000001), (1, 1, 1, -0.51), (1, 1, 1, np.nan)]]
_later = plans()
_later[1, 7] = 0.7
BAD_PLANS.append(_later)


@pytest.mark.parametrize("i", range(len(BAD_PLANS)))
def test_plan_check_matches_the_launching_call(i):
    plan = BAD_PLANS[i]
    n0 = _lib.launch_count()
    assert _lib.lib.ffb6d_color_jitter(P, B, 5, 7, plan.ctypes.data, FAR, FAR + 256, P, FAR + 512, None) \
        == _lib.ERR_INVALID
    want = _lib.last_error()
    assert "bad plan" in want
    assert _lib.lib.ffb6d_color_jitter_check_plans(plan.ctypes.data, B) == _lib.ERR_INVALID
    assert _lib.last_error() == want
    assert _lib.launch_count() == n0
    from ffb6d_b200 import ops
    with pytest.raises(_lib.FFB6DError, match="bad plan"):
        ops.color_jitter_check_plans(plan)


def test_plan_check_arguments():
    plan = plans()
    assert _lib.lib.ffb6d_color_jitter_check_plans(plan.ctypes.data, B) == _lib.OK
    for b in (0, -1, 65536):
        assert _lib.lib.ffb6d_color_jitter_check_plans(plan.ctypes.data, b) == _lib.ERR_INVALID
        assert "bad size" in _lib.last_error()
    assert _lib.lib.ffb6d_color_jitter_check_plans(None, B) == _lib.ERR_INVALID and "null" in _lib.last_error()
    raw = np.zeros(B * A.JITTER_PLAN_LEN + 1)
    assert _lib.lib.ffb6d_color_jitter_check_plans(raw.ctypes.data + 4, B) == _lib.ERR_INVALID
    assert "misaligned" in _lib.last_error()


# the size limits of ffb6d_rgb_add_noise / ffb6d_sample_pixels hold for their _dseed twins
@pytest.mark.parametrize("kw", [dict(B=-1), dict(B=65536), dict(H=31), dict(W=31), dict(H=1 << 16, W=1 << 15),
                                dict(H=65535 * 8 + 1, W=32)])
def test_noise_dseed_sizes(kw):
    plan = records()
    a = dict(B=B, H=H, W=W)
    a.update(kw)
    assert _lib.lib.ffb6d_rgb_add_noise_dseed(P, a["B"], a["H"], a["W"], plan.ctypes.data, P, P + 64, None, P + 8,
                                              P + 16, None) == _lib.ERR_INVALID
    assert "bad size" in _lib.last_error()


def test_noise_dseed_seed_pointer():
    plan = records()
    assert _lib.lib.ffb6d_rgb_add_noise_dseed(P, B, H, W, plan.ctypes.data, P, None, None, P + 8, P + 16, None) \
        == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
    assert _lib.lib.ffb6d_rgb_add_noise_dseed(P, B, H, W, plan.ctypes.data, P, P + 4, None, P + 8, P + 16, None) \
        == _lib.ERR_INVALID and "misaligned" in _lib.last_error()
    assert _lib.lib.ffb6d_rgb_add_noise_dseed(None, 0, H, W, None, None, None, None, None, None, None) == _lib.OK


def sample(seed_dev=P + 64, B_=1, H_=8, W_=8, N=16, ws_bytes=1 << 20):
    return _lib.lib.ffb6d_sample_pixels_dseed(P, B_, H_, W_, 0.0, N, seed_dev, P + 128, None, FAR, ws_bytes, None)


@pytest.mark.parametrize("kw", [dict(B_=-1), dict(B_=65536), dict(H_=0), dict(N=-1), dict(H_=1 << 15, W_=1 << 15),
                                dict(N=1 << 30)])
def test_sample_dseed_sizes(kw):
    assert sample(**kw) == _lib.ERR_INVALID and "bad size" in _lib.last_error()


def test_sample_dseed_arguments():
    assert sample(seed_dev=None) == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
    assert sample(seed_dev=P + 4) == _lib.ERR_INVALID and "misaligned" in _lib.last_error()
    assert sample(ws_bytes=16) == _lib.ERR_INVALID and "workspace too small" in _lib.last_error()
    assert sample(seed_dev=None, B_=0) == _lib.OK and sample(seed_dev=None, N=0) == _lib.OK


def test_train_item_checks_need_no_gpu():
    import ffb6d_b200 as F
    with pytest.raises(ValueError, match="dataset"):
        F.build_ffb6d_train_item({}, dataset="coco", cam_scale=1e4, K=np.eye(3), n_points=256, seed=0)
    with pytest.raises(ValueError, match="lacks"):
        F.build_ffb6d_train_item({"rgb": None}, dataset="ycb", cam_scale=1e4, K=np.eye(3), n_points=256, seed=0)
