"""CPU: the numpy restatement of the augmentation kernels against the reference's own functions
(tests/golden/aug_cases.npz), and the host draw helpers against the reference's sequence of rng calls."""
import hashlib
import os

import numpy as np
import pytest

from conftest import GOLDEN, _npz_groups
from ffb6d_b200 import augment as A
from ffb6d_b200.synthetic import make_aug_frame
from oracle import aug_oracle as O

G = _npz_groups(os.path.join(GOLDEN, "aug_cases.npz"))
NOISE_CASES = sorted(k for k, v in G.items() if "record" in v)
BACK_CASES = sorted(k for k in G if k.startswith("back_"))
CALL_CASES = sorted(k for k in G if k.startswith("calls_"))
DS = ("ycb", "linemod")


def case_frame(c):
    d, seed, h, w, ch = (int(x) for x in c["meta"][:5])
    return DS[d], make_aug_frame(seed, h, w, DS[d], ch)


def dft_path(rec):
    """OpenCV's filter2D convolves through a DFT for 8-bit kernels of 130 or more taps (measured with OpenCV 4.13
    on x86-64: 11x11 is direct, 12x12 is not), where it may round differently by 1."""
    return rec[A.I_MOTION_A] >= 12


@pytest.mark.parametrize("name", NOISE_CASES)
def test_oracle_matches_reference_rgb_add_noise(name):
    c = G[name]
    d, fr = case_frame(c)
    rec = c["record"]
    f = c.get("fields", np.zeros((2,) + fr["rgb"].shape))
    got = O.rgb_add_noise(fr["rgb"], rec, f[0], f[1])
    if "sha256_out" in c:
        assert hashlib.sha256(got.tobytes()).hexdigest() == str(c["sha256_out"])
        return
    want = c["out"]
    diff = np.abs(got.astype(int) - want)
    if dft_path(rec):
        assert diff.max() <= 1, name
    else:
        assert np.array_equal(got, want), (name, np.count_nonzero(diff))


@pytest.mark.parametrize("name", BACK_CASES)
def test_oracle_matches_reference_add_real_back(name):
    c = G[name]
    d, fr = case_frame(c)
    rgb, dpt = O.add_real_back(fr["rgb"], fr["labels"], fr["raw"], fr["back_rgb"], fr["back_labels"],
                               fr["back_dpt"], bool(c["meta"][5]), d)
    assert np.array_equal(rgb, c["rgb"]) and np.array_equal(dpt, c["dpt"])


def test_fixture_covers_the_issue_cases():
    recs = [G[n]["record"] for n in NOISE_CASES]
    a = {int(r[A.I_MOTION_A]) for r in recs}
    assert {1, 2, 14, 30} <= a and any(x >= 12 for x in a)
    assert {3, 5} <= {int(r[A.I_GAUSS_K]) for r in recs}
    assert 0.0 in {r[A.I_GAUSS_SIGMA] for r in recs if r[A.I_GAUSS_K]}
    assert {0, 24} <= {int(r[A.I_NOISE_SIGMA]) for r in recs if r[A.I_NOISE]}
    assert any(r[A.I_FINAL] for r in recs)
    assert any(int(G[n]["meta"][2]) % 2 for n in NOISE_CASES)


def test_dft_exception_is_rare_and_one_lsb():
    """Count the pixels where OpenCV's DFT path differs from the direct sum, over the fixture's large motion blurs."""
    n_diff = n_all = 0
    for name in NOISE_CASES:
        c = G[name]
        if "out" not in c or not dft_path(c["record"]):
            continue
        _, fr = case_frame(c)
        f = c.get("fields", np.zeros((2,) + fr["rgb"].shape))
        d = np.abs(O.rgb_add_noise(fr["rgb"], c["record"], f[0], f[1]).astype(int) - c["out"])
        assert d.max() <= 1
        n_diff += np.count_nonzero(d)
        n_all += d.size
    assert n_all > 0 and n_diff == 0       # measured: none of the fixture's 96 465 values differ


class Recorder:
    def __init__(self, seed):
        self.rs, self.log = np.random.RandomState(seed), []

    def rand(self):
        self.log.append("rand")
        return self.rs.rand()

    def randint(self, *a):
        self.log.append("randint%r" % (a,))
        return self.rs.randint(*a)


@pytest.mark.parametrize("name", CALL_CASES)
def test_draws_follow_reference_order(name):
    _, d, typ, seed = name.split("_")
    want = [s for s in G[name]["log"].tolist() if s not in ("randn", "normal")]
    rng = Recorder(int(seed))
    plan = A.draw_frame_augmentation(rng, d, 7, rnd_typ=typ if d == "linemod" else "syn")
    assert rng.log == want
    if plan["augment"]:
        assert 0 <= plan["back_index"] < 7


def test_helpers_refuse_unknown_dataset():
    with pytest.raises(ValueError):
        A.draw_rgb_noise(np.random.RandomState(0), "coco")
    with pytest.raises(ValueError):
        A.draw_frame_augmentation(np.random.RandomState(0), "linemod", 3, rnd_typ="real")
