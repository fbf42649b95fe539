"""CPU: the numpy restatement of the colour jitter against torchvision and Pillow's outputs
(tests/golden/jitter_cases.npz), and draw_color_jitter against the draws of ColorJitter.get_params."""
import hashlib
import itertools
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, _npz_groups
from ffb6d_b200 import augment as A
from ffb6d_b200.synthetic import make_aug_frame
from oracle import jitter_oracle as O

G = _npz_groups(os.path.join(GOLDEN, "jitter_cases.npz"))
CASES = sorted(k for k, v in G.items() if "plan" in v)
DRAWS = sorted(k for k in G if k.startswith("draws_"))
SEEDS = sorted(k for k in G if k.startswith("seed_"))


def case_input(c):
    if "rgb" in c:
        return c["rgb"]
    seed, h, w = (int(x) for x in c["meta"])
    return make_aug_frame(seed, h, w)["rgb"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_torchvision(name):
    c = G[name]
    got = O.color_jitter(case_input(c), c["plan"])
    if "sha256_out" in c:
        assert hashlib.sha256(got.tobytes()).hexdigest() == str(c["sha256_out"])
    else:
        assert np.array_equal(got, c["out"]), (name, np.count_nonzero(got != c["out"]))


def test_fixture_covers_the_contract():
    plans = {n: G[n]["plan"] for n in CASES}
    orders = {tuple(p[:4].astype(int)) for p in plans.values()}
    assert orders >= set(itertools.permutations(range(4)))
    shifts = {O.hue_shift(p[7]) for p in plans.values()}
    assert shifts >= set(range(-12, 13))
    hues = {p[7] for p in plans.values()}
    assert any(0 < h < 1 / 255 for h in hues) and any(1 / 255 < h < 1.01 / 255 for h in hues)
    for op in range(3):
        f = {p[4 + op] for p in plans.values()}
        assert {0.8, 1.0, 1.2} <= f and any(0.8 < x < 1.0 for x in f) and any(1.0 < x < 1.2 for x in f)
    shapes = {case_input(G[n]).shape[:2] for n in CASES}
    assert (1, 1) in shapes and (480, 640) in shapes and any(h % 2 and w % 2 for h, w in shapes)
    assert any(n.startswith("rgba_") for n in CASES) and any(n.startswith("contrast_half") for n in CASES)


def test_contrast_mean_on_the_half_boundary_rounds_up():
    n = 0
    for name in (n for n in CASES if n.startswith("contrast_half")):
        c = G[name]
        if int(c["plan"][0]) == 1:                  # contrast first: the mean is over the input
            L = O.luma(case_input(c))
            assert L.sum() % L.size == L.size // 2 and L.size % 2 == 0
            assert int(float(L.sum()) / L.size + 0.5) == L.sum() // L.size + 1
            n += 1
    assert n >= 2


def test_rgba_keeps_the_rgb_bands():
    """The fixture's RGBA outputs (first three bands) are what the RGB input gives."""
    names = [n for n in CASES if n.startswith("rgba_")]
    assert len(names) >= 6
    for n in names:
        assert np.array_equal(O.color_jitter(case_input(G[n]), G[n]["plan"]), G[n]["out"])


@pytest.mark.parametrize("name", DRAWS)
def test_draws_reproduce_get_params(name):
    c = G[name]
    want = c["plans"]
    torch.manual_seed(int(c["torch_seed"]))
    assert np.array_equal(A.draw_color_jitter(len(want)), want)
    g = torch.Generator().manual_seed(int(c["torch_seed"]))
    state = torch.get_rng_state()
    assert np.array_equal(A.draw_color_jitter(len(want), generator=g), want)
    assert torch.equal(torch.get_rng_state(), state)         # an explicit generator leaves the default alone


@pytest.mark.parametrize("name", SEEDS)
def test_draws_reproduce_whole_calls(name):
    c = G[name]
    torch.manual_seed(int(c["torch_seed"]))
    assert np.array_equal(A.draw_color_jitter(1)[0], c["plan"])


def test_draws_match_torchvision_live():
    T = pytest.importorskip("torchvision.transforms")
    cj = T.ColorJitter(0.2, 0.2, 0.2, 0.05)
    for seed in (5, 6, 99):
        torch.manual_seed(seed)
        want = []
        for _ in range(4):
            fn_idx, b, c, s, h = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
            want.append(fn_idx.tolist() + [b, c, s, h])
        after = torch.get_rng_state()
        torch.manual_seed(seed)
        assert np.array_equal(A.draw_color_jitter(4), np.array(want))
        assert torch.equal(torch.get_rng_state(), after)      # the generator is left where get_params leaves it


def test_draw_ranges():
    torch.manual_seed(0)
    p = A.draw_color_jitter(500)
    assert p.shape == (500, A.JITTER_PLAN_LEN) and p.dtype == np.float64
    assert all(sorted(r) == [0, 1, 2, 3] for r in p[:, :4])
    assert np.all((p[:, 4:7] >= 0.8) & (p[:, 4:7] <= 1.2)) and np.all(np.abs(p[:, 7]) <= 0.05)
    assert np.array_equal(p[:, 4:], p[:, 4:].astype(np.float32))      # float32 draws, widened
    assert A.draw_color_jitter(0).shape == (0, A.JITTER_PLAN_LEN)
