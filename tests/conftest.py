import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _npz_groups(path):
    z = np.load(path)
    groups = {}
    for key in z.files:
        if "/" in key:
            g, f = key.split("/", 1)
            groups.setdefault(g, {})[f] = z[key]
        else:
            groups[key] = z[key]
    return groups


@pytest.fixture(scope="session")
def knn_golden():
    return _npz_groups(os.path.join(GOLDEN, "knn_cases.npz"))


@pytest.fixture(scope="session")
def gather_golden():
    return _npz_groups(os.path.join(GOLDEN, "gather_cases.npz"))


@pytest.fixture(scope="session")
def grid_golden():
    return _npz_groups(os.path.join(GOLDEN, "grid_cases.npz"))


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test ran without a CUDA device")
    return torch.device("cuda:0")


def frame_point_sets(frame, n_points):
    from ffb6d_b200.synthetic import image_pyramid_np
    sets = {("cld", i): frame["cld"][: n_points // 4 ** i] for i in range(5)}
    for sr, p in image_pyramid_np(frame["dpt_xyz"]).items():
        sets[("img", sr)] = p
    return sets
