"""CPU: what :class:`ffb6d_b200.GraphedTrainStep` rejects before any CUDA work, and its item helpers."""
import os
import subprocess
import sys

import pytest
import torch

from ffb6d_b200 import _lib, graphed
from ffb6d_b200.model import FFB6DFusionNet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _setup(capturable=True):
    model = FFB6DFusionNet(n_classes=2, n_pts=256).train()
    opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4), capturable=capturable)
    return model, opt, {"rgb_feats": [], "labels": torch.zeros(2, 256)}


def test_rejects_wrappers_and_other_models():
    model, opt, item = _setup()
    with pytest.raises(ValueError, match="DataParallel"):
        graphed.GraphedTrainStep(torch.nn.DataParallel(model), opt, item)
    with pytest.raises(ValueError, match="FFB6DFusionNet or FFB6D"):
        graphed.GraphedTrainStep(torch.nn.Linear(2, 2), opt, item)
    with pytest.raises(ValueError, match="rgb_feats"):
        graphed.GraphedTrainStep(model, opt, {"labels": item["labels"]})
    with pytest.raises(ValueError, match="warmup"):
        graphed.GraphedTrainStep(model, opt, item, warmup=0)


def test_rejects_settings_that_cannot_be_captured(monkeypatch):
    model, opt, item = _setup(capturable=False)
    with pytest.raises(ValueError, match="capturable=True"):
        graphed.GraphedTrainStep(model, opt, item)
    model, opt, item = _setup()
    model.rndla_pre_stages.bn.bn.momentum = None
    with pytest.raises(ValueError, match="rndla_pre_stages.bn.bn.*momentum=None"):
        graphed.GraphedTrainStep(model, opt, item)
    model, opt, item = _setup()
    model.eval()
    with pytest.raises(ValueError, match="eval mode"):
        graphed.GraphedTrainStep(model, opt, item)
    model.train()
    # the library reads the variable once, at its first use: let it read it unset before the variable is set here
    assert not _lib.lib.ffb6d_check_indices_enabled()
    for value, rejected in (("1", True), ("yes", True), ("0", False), ("", False)):
        monkeypatch.setenv("FFB6D_CHECK_INDICES", value)
        assert graphed._check_indices_on() is rejected
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="FFB6D_CHECK_INDICES"):
        graphed.GraphedTrainStep(model, opt, item)


def test_item_tree_helpers():
    cpu = torch.zeros(3)
    tree = {"a": cpu, "b": [cpu, (cpu,)], "c": 4}
    assert graphed._tensors(tree) == []              # CPU tensors and other values get no input buffer
    assert graphed._lookup(tree, ("b", 1, 0)) is cpu
    assert graphed._lookup(tree, ("b", 2)) is None
    assert graphed._lookup(tree, ("d",)) is None
    copied = graphed._static_copy(tree)
    assert copied["b"][1][0] is cpu and copied["c"] == 4 and isinstance(copied["b"][1], tuple)


def test_rejects_optimizers_whose_fresh_state_is_not_zero():
    model, _, item = _setup()
    for opt in (torch.optim.NAdam(model.parameters(), lr=torch.tensor(1e-4), capturable=True),
                torch.optim.ASGD(model.parameters(), lr=torch.tensor(1e-4), capturable=True),
                torch.optim.SGD(model.parameters(), lr=1e-4)):
        with pytest.raises(ValueError, match="Adam or AdamW"):
            graphed.GraphedTrainStep(model, opt, item)
    # AdamW passes the host checks
    opt = torch.optim.AdamW(model.parameters(), lr=torch.tensor(1e-4), capturable=True)
    step = graphed.GraphedTrainStep.__new__(graphed.GraphedTrainStep)
    step.model, step.optimizer = model, opt
    step._read_modules()
    step._check(True)


def test_check_indices_as_the_library_read_it():
    """Set when the library loaded, unset later: the gathers still synchronise, so the step still refuses."""
    code = ("import os, ffb6d_b200._lib as L; assert L.lib.ffb6d_check_indices_enabled() == 1; "
            "del os.environ['FFB6D_CHECK_INDICES']; from ffb6d_b200 import graphed; "
            "assert graphed._check_indices_on(); print('ok')")
    env = dict(os.environ, FFB6D_CHECK_INDICES="1")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stderr[-2000:]
