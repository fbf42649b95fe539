"""CPU: what :class:`ffb6d_b200.GraphedEvalStep` rejects before any CUDA work."""
import pytest
import torch

from ffb6d_b200 import _lib, graphed
from ffb6d_b200.model import FFB6DFusionNet


def _setup():
    model = FFB6DFusionNet(n_classes=2, n_pts=256).eval()
    return model, {"rgb_feats": [], "labels": torch.zeros(2, 256)}


def test_rejects_wrappers_and_other_models():
    model, item = _setup()
    with pytest.raises(ValueError, match=r"GraphedEvalStep: .*DataParallel.*\.module"):
        graphed.GraphedEvalStep(torch.nn.DataParallel(model), item)
    with pytest.raises(ValueError, match="FFB6DFusionNet or FFB6D"):
        graphed.GraphedEvalStep(torch.nn.Linear(2, 2), item)
    with pytest.raises(ValueError, match="example_item must be a dict"):
        graphed.GraphedEvalStep(model, [item])
    with pytest.raises(ValueError, match="rgb_feats"):
        graphed.GraphedEvalStep(model, {"labels": item["labels"]})
    with pytest.raises(ValueError, match="warmup"):
        graphed.GraphedEvalStep(model, item, warmup=0)


def test_rejects_training_mode_and_the_index_check(monkeypatch):
    model, item = _setup()
    model.train()
    with pytest.raises(ValueError, match="GraphedEvalStep: the model is in training mode"):
        graphed.GraphedEvalStep(model, item)
    model.eval()
    # the library reads the variable once, at its first use: let it read it unset before the variable is set here
    assert not _lib.lib.ffb6d_check_indices_enabled()
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="GraphedEvalStep: FFB6D_CHECK_INDICES"):
        graphed.GraphedEvalStep(model, item)


def test_accepts_sync_batchnorm_and_any_batchnorm_momentum():
    """Eval normalises with the running statistics: SyncBatchNorm and momentum=None pass the host checks."""
    model, _ = _setup()
    model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model).eval()
    model.rndla_pre_stages.bn.bn.momentum = None
    step = graphed.GraphedEvalStep.__new__(graphed.GraphedEvalStep)
    step.model = model
    step._read_modules()
    step._check()

