"""CPU: the image branch of :mod:`ffb6d_b200.cnn` against the reference's own modules, and ``FFB6D``'s state dict and
checkpoint loading against the reference's.

``cnn_cases.npz`` (tests/golden/make_cnn_golden.py) holds the reference's float64 outputs of every stage, run in a
chain from one stored image with the seeded weights of oracle/cnn_oracle.py, at a few thousand sampled positions per
stage.  The modules here run the same chain in float64 and are compared at those positions, stage by stage, so the
first stage that differs is the one reported.  ``ffb6d_state_keys.json`` lists every key and shape of the
reference's ``FFB6D(n_classes=22)``."""
import io
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import GOLDEN
from ffb6d_b200 import cnn
from ffb6d_b200.model import FFB6D, FFB6DFusionNet, load_reference_checkpoint
from oracle import cnn_oracle

NAMES = ["cnn_pre_stages"] + ["cnn_ds_stages.%d" % j for j in range(4)] + ["cnn_up_stages.%d" % j for j in range(4)]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "cnn_cases.npz")))


@pytest.fixture(scope="module")
def branch():
    m = nn.Module()
    m.cnn_pre_stages, m.cnn_ds_stages, m.cnn_up_stages = cnn.image_branch()
    return cnn_oracle.load_seeded(m.double(), seed=0).eval()


@pytest.fixture(scope="module")
def chain(branch, golden):
    """The outputs of the nine stages on the fixture's image, each stage fed its predecessor's output."""
    x = torch.from_numpy(golden["rgb"]).double()
    outs = []
    with torch.no_grad():
        for st in [branch.cnn_pre_stages] + list(branch.cnn_ds_stages) + list(branch.cnn_up_stages):
            x = st(x)
            outs.append(x.numpy())
    return outs


@pytest.mark.parametrize("k", range(9), ids=NAMES)
def test_stage_matches_reference(golden, chain, k):
    got = chain[k]
    assert got.shape == tuple(golden["shape%d" % k]), NAMES[k]
    got = got.reshape(-1)[golden["idx%d" % k]]
    want = golden["out%d" % k]
    scale = np.abs(want).max()
    err = np.abs(got - want).max()
    # float64 on both sides, from the same float32 image: only the order of the sums differs
    assert err <= 1e-9 * scale, "%s: max abs err %.3e at scale %.3e" % (NAMES[k], err, scale)


def test_state_dict_matches_reference_keys():
    with open(os.path.join(GOLDEN, "ffb6d_state_keys.json")) as fh:
        want = {k: tuple(s) for k, s in json.load(fh)}
    got = {k: tuple(v.shape) for k, v in FFB6D(n_classes=22).state_dict().items()}
    assert sorted(set(want) - set(got)) == [] and sorted(set(got) - set(want)) == []
    assert got == want
    # the part FFB6DFusionNet already had is unchanged
    base = {k: tuple(v.shape) for k, v in FFB6DFusionNet(n_classes=22).state_dict().items()}
    assert base == {k: s for k, s in want.items() if not k.startswith("cnn_")}


def test_final_and_drop_2_are_shared():
    m = FFB6D(n_classes=22)
    assert m.cnn_up_stages[2][0] is m.cnn_up_stages[3][1]
    assert m.cnn_up_stages[0][1] is m.cnn_up_stages[1][1]
    sd = m.state_dict()
    for leaf in ("weight", "bias"):
        assert sd["cnn_up_stages.2.0.0." + leaf].data_ptr() == sd["cnn_up_stages.3.1.0." + leaf].data_ptr()
    names = [n for n, _ in m.named_parameters()]
    assert "cnn_up_stages.2.0.0.weight" in names and "cnn_up_stages.3.1.0.weight" not in names


def test_unused_reference_parts_absent():
    keys = [k for k in FFB6D(n_classes=22).state_dict() if k.startswith("cnn_")]
    for bad in ("avgpool", ".fc.", "final_seg", "classifier"):
        assert not any(bad in k for k in keys), bad


def test_trunk_has_no_dilation_and_reference_strides():
    pre, ds, up = cnn.image_branch()
    convs = [m for m in list(ds[0].modules()) + list(ds[1].modules()) + list(ds[2].modules()) if isinstance(m, nn.Conv2d)]
    assert all(c.dilation == (1, 1) for c in convs)
    assert ds[0][0].downsample is None
    assert ds[1][0].downsample[0].stride == (2, 2)
    assert ds[2][0][0].downsample[0].stride == (1, 1) and ds[2][1][0].downsample[0].stride == (1, 1)
    x = torch.zeros(1, 3, 64, 96)
    with torch.no_grad():
        y = ds[2](ds[1](ds[0](pre(x))))
    assert tuple(y.shape) == (1, 512, 8, 12)


def test_construction_never_downloads(monkeypatch):
    import torch.hub
    import torch.utils.model_zoo

    def boom(*a, **k):
        raise AssertionError("network access")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", boom)
    monkeypatch.setattr(torch.utils.model_zoo, "load_url", boom)
    FFB6D(n_classes=22)


def _reference_like_state(seed):
    m = FFB6D(n_classes=22)
    g = torch.Generator().manual_seed(seed)
    return {k: (torch.randn(v.shape, generator=g) if v.dtype.is_floating_point else v.clone())
            for k, v in m.state_dict().items()}


@pytest.mark.parametrize("wrap", ["bare", "model_state"])
@pytest.mark.parametrize("prefix", ["", "module."])
@pytest.mark.parametrize("source", ["dict", "path", "buffer"])
def test_load_reference_checkpoint_round_trip(tmp_path, wrap, prefix, source):
    sd = _reference_like_state(5)
    sd["cnn_up_stages.3.1.0.weight"] = sd["cnn_up_stages.2.0.0.weight"].clone()     # one module, two keys
    sd["cnn_up_stages.3.1.0.bias"] = sd["cnn_up_stages.2.0.0.bias"].clone()
    st = {prefix + k: v for k, v in sd.items()}
    ck = {"epoch": 3, "it": 10, "best_prec": None, "model_state": st, "optimizer_state": None} if wrap == "model_state" else st
    if source == "path":
        path = str(tmp_path / "ffb6d_best.pth.tar")
        torch.save(ck, path)
        arg = path
    elif source == "buffer":
        buf = io.BytesIO()
        torch.save(ck, buf)
        buf.seek(0)
        arg = torch.load(buf, weights_only=False)
    else:
        arg = ck
    m = FFB6D(n_classes=22)
    load_reference_checkpoint(m, arg)
    got = m.state_dict()
    for k, v in sd.items():
        assert torch.equal(got[k], v), k


def test_load_reference_checkpoint_is_strict():
    sd = _reference_like_state(6)
    sd.pop("cnn_ds_stages.3.0.bottleneck.bias")
    with pytest.raises(RuntimeError, match="bottleneck.bias"):
        load_reference_checkpoint(FFB6D(n_classes=22), sd)
    sd = _reference_like_state(6)
    sd["cnn_ds_stages.3.0.final_seg.0.weight"] = torch.zeros(1)
    with pytest.raises(RuntimeError, match="final_seg"):
        load_reference_checkpoint(FFB6D(n_classes=22), sd)
