"""CPU: the float64 restatements the GPU tests trust (tests/ffb6d_restatement.py) against the reference's own
``FFB6D``, whole network, forward and one training step.

``ffb6d_net_cases.npz`` (tests/golden/make_ffb6d_golden.py) holds the reference's outputs, run in float64 and in
float32 on two 120x160 frames with 4096 points, with the seeded weights and inputs of oracle/net_oracle.py: every
stage of the eval forward, and of one training step (dropouts off) the losses, the ``end_points``, the gradient of
every parameter and the updated running statistics, each at sampled positions.  ``FullRef`` in float64 from the same
state dict must reproduce them to summation order, stage by stage, so the first stage that differs is the one named;
a restatement with one wiring edit must be caught at the stage of the edit."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from ffb6d_b200.model import FFB6D, load_reference_checkpoint
from ffb6d_b200.tables import knn_schedule
from ffb6d_restatement import FullRef, first_divergence, unit
from oracle import loss_oracle, net_oracle as N


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "ffb6d_net_cases.npz")))


@pytest.fixture(scope="module")
def data(golden):
    d = N.make_inputs()
    N.check_inputs(d, golden)
    return d


@pytest.fixture(scope="module")
def inputs(golden, data):
    idx = N.oracle_indices(data)
    N.check_indices(idx, golden)
    return N.network_inputs(data, idx, dtype=torch.float64)


@pytest.fixture(scope="module")
def model():
    return FFB6D(n_classes=N.N_CLASSES, n_pts=N.N_POINTS, n_kps=N.N_KPS)


def eval_stages(ref, inputs):
    """``{name: output}`` of every stage and end point of ``ref``'s eval forward."""
    ref.trace = []
    with torch.no_grad():
        out = ref.forward(inputs, inputs["rgb"])
    return dict(ref.trace, **{k: out[k] for k in N.END_POINTS})


def test_inputs_match_fixture_digests(golden, data):
    assert sorted(k[7:] for k in golden if k.startswith("digest/")) == sorted(N.INPUT_KEYS)


def test_cpu_oracle_reproduces_reference_indices(golden, data):
    idx = N.oracle_indices(data)
    assert sorted(idx) == sorted(c[0] for c in knn_schedule(N.N_POINTS, N.H, N.W))
    N.check_indices(idx, golden)
    bad = dict(idx, cld_interp_idx2=idx["cld_interp_idx2"][:, ::-1].copy())
    with pytest.raises(AssertionError, match="cld_interp_idx2"):
        N.check_indices(bad, golden)


def test_eval_forward_matches_reference_stage_by_stage(golden, inputs, model):
    stored = N.unpack(golden, "eval", N.STAGE_SAMPLES)
    assert len(stored) == 46 + 3
    got = eval_stages(FullRef(model, N.eval_tensors(model.state_dict(), golden), N.N_KPS), inputs)
    assert sorted(got) == sorted(stored)
    # float64 on both sides, from the same float32 inputs and weights: only the order of the sums differs
    first, worst = first_divergence(got, stored, N.STAGE_SEED, N.STAGE_SAMPLES, lambda e32: 1e-9)
    assert first is None, first


class Miswired(FullRef):
    """FullRef with one wiring edit in the first fusion; every index stays in range, every shape the same."""

    def __init__(self, edit, *a):
        super().__init__(*a)
        self.edit = edit

    def fuse(self, tag, i, rgb0, p0, p2r_idx, r2p_idx):
        if (tag, i) != ("ds", 0):
            return super().fuse(tag, i, rgb0, p0, p2r_idx, r2p_idx)
        bs, c, hr, wr = rgb0.shape
        p2r = self.nearest(self.note("ds_fuse_p2r_pre_layers.0", self.fconv("ds_fuse_p2r_pre_layers.0", p0)), p2r_idx)
        rgb = self.note("ds_fuse_p2r_fuse_layers.0",
                        self.fconv("ds_fuse_p2r_fuse_layers.0", torch.cat((rgb0, p2r.view(bs, -1, hr, wr)), 1)))
        src = rgb if self.edit == "r2p_from_fused_map" else rgb0
        r2p = self.note("ds_fuse_r2p_pre_layers.0",
                        self.fconv("ds_fuse_r2p_pre_layers.0", self.random_sample(src.reshape(bs, c, hr * wr, 1), r2p_idx)))
        cat = (r2p, p0) if self.edit == "r2p_concat_swapped" else (p0, r2p)
        return rgb, self.note("ds_fuse_r2p_fuse_layers.0", self.fconv("ds_fuse_r2p_fuse_layers.0", torch.cat(cat, 1)))


@pytest.mark.parametrize("edit,stage", [("r2p_from_fused_map", "ds_fuse_r2p_pre_layers.0"),
                                        ("r2p_concat_swapped", "ds_fuse_r2p_fuse_layers.0")])
def test_one_wiring_edit_is_caught_at_its_stage(golden, inputs, model, edit, stage):
    stored = N.unpack(golden, "eval", N.STAGE_SAMPLES)
    got = eval_stages(Miswired(edit, model, N.eval_tensors(model.state_dict(), golden), N.N_KPS), inputs)
    # at the float64 bound, and at the bound the float32 network is held to
    for bound in (lambda e32: 1e-9, lambda e32: max(5e-5, 4 * e32)):
        first, _ = first_divergence(got, stored, N.STAGE_SEED, N.STAGE_SAMPLES, bound)
        assert first is not None and first.startswith(stage + " is the first stage"), first


def test_training_step_matches_reference(golden, data, inputs, model):
    ref = FullRef(model, N.seeded_tensors(model.state_dict()), N.N_KPS, train=True)
    out = ref.forward(inputs, inputs["rgb"])
    loss, info = loss_oracle.ffb6d_loss_torch(out, N.targets(data, dtype=torch.float64))
    loss.backward()
    for k, want in zip(N.LOSSES, golden["train/loss"]):
        assert abs(info[k].item() - want) <= 1e-9 * abs(want), (k, info[k].item(), want)
    first, _ = first_divergence(out, N.unpack(golden, "train/out", N.STAGE_SAMPLES), N.STAGE_SEED, N.STAGE_SAMPLES,
                                lambda e32: 1e-9)
    assert first is None, first
    # gradients: every parameter of the reference, by norm and at the sampled positions, against its layer's scale
    grads = {k: v.grad for k, v in ref.p.items() if v.requires_grad}
    grads.update({k: v.grad for k, v in ref.cnn.named_parameters() if k.startswith("cnn_")})
    stored = N.unpack(golden, "train/grad", N.PARAM_SAMPLES)
    assert sorted(grads) == sorted(stored)
    scale = {}
    for name, e in stored.items():
        scale[unit(name)] = max(scale.get(unit(name), 1e-12), e["norm"])
    for name, e in stored.items():
        g = grads[name]
        assert g is not None and tuple(g.shape) == e["shape"], name
        err = np.linalg.norm(N.sample(g, N.GRAD_SEED + e["k"], N.PARAM_SAMPLES) - e["f64"])
        assert err <= 1e-8 * scale[unit(name)] and abs(g.norm().item() - e["norm"]) <= 1e-8 * scale[unit(name)], \
            "grad %s: %.3e of its layer's gradient scale" % (name, err / scale[unit(name)])
    # running statistics after the step
    after = dict(ref.after, **{k: v for k, v in ref.cnn.state_dict().items() if k.startswith("cnn_")})
    stored = N.unpack(golden, "train/stat", N.PARAM_SAMPLES)
    assert sorted(stored) == sorted(N.running_keys(model.state_dict()))
    for name, e in stored.items():
        err = np.abs(N.sample(after[name], N.STAT_SEED + e["k"], N.PARAM_SAMPLES) - e["f64"]).max()
        assert err <= 1e-9 * max(np.abs(e["f64"]).max(), 1e-3), "%s after the step: %.3e" % (name, err)
    assert (golden["train/num_batches_tracked"] == 1).all()
    assert all(int(v) == 1 for k, v in ref.cnn.state_dict().items() if k.startswith("cnn_") and k.endswith("tracked"))


def test_seeded_checkpoint_loads_through_reference_loader(model):
    sd = N.seeded_tensors(model.state_dict())
    assert "cnn_up_stages.2.0.0.weight" in sd and torch.equal(sd["cnn_up_stages.3.1.0.weight"], sd["cnn_up_stages.2.0.0.weight"])
    m = FFB6D(n_classes=N.N_CLASSES, n_pts=N.N_POINTS, n_kps=N.N_KPS)
    load_reference_checkpoint(m, {"epoch": 1, "model_state": {"module." + k: v for k, v in sd.items()}})
    got = m.state_dict()
    assert list(got) == list(sd)
    for k, v in sd.items():
        assert got[k].dtype == v.dtype and torch.equal(got[k], v), k
