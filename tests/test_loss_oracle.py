"""CPU: the loss oracle (float64 numpy and float32 torch restatements) against the reference's own models/loss.py,
as recorded in tests/golden/loss_cases.npz by tests/golden/make_loss_golden.py."""
import os

import numpy as np
import pytest
import torch

from oracle import loss_oracle as O

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_cases.npz"))


def _case_names(kind):
    return sorted({k.split("/")[1] for k in G.files if k.startswith(kind + "/")})


def case(kind, name):
    p = "%s/%s/" % (kind, name)
    return {k[len(p):]: G[k] for k in G.files if k.startswith(p)}


def alpha_of(c):
    return [None, float(c["alpha"][0]), list(c["alpha"])][int(c["alpha_kind"])]


def rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


def test_fixture_covers_the_cases():
    assert len(_case_names("focal")) >= 9 and len(_case_names("of")) >= 6 and len(_case_names("model")) >= 3


@pytest.mark.parametrize("name", _case_names("focal"))
def test_focal_oracle(name):
    c = case("focal", name)
    loss, _, grad = O.focal_loss(c["logits"], c["labels"], float(c["gamma"]), alpha_of(c), bool(c["size_average"]),
                                 grad_loss=float(c["g"]))
    assert rel(loss, c["loss"]) <= 1e-5
    assert np.abs(grad - c["grad"]).max() <= 1e-6 * abs(float(c["g"]))


@pytest.mark.parametrize("name", _case_names("focal"))
def test_focal_torch_restatement(name):
    c = case("focal", name)
    x = torch.tensor(c["logits"], requires_grad=True)
    loss = O.focal_loss_torch(x, torch.from_numpy(c["labels"]), float(c["gamma"]), alpha_of(c),
                              bool(c["size_average"]))
    loss.backward(torch.tensor(float(c["g"])))
    assert rel(loss.item(), c["loss"]) <= 1e-6
    assert np.abs(x.grad.numpy() - c["grad"]).max() <= 1e-6 * abs(float(c["g"]))


def test_focal_arg_max_takes_the_lowest_class_on_ties():
    c = case("focal", "extreme")
    rows = c["logits"][0].T
    _, acc, _ = O.focal_loss(c["logits"], c["labels"], 2.0)
    assert acc == np.mean(rows.argmax(1) == c["labels"][0])
    assert (torch.from_numpy(rows).max(1)[1].numpy() == rows.argmax(1)).all()
    assert rows[:20].argmax(1).max() == 0


@pytest.mark.parametrize("name", _case_names("of"))
def test_of_oracle(name):
    c = case("of", name)
    out = O.of_l1_loss(c["pred"], c["targ"], c["labels"])
    assert np.all(np.abs(out - c["out"]) <= 1e-5 * np.maximum(np.abs(c["out"]), 1e-30))
    g = O.of_l1_grad_f32(c["pred"], c["targ"], c["labels"], c["g"])
    assert np.array_equal(g.view(np.uint32), c["grad"].view(np.uint32))     # bitwise, signed zeros included


def test_of_frame_without_positive_labels_is_zero():
    c = case("of", "no_positive")
    assert np.all(c["out"][1] == 0) and np.all(c["grad"][1] == 0)
    assert np.all(O.of_l1_loss(c["pred"], c["targ"], c["labels"])[1] == 0)


@pytest.mark.parametrize("name", _case_names("of"))
def test_of_torch_restatement(name):
    c = case("of", name)
    p = torch.tensor(c["pred"], requires_grad=True)
    K = p.shape[1]
    out = O.of_l1_loss_torch(p, torch.from_numpy(c["targ"]).reshape(p.shape[0], -1, K, 3),
                             torch.from_numpy(c["labels"]).long().reshape(p.shape[0], -1))
    out.backward(torch.from_numpy(c["g"]))
    assert np.array_equal(out.detach().numpy(), c["out"])
    assert np.array_equal(p.grad.numpy().view(np.uint32), c["grad"].view(np.uint32))


KEYS = ("loss_rgbd_seg", "loss_kp_of", "loss_ctr_of", "loss_all", "acc_rgbd")


def _model_inputs(c):
    ep = {k: c[k] for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")}
    item = {k: c[k] for k in ("labels", "kp_targ_ofst", "ctr_targ_ofst")}
    return ep, item


@pytest.mark.parametrize("name", _case_names("model"))
def test_model_block_oracle(name):
    c = case("model", name)
    ep, item = _model_inputs(c)
    got = O.ffb6d_loss(ep, item, valid=c["valid"])
    for k in KEYS:
        assert rel(got[k], c[k]) <= 1e-5, k


@pytest.mark.parametrize("name", _case_names("model"))
def test_model_block_torch_restatement(name):
    c = case("model", name)
    ep, item = _model_inputs(c)
    ep = {k: torch.tensor(a, requires_grad=True) for k, a in ep.items()}
    loss, info = O.ffb6d_loss_torch(ep, {k: torch.from_numpy(a) for k, a in item.items()},
                                    valid=torch.from_numpy(c["valid"]))
    loss.backward()
    for k in KEYS:
        assert rel(info[k].item(), c[k]) <= 1e-6, k
    for k in ("pred_kp_ofs", "pred_ctr_ofs"):
        # equal values; the backward of the boolean indexing adds into zeros, which turns the reference's -0 into +0
        assert np.array_equal(ep[k].grad.numpy(), c["grad_" + k]), k
    assert np.abs(ep["pred_rgbd_segs"].grad.numpy() - c["grad_pred_rgbd_segs"]).max() <= 1e-6


def test_masked_frames_have_zero_gradients_in_the_fixture():
    c = case("model", "lm_masked")
    v = c["valid"]
    assert not v.all() and v.any()
    for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs"):
        assert np.all(c["grad_" + k][~v] == 0)
