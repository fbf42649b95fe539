"""GPU: FFB6D's eval forward and its loss captured in one CUDA graph (:class:`ffb6d_b200.GraphedEvalStep`,
DESIGN.md §4.21).

Three replays on three items against eager eval of the same model, bit for bit, with and without the loss keys, for
FFB6DFusionNet (default and restructured), the whole FFB6D (PSP head and ``final`` on the kernels) and a model loaded
from a reference-shaped checkpoint; replays after eager Adam steps, ``load_state_dict`` and new running statistics,
with no new capture; alternation with :class:`ffb6d_b200.GraphedTrainStep`; an eager eval between a weight update
and a replay (the replaced cache must not be what the graph reads); re-capture; SyncBatchNorm over two gloo ranks;
and the rejections.  Items and models are those of test_gpu_graphed_step: B = 2, 120x160, 4096 points."""
import copy
import datetime
import multiprocessing as mp
import os
import sys
import traceback

import pytest
import torch
import torch.distributed as dist

import ffb6d_b200 as F
from ffb6d_b200 import _lib
from ffb6d_b200.loss import ffb6d_loss
from ffb6d_b200.model import FFB6D, load_reference_checkpoint
from test_gpu_graphed_step import N, N_CLS, N_KPS, adam, deterministic, eager_step, items, make_item, make_model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOSS_KEYS = ("labels", "kp_targ_ofst", "ctr_targ_ofst")


def eval_model(kind):
    """``make_model``'s models in eval mode; ``checkpoint``: an FFB6D loaded through ``load_reference_checkpoint``
    from what the reference's trainer saves (``{"model_state": ...}`` with DataParallel's ``module.`` prefix)."""
    if kind != "checkpoint":
        return make_model(kind).eval()
    src = make_model("ffb6d")
    ck = {"epoch": 1, "model_state": {"module." + k: v.detach().cpu() for k, v in src.state_dict().items()}}
    model = FFB6D(n_classes=N_CLS, n_pts=N, n_kps=N_KPS).cuda()
    load_reference_checkpoint(model, ck)
    return model.eval()


def eager_eval(model, item, with_loss=True):
    with torch.no_grad():
        out = model(item) if isinstance(model, FFB6D) else model(item, item["rgb_feats"])
        if not with_loss:
            return out, None, None
        loss, info = ffb6d_loss(out, item, valid=item.get("valid"))
    return out, loss, info


def flat(out):
    return [(k, out[k]) for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")] + \
           [("fused_rgb[%d]" % i, t) for i, t in enumerate(out["fused_rgb"])]


def assert_equal(got, want, when):
    out, loss, info = got
    w_out, w_loss, w_info = want
    diff = [k for (k, a), (_, b) in zip(flat(out), flat(w_out)) if not torch.equal(a, b)]
    assert diff == [], "%s: end points differ: %s" % (when, diff)
    if w_loss is None:
        assert loss is None and info is None, when
        return
    assert torch.equal(loss, w_loss), "%s: loss %r vs eager %r" % (when, loss.item(), w_loss.item())
    assert sorted(info) == sorted(w_info)
    for k in w_info:
        assert torch.equal(info[k], w_info[k]), "%s: info %s" % (when, k)


def without_loss(item):
    return {k: v for k, v in item.items() if k not in LOSS_KEYS}


# ------------------------------------------------------------------------------------------ bitwise
@pytest.mark.parametrize("with_loss", [True, False], ids=["loss", "no_loss"])
@pytest.mark.parametrize("kind", ["default", "restructured", "ffb6d", "checkpoint"])
def test_graphed_eval_bitwise_equal_eager(cuda, kind, with_loss):
    seq = items(kind in ("ffb6d", "checkpoint"))
    if not with_loss:
        seq = [without_loss(it) for it in seq]
    model = eval_model(kind)
    step = F.GraphedEvalStep(model, seq[0])
    for i, item in enumerate(seq):
        got = step(item)
        assert_equal(got, eager_eval(model, item, with_loss), "%s replay %d" % (kind, i))
    assert step.captures == 1


# ------------------------------------------------------------------------------------------ weight updates
@pytest.mark.parametrize("kind", ["restructured", "ffb6d"])
def test_weight_updates_need_no_recapture(cuda, kind):
    """Eager Adam steps, ``load_state_dict`` and new BatchNorm running statistics between replays: each next replay
    equals eager eval at the new weights, from the one capture."""
    seq = items(kind == "ffb6d")
    model = eval_model(kind)
    step = F.GraphedEvalStep(model, seq[0])
    assert_equal(step(seq[0]), eager_eval(model, seq[0]), "before any update")
    opt = adam(model, capturable=False)
    model.train()
    for item in seq[:2]:
        eager_step(model, opt, item)
    model.eval()
    assert_equal(step(seq[1]), eager_eval(model, seq[1]), "after eager Adam steps")
    other = make_model(kind).eval()          # its activations' modules are shared with the model's (default args)
    with torch.no_grad():
        for p in other.parameters():
            p.mul_(0.75)
    model.load_state_dict(other.state_dict())
    assert_equal(step(seq[2]), eager_eval(model, seq[2]), "after load_state_dict")
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
                m.running_mean.add_(0.05)
                m.running_var.mul_(1.25)
    assert_equal(step(seq[0]), eager_eval(model, seq[0]), "after new running statistics")
    assert step.captures == 1


@pytest.mark.parametrize("kind", ["restructured", "ffb6d"])
def test_eager_eval_between_update_and_replay(cuda, kind):
    """Capture with every cache warm, update the weights, run one eager eval (which replaces the caches and frees the
    packs they held), then replay: the replay packs the new weights itself.  A graph that had reused a cached pack at
    capture would compute with the weights of the capture, out of memory the eager eval released."""
    seq = items(kind == "ffb6d")
    model = eval_model(kind)
    eager_eval(model, seq[0])                           # every eval cache filled before the step is built
    step = F.GraphedEvalStep(model, seq[0])
    with torch.no_grad():
        for p in model.parameters():
            p.add_(0.01 * torch.randn_like(p))
    eager_eval(model, seq[1])
    for i in (2, 0):
        want = eager_eval(model, seq[i])
        assert_equal(step(seq[i]), want, "replay on item %d after the update" % i)
    assert step.captures == 1


def test_alternation_with_the_train_step(cuda):
    """A GraphedTrainStep and a GraphedEvalStep on one model, alternated as validation interleaves training, against
    eager training and eval of a deep copy, bit for bit under deterministic mode."""
    seq = items(False)
    with deterministic():
        mg = make_model("default")
        me = copy.deepcopy(mg)
        og, oe = adam(mg), adam(me)
        train = F.GraphedTrainStep(mg, og, seq[0])
        mg.eval()
        evaluate = F.GraphedEvalStep(mg, seq[0])
        for i in range(4):
            mg.train()
            me.train()
            loss, _ = train(seq[i % 3])
            want, _ = eager_step(me, oe, seq[i % 3])
            assert torch.equal(loss, want), "train step %d" % i
            mg.eval()
            me.eval()
            item = seq[(i + 1) % 3]
            assert_equal(evaluate(item), eager_eval(me, item), "eval after train step %d" % i)
        assert train.captures == 1 and evaluate.captures == 1


# ------------------------------------------------------------------------------------------ re-capture
def test_switches_and_module_swaps_recapture(cuda):
    seq = items(False)
    model = eval_model("default")
    step = F.GraphedEvalStep(model, seq[0], warmup=1)
    step(seq[0])
    model.restructured = True
    assert_equal(step(seq[1]), eager_eval(model, seq[1]), "restructured switched on")
    assert step.captures == 2
    with deterministic():
        assert_equal(step(seq[2]), eager_eval(model, seq[2]), "deterministic mode")
        assert step.captures == 3
    new_head = copy.deepcopy(model.rgbd_seg_layer[3])
    with torch.no_grad():
        new_head.conv.weight.mul_(0.5)
    model.rgbd_seg_layer[3] = new_head
    assert_equal(step(seq[0]), eager_eval(model, seq[0]), "swapped head")
    assert step.captures == 4
    step(seq[1])
    assert step.captures == 4


# ------------------------------------------------------------------------------------------ SyncBatchNorm
def _worker(rank, world, init_file, out_dir):
    sys.path.insert(0, ROOT)
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world,
                                timeout=datetime.timedelta(seconds=120))
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(make_model("default")).eval()
        assert dist.get_world_size() == world and any(isinstance(m, torch.nn.SyncBatchNorm) for m in model.modules())
        seq = [make_item(3 + 10 * rank, False), make_item(5 + 10 * rank, False)]
        step = F.GraphedEvalStep(model, seq[0])
        for i, item in enumerate(seq):
            assert_equal(step(item), eager_eval(model, item), "rank %d replay %d" % (rank, i))
        assert step.captures == 1
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()
        with open(os.path.join(out_dir, "rank%d.ok" % rank), "w") as fh:
            fh.write("ok")
    except BaseException:
        with open(os.path.join(out_dir, "rank%d.err" % rank), "w") as fh:
            fh.write(traceback.format_exc())
        raise


def test_sync_batchnorm_two_gloo_ranks(cuda, tmp_path):
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, 2, str(tmp_path / "pg_init"), str(tmp_path))) for r in range(2)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=600)
        errs = [(tmp_path / ("rank%d.err" % r)).read_text() for r in range(2) if (tmp_path / ("rank%d.err" % r)).exists()]
        assert not errs, "\n".join(errs)
        assert [p.exitcode for p in procs] == [0, 0]
        assert all((tmp_path / ("rank%d.ok" % r)).exists() for r in range(2))
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()


# ------------------------------------------------------------------------------------------ rejections
def test_rejects_mismatched_items(cuda):
    seq = items(False)
    model = eval_model("default")
    step = F.GraphedEvalStep(model, seq[0], warmup=1)
    bad_key = {k: v for k, v in seq[1].items() if k != "labels"}
    bad_shape = dict(seq[1], labels=seq[1]["labels"][:, :N // 2])
    bad_dtype = dict(seq[1], labels=seq[1]["labels"].long())
    bad_device = dict(seq[1], labels=seq[1]["labels"].cpu())
    bad_feat = dict(seq[1], rgb_feats=seq[1]["rgb_feats"][:7])
    for bad, what in ((bad_key, "missing"), (bad_shape, "captured for"), (bad_dtype, "captured for"),
                      (bad_device, "captured for"), (bad_feat, "missing"), ([seq[1]], "must be a dict")):
        with pytest.raises(ValueError, match="GraphedEvalStep: .*" + what):
            step(bad)
    assert step.captures == 1
    assert_equal(step(seq[1]), eager_eval(model, seq[1]), "after the rejections")
    torch.cuda.synchronize()


def test_rejects_what_cannot_be_captured(cuda, monkeypatch):
    # the library reads FFB6D_CHECK_INDICES once, at its first use: let it read it unset before the test sets it
    assert not _lib.lib.ffb6d_check_indices_enabled()
    item = make_item(3, False)
    model = make_model("default")
    with pytest.raises(ValueError, match="training mode"):
        F.GraphedEvalStep(model, item)
    model.eval()
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="FFB6D_CHECK_INDICES"):
        F.GraphedEvalStep(model, item)
    monkeypatch.delenv("FFB6D_CHECK_INDICES")
    step = F.GraphedEvalStep(model, item, warmup=1)
    monkeypatch.setenv("FFB6D_CHECK_INDICES", "1")
    with pytest.raises(ValueError, match="FFB6D_CHECK_INDICES"):
        step(item)
    monkeypatch.delenv("FFB6D_CHECK_INDICES")
    model.train()
    with pytest.raises(ValueError, match="training mode"):
        step(item)
    model.eval()
    assert step.captures == 1
    torch.cuda.synchronize()


def test_rejects_ddp(cuda, tmp_path):
    dist.init_process_group("gloo", init_method="file://%s" % (tmp_path / "store"), rank=0, world_size=1)
    try:
        model = make_model("default").eval()
        ddp = torch.nn.parallel.DistributedDataParallel(model)
        with pytest.raises(ValueError, match=r"DataParallel.*\.module"):
            F.GraphedEvalStep(ddp, make_item(3, False))
    finally:
        dist.destroy_process_group()
    torch.cuda.synchronize()
