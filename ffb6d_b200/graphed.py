"""FFB6D's training step and its eval step, each as one CUDA graph captured once and replayed per batch
(DESIGN.md §4.20, §4.21).

    opt = torch.optim.Adam(model.parameters(), lr=torch.tensor(1e-4, device="cuda"), capturable=True)
    step = GraphedTrainStep(model, opt, example_item)
    for batch in loader:
        item = build_ffb6d_item(...)
        loss, info = step(item)          # copy the item in, replay

One replay is ``opt.zero_grad()``, ``loss, info = ffb6d_loss(model(item), item, valid=item["valid"])``,
``loss.backward()``, ``opt.step()``, as eager training issues them; only the host is left out.  What capture bakes in
(the train/eval flags, the model's path switches, torch's deterministic and TF32 switches, BatchNorm momentum and
eps, dropout rates, the optimizer's non-tensor hyperparameters, ``requires_grad`` and the storage of every parameter,
buffer and gradient) is compared on the host before every replay; when any of it changed, the step captures again.

    model.eval()
    evaluate = GraphedEvalStep(model, example_item)
    end_points, loss, info = evaluate(item)     # model(item) and ffb6d_loss under torch.no_grad(), replayed

The eval step reads the weights on the device at every replay, so it follows optimizer steps, ``load_state_dict``
and graphed training steps without capturing again.
"""
import os

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.autograd.graph import increment_version

from .loss import ffb6d_loss
from .model import FFB6D, FFB6DFusionNet


# Adam's (and AdamW's) state, each created as zeros by its first step: what the warm-up's own first step created is
# zeroed after it (an optimizer whose fresh state is not zero -- NAdam's mu_product, ASGD's eta -- is rejected)
_ADAM_STATE = frozenset(("step", "exp_avg", "exp_avg_sq", "max_exp_avg_sq"))

# the item keys ffb6d_loss reads: an eval step whose example item carries them also captures the loss
_LOSS_KEYS = ("labels", "kp_targ_ofst", "ctr_targ_ofst")


def _check_indices_on():
    """Whether the gathers would run the synchronising index check: ``FFB6D_CHECK_INDICES`` set (non-empty, not "0")
    now, or when the library read it, once, at its first use (``ffb6d_check_indices_enabled``)."""
    from ._lib import lib
    v = os.environ.get("FFB6D_CHECK_INDICES")
    return (bool(v) and v != "0") or bool(lib.ffb6d_check_indices_enabled())


def _tensors(obj, path=()):
    """``(path, tensor)`` of every CUDA tensor in a dict / list / tuple tree, in a fixed order."""
    if isinstance(obj, torch.Tensor):
        return [(path, obj)] if obj.is_cuda else []
    if isinstance(obj, dict):
        return [pt for k in obj for pt in _tensors(obj[k], path + (k,))]
    if isinstance(obj, (list, tuple)):
        return [pt for i, v in enumerate(obj) for pt in _tensors(v, path + (i,))]
    return []


def _static_copy(obj):
    """The tree with every CUDA tensor replaced by a detached copy (the graph's input buffers); other values kept."""
    if isinstance(obj, torch.Tensor):
        return obj.detach().clone() if obj.is_cuda else obj
    if isinstance(obj, dict):
        return {k: _static_copy(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_static_copy(v) for v in obj)
    return obj


def _lookup(obj, path):
    for k in path:
        if isinstance(obj, dict):
            if k not in obj:
                return None
        elif not isinstance(obj, (list, tuple)) or k >= len(obj):
            return None
        obj = obj[k]
    return obj


def _state_tensors(optimizer):
    return [t for p in optimizer.state for t in optimizer.state[p].values() if isinstance(t, torch.Tensor)]


class _GraphedStep:
    """What the train and eval steps share: the argument checks, the static input buffers and their copy-in, the
    baked key of the model, the side-stream warm-up and the capture.  A subclass defines ``_check`` (what cannot be
    captured), ``_step`` (the captured work), ``_capture`` and ``__call__``; ``_module_key`` / ``_extra_key`` add
    what only it bakes in."""

    _wrapper_hint = ""

    def __init__(self, model, example_item, warmup):
        name = type(self).__name__
        self._check_model(model)
        if not isinstance(example_item, dict):
            raise ValueError("%s: example_item must be a dict, got %s" % (name, type(example_item).__name__))
        if not isinstance(model, FFB6D) and not isinstance(example_item.get("rgb_feats"), (list, tuple)):
            raise ValueError("%s: an FFB6DFusionNet item needs 'rgb_feats', the list of image-branch maps" % name)
        if int(warmup) < 1:
            raise ValueError("%s: warmup must be at least 1, got %r" % (name, warmup))
        self.model = model
        self._read_modules()
        self._check(True)
        self._static = _static_copy(example_item)
        self._inputs = _tensors(self._static)
        self._graph = None
        self._key = None
        self.captures = 0
        self._capture(int(warmup))

    def _check_model(self, model):
        name = type(self).__name__
        if isinstance(model, (nn.parallel.DistributedDataParallel, nn.DataParallel)):
            raise ValueError("%s: a (Distributed)DataParallel model cannot be captured; %s" % (name, self._wrapper_hint))
        if not isinstance(model, FFB6DFusionNet):
            raise ValueError("%s: model must be an FFB6DFusionNet or FFB6D, got %s" % (name, type(model).__name__))

    def _read_modules(self):
        """The module tree as a list, walked by every call's key (which also holds each module's children, so a
        swapped submodule changes the key and the next capture reads the tree again)."""
        self._modules = list(self.model.modules())

    def _refuse_index_check(self):
        if _check_indices_on():
            raise ValueError("%s: FFB6D_CHECK_INDICES is set; the index check synchronises the host and cannot be "
                             "captured" % type(self).__name__)

    def _module_key(self, m):
        return ()

    def _extra_key(self):
        return ()

    def _baked(self):
        """Every host value the captured step depends on, as one comparable tuple (about 0.6 ms for FFB6D)."""
        model = self.model
        key = [torch.are_deterministic_algorithms_enabled(), torch.backends.cudnn.deterministic,
               torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32,
               bool(model.restructured), bool(model.fused_lfa), bool(getattr(model, "fused_image_head", False)),
               bool(getattr(model, "fused_upsample", False))]
        for m in self._modules:
            key += (m.training, tuple(map(id, m._modules.values())))
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                key.append(m.eps)
            key += self._module_key(m)
            for p in m._parameters.values():
                if p is not None:
                    key += (id(p), p.data_ptr())
            for b in m._buffers.values():
                if b is not None:
                    key += (id(b), b.data_ptr())
        key += self._extra_key()
        return tuple(key)

    def _warm_up(self, n):
        """``n`` eager steps on a side stream, ordered after the current stream's work and before what follows it:
        cuDNN plans, the package's workspaces and its constant caches exist before capture starts."""
        dev = next(self.model.parameters()).device
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(n):
                self._step()
        torch.cuda.current_stream(dev).wait_stream(side)

    def _record(self):
        """Capture one ``_step`` into a new graph; returns its outputs, which every replay overwrites."""
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = self._step()
        self._graph = graph
        self.captures += 1
        return out

    def _copy_in(self, item):
        name = type(self).__name__
        if not isinstance(item, dict):
            raise ValueError("%s: the item must be a dict, got %s" % (name, type(item).__name__))
        pairs = []
        for path, buf in self._inputs:
            t = _lookup(item, path)
            where = "item" + "".join("[%r]" % k for k in path)
            if t is None:
                raise ValueError("%s: %s is missing" % (name, where))
            if not isinstance(t, torch.Tensor):
                raise ValueError("%s: %s must be a tensor, got %s" % (name, where, type(t).__name__))
            if t.shape != buf.shape or t.dtype != buf.dtype or t.device != buf.device:
                raise ValueError("%s: %s is %s %s on %s; the step was captured for %s %s on %s (it does not capture "
                                 "again for new shapes: build a new step)"
                                 % (name, where, tuple(t.shape), t.dtype, t.device, tuple(buf.shape), buf.dtype,
                                    buf.device))
            pairs.append((buf, t))
        for buf, t in pairs:
            if t.data_ptr() != buf.data_ptr():
                buf.copy_(t)


class GraphedTrainStep(_GraphedStep):
    """A training step of ``model`` (an :class:`~ffb6d_b200.model.FFB6DFusionNet` or
    :class:`~ffb6d_b200.model.FFB6D` in training mode) with ``optimizer``, captured in a CUDA graph.

    :param example_item: the dict one step takes, as :func:`ffb6d_b200.build_ffb6d_item` returns it (``rgb`` as a
      float tensor for :class:`FFB6D`, as its forward takes it).  :class:`FFB6DFusionNet` has no image branch: its
      item carries the eight image-branch maps as ``item["rgb_feats"]`` (a list, see ``FFB6DFusionNet.forward``).
      Every CUDA tensor in it, nested lists included, gets a static input buffer of the same shape, dtype and device;
      other values are used as they are at capture.
    :param warmup: eager steps run on a side stream before the first capture (cuDNN plans, the optimizer's state,
      the package's workspaces).  Every parameter, buffer, optimizer state tensor and the CUDA generator are then
      restored in place, so the first replay is the model's first step; state tensors the warm-up created are
      zeroed, their initial value in Adam and AdamW, the optimizers the step accepts.

    Calling the step copies the item's tensors into the input buffers on the current stream and replays the graph
    there.  It returns ``(loss, info)`` of :func:`ffb6d_b200.loss.ffb6d_loss`: the graph's output tensors, which the
    next replay overwrites (clone what you keep).  ``captures`` counts the captures so far.  Every call compares what
    capture baked in (DESIGN.md §4.20), the model's module tree included: a submodule or parameter swapped after
    construction makes the next call capture again, with the new modules.

    Rejected with ``ValueError``: a ``DistributedDataParallel`` / ``DataParallel`` wrapper or an ``nn.SyncBatchNorm``
    that synchronises over more than one rank (a captured step would hold collectives); a BatchNorm with
    ``momentum=None`` (its factor is read from ``num_batches_tracked`` on the host); an optimizer other than
    ``torch.optim.Adam`` / ``AdamW``, or a param group without ``capturable=True``; ``FFB6D_CHECK_INDICES`` set now or
    when the library loaded (the index check synchronises); a model in eval mode.
    """

    _wrapper_hint = "multi-rank capture is not supported, pass the module of a single-rank run"

    def __init__(self, model, optimizer, example_item, warmup=3):
        self.optimizer = optimizer
        self._loss = self._info = None
        self._written = []
        super().__init__(model, example_item, warmup)

    # ------------------------------------------------------------------------------------------ host checks
    def _read_modules(self):
        super()._read_modules()
        self._sync = any(isinstance(m, nn.SyncBatchNorm) for m in self._modules)

    def _check(self, modules):
        """What cannot be captured at all: raise ``ValueError`` before any CUDA work.  ``modules``: also walk the
        BatchNorms (momentum=None, SyncBatchNorm over several ranks)."""
        model, opt = self.model, self.optimizer
        if not model.training:
            raise ValueError("GraphedTrainStep: the model is in eval mode; it captures training steps only")
        self._refuse_index_check()
        if not isinstance(opt, torch.optim.Adam):      # AdamW is an Adam
            raise ValueError("GraphedTrainStep: the optimizer must be torch.optim.Adam or AdamW, got %s (the warm-up "
                             "is undone by restoring Adam's zero initial state)" % type(opt).__name__)
        for i, g in enumerate(opt.param_groups):
            if not g.get("capturable", False):
                raise ValueError("GraphedTrainStep: optimizer param group %d needs capturable=True" % i)
        if not modules:
            return
        multi_rank = dist.is_available() and dist.is_initialized()
        for name, m in model.named_modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                if m.momentum is None:
                    raise ValueError("GraphedTrainStep: BatchNorm %r has momentum=None (a cumulative average read "
                                     "from num_batches_tracked on the host); give it a float momentum" % name)
                if isinstance(m, nn.SyncBatchNorm) and multi_rank:
                    group = m.process_group if m.process_group is not None else dist.group.WORLD
                    if dist.get_world_size(group) > 1:
                        raise ValueError("GraphedTrainStep: SyncBatchNorm %r synchronises over several ranks; "
                                         "multi-rank capture is not supported" % name)

    def _module_key(self, m):
        """BatchNorm momentum, dropout rates, and ``requires_grad`` and the gradient storage of every parameter."""
        key = []
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            if m.momentum is None:
                self._check(True)                  # raises, naming the layer
            key.append(m.momentum)
        elif isinstance(m, nn.modules.dropout._DropoutNd):
            key.append(m.p)
        for p in m._parameters.values():
            if p is not None:
                g = p.grad
                key += (p.requires_grad, id(g), g.data_ptr() if g is not None else 0)
        return key

    def _extra_key(self):
        """The optimizer's hyperparameters (it reads the keys of its defaults, not e.g. initial_lr)."""
        opt, key = self.optimizer, []
        for group in opt.param_groups:
            key.append(tuple(id(p) for p in group["params"]))
            for k in sorted(opt.defaults):
                v = group.get(k)
                if isinstance(v, torch.Tensor):      # a tensor lr: read on the device, only its storage is baked
                    key += (k, id(v), v.data_ptr())
                else:
                    key += (k, v)
        return key

    # ------------------------------------------------------------------------------------------ capture
    def _step(self):
        opt, item = self.optimizer, self._static
        opt.zero_grad(set_to_none=True)
        out = self.model(item) if isinstance(self.model, FFB6D) else self.model(item, item["rgb_feats"])
        loss, info = ffb6d_loss(out, item, valid=item.get("valid"))
        loss.backward()
        opt.step()
        return loss.detach(), info

    def _capture(self, warmup):
        """Warm up on a side stream, restore everything the warm-up changed, then capture one step."""
        model, opt = self.model, self.optimizer
        self._graph = self._loss = self._info = None     # release the previous graph's pool before the new one fills
        self._written = []
        self._read_modules()
        self._check(True)
        opt.zero_grad(set_to_none=True)
        dev = next(model.parameters()).device
        tracked = list(model.parameters()) + list(model.buffers())
        before = {id(t): t for t in _state_tensors(opt)}
        had_state = {p for p in opt.state if opt.state[p]}
        saved = [t.detach().clone() for t in tracked]
        saved_state = {k: t.detach().clone() for k, t in before.items()}
        rng = torch.cuda.get_rng_state(dev)
        self._warm_up(warmup)
        with torch.no_grad():
            for t, s in zip(tracked, saved):
                t.copy_(s)
            unknown = sorted({k for p, st in opt.state.items() for k, t in st.items() if isinstance(t, torch.Tensor)
                              and not (id(t) in before and before[id(t)] is t) and k not in _ADAM_STATE})
            for p, st in opt.state.items():
                for k, t in st.items():
                    if not isinstance(t, torch.Tensor):
                        continue
                    if id(t) in before and before[id(t)] is t:
                        t.copy_(saved_state[id(t)])
                    else:
                        t.zero_()
        torch.cuda.set_rng_state(rng, dev)
        if unknown:              # a subclass of Adam with state of its own: drop what the warm-up created, refuse
            for p in [p for p in opt.state if p not in had_state]:
                del opt.state[p]
            raise ValueError("GraphedTrainStep: the optimizer created state %s whose initial value is not known to be "
                             "zero; only Adam's own state can be restored after the warm-up" % (unknown,))
        del saved, saved_state
        opt.zero_grad(set_to_none=True)
        self._loss, self._info = self._record()
        # what a replay writes: its host version counters are advanced after each replay, as eager in-place
        # updates advance them, so version-keyed caches (the eval path's packed weights) see the new values
        self._written = (tracked + _state_tensors(opt) +
                         [p.grad for p in model.parameters() if p.grad is not None])
        self._key = self._baked()

    # ------------------------------------------------------------------------------------------ a step
    def __call__(self, item):
        self._check(self._sync)
        self._copy_in(item)
        if self._baked() != self._key:
            self._capture(1)
        self._graph.replay()
        increment_version(self._written)
        return self._loss, self._info


class GraphedEvalStep(_GraphedStep):
    """An eval step of ``model`` (an :class:`~ffb6d_b200.model.FFB6DFusionNet` or :class:`~ffb6d_b200.model.FFB6D`
    in eval mode), captured in a CUDA graph: under ``torch.no_grad()``, ``model(item)`` (``model(item,
    item["rgb_feats"])`` for :class:`FFB6DFusionNet`) and, when the example item carries ``labels``,
    ``kp_targ_ofst`` and ``ctr_targ_ofst``, ``ffb6d_loss(end_points, item, valid=item.get("valid"))``, as
    ``model_fn`` computes them with ``is_eval=True``.

    :param example_item: as for :class:`GraphedTrainStep`; every CUDA tensor in it gets a static input buffer.
    :param warmup: eager eval steps run on a side stream before the first capture.  Eval writes no parameter or
      buffer, so nothing is restored after them.

    Calling the step copies the item's tensors into the input buffers and replays the graph on the current stream.
    It returns ``(end_points, loss, info)``: the network's outputs and :func:`ffb6d_b200.loss.ffb6d_loss`'s
    ``(loss, info)``, or ``None, None`` without the loss keys.  They are the graph's tensors, which the next replay
    overwrites (clone what you keep).

    Every pack of weights or running statistics is made inside the graph, so each replay reads the parameters and
    buffers as they are then: optimizer steps, ``load_state_dict``, new running statistics and
    :class:`GraphedTrainStep` replays between calls need no new capture.  What capture bakes in is compared before
    every replay (DESIGN.md §4.21): the module tree and every module's ``training``, ``restructured``,
    ``fused_lfa``, ``fused_image_head``, ``fused_upsample``, torch's deterministic, cuDNN and TF32 switches, BatchNorm ``eps``, and the
    identity and storage of every parameter and buffer; any change captures again (``captures`` counts).

    Rejected with ``ValueError``: a model in training mode; a ``DistributedDataParallel`` / ``DataParallel`` wrapper
    (pass its ``.module``); ``FFB6D_CHECK_INDICES`` set now or when the library loaded; an item whose keys, shapes,
    dtypes or devices differ from the example's.  An ``nn.SyncBatchNorm`` over several ranks is accepted: in eval mode
    it normalises with its running statistics and issues no collective, so each rank can evaluate through its own
    step.
    """

    _wrapper_hint = "pass its .module (each rank evaluates through a step of its own)"

    def __init__(self, model, example_item, warmup=3):
        self._out = None
        self._with_loss = isinstance(example_item, dict) and all(k in example_item for k in _LOSS_KEYS)
        super().__init__(model, example_item, warmup)

    def _check(self, modules=False):
        """What cannot be captured at all: raise ``ValueError`` before any CUDA work."""
        if self.model.training:
            raise ValueError("GraphedEvalStep: the model is in training mode; call model.eval() first, it captures "
                             "eval steps only")
        self._refuse_index_check()

    def _step(self):
        item = self._static
        with torch.no_grad():
            out = self.model(item) if isinstance(self.model, FFB6D) else self.model(item, item["rgb_feats"])
            loss = info = None
            if self._with_loss:
                loss, info = ffb6d_loss(out, item, valid=item.get("valid"))
        return out, loss, info

    def _capture(self, warmup):
        self._graph = self._out = None     # release the previous graph's pool before the new one fills
        self._read_modules()
        self._check()
        self._warm_up(warmup)
        self._out = self._record()
        self._key = self._baked()

    def __call__(self, item):
        self._check()
        self._copy_in(item)
        if self._baked() != self._key:
            self._capture(1)
        self._graph.replay()
        return self._out
