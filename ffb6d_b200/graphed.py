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

    step = GraphedFrameTrainStep(model, opt, example_batch, dataset="ycb", cam_scale=10000.0, K=K)
    for it, batch in enumerate(loader):
        loss, info = step(batch, seed=it)     # build_ffb6d_train_item and the training step, replayed

:class:`GraphedFrameTrainStep` also captures the training ``get_item`` (DESIGN.md §4.28): the augmentation, the
depth completion, the sampling, the 22 searches and the point arrays, from the collated batch's decoded frames.
"""
import os

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
from torch.autograd.graph import increment_version

from . import ops
from .loss import ffb6d_loss
from .model import FFB6D, FFB6DFusionNet
from .schedule import TRAIN_RECORD_KEYS, _train_item, check_fuse_batch, check_render_batch, check_train_batch


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


def _check_image_branch(model, name):
    """``ValueError`` for an :class:`FFB6DFusionNet` that is not a whole :class:`FFB6D`: work that starts from decoded
    frames needs the image branch."""
    if isinstance(model, FFB6DFusionNet) and not isinstance(model, FFB6D):
        raise ValueError("%s: an FFB6DFusionNet has no image branch; working from decoded frames needs the whole FFB6D"
                         % name)


def _forward(model, item):
    """``model(item)``; an :class:`FFB6DFusionNet` also takes the item's image-branch maps."""
    return model(item) if isinstance(model, FFB6D) else model(item, item["rgb_feats"])


class _GraphedStep:
    """What every graphed step shares: the argument checks, the static input buffers and their copy-in, the baked key
    of the model, the side-stream warm-up, the capture and the replay.  A subclass defines ``_check`` (what cannot be
    captured) and ``_step`` (the captured work); ``_module_key`` / ``_extra_key`` add what only it bakes in,
    ``_warm_up`` what a warm-up must undo and ``_writes`` the tensors a replay writes in place.

    Each subclass's constructor checks the model with :meth:`_check_model` first, before its own checks and any CUDA
    work, and then calls this one."""

    _wrapper_hint = ""
    _needs_image_branch = False      # the step starts from decoded frames: an FFB6DFusionNet is rejected
    _keys = None                     # the keys of a flat batch, checked by every call (see _check_keys)

    def __init__(self, model, example_item, warmup):
        name = type(self).__name__
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
        self._graph = self._out = self._key = None
        self._written = []
        self.captures = 0
        self._capture(int(warmup))

    def _check_model(self, model):
        name = type(self).__name__
        if isinstance(model, (nn.parallel.DistributedDataParallel, nn.DataParallel)):
            raise ValueError("%s: a (Distributed)DataParallel model cannot be captured; %s" % (name, self._wrapper_hint))
        if not isinstance(model, FFB6DFusionNet):
            raise ValueError("%s: model must be an FFB6DFusionNet or FFB6D, got %s" % (name, type(model).__name__))
        if self._needs_image_branch:
            _check_image_branch(model, name)

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

    def _writes(self):
        """The tensors a replay updates in place whose host version counters it advances (none for an eval step)."""
        return []

    def _capture(self, warmup):
        """Warm up on a side stream (undoing what the warm-up changed, see ``_warm_up``), then capture one step."""
        self._graph = self._out = None     # release the previous graph's pool before the new one fills
        self._written = []
        self._read_modules()
        self._check(True)
        self._warm_up(warmup)
        self._out = self._record()
        self._written = self._writes()
        self._key = self._baked()

    def _replay(self):
        """Capture again if a baked value changed, then replay; returns the graph's outputs."""
        if self._baked() != self._key:
            self._capture(1)
        self._graph.replay()
        if self._written:
            # as eager in-place updates advance them, so version-keyed caches (the eval path's packs) see new values
            increment_version(self._written)
        return self._out

    def _check_keys(self, batch):
        """A step built from a flat batch takes batches with the example's keys only."""
        if self._keys is not None and (not isinstance(batch, dict) or set(batch) != self._keys):
            raise ValueError("%s: the batch holds keys %s; the step was captured for %s"
                             % (type(self).__name__,
                                sorted(map(str, batch)) if isinstance(batch, dict) else type(batch).__name__,
                                sorted(map(str, self._keys))))

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
        self._check_model(model)
        self.optimizer = optimizer
        super().__init__(model, example_item, warmup)

    # ------------------------------------------------------------------------------------------ host checks
    def _read_modules(self):
        super()._read_modules()
        self._sync = any(isinstance(m, nn.SyncBatchNorm) for m in self._modules)

    def _check(self, modules):
        """What cannot be captured at all: raise ``ValueError`` before any CUDA work.  ``modules``: also walk the
        BatchNorms (momentum=None, SyncBatchNorm over several ranks)."""
        model, opt, name = self.model, self.optimizer, type(self).__name__
        if not model.training:
            raise ValueError("%s: the model is in eval mode; it captures training steps only" % name)
        self._refuse_index_check()
        if not isinstance(opt, torch.optim.Adam):      # AdamW is an Adam
            raise ValueError("%s: the optimizer must be torch.optim.Adam or AdamW, got %s (the warm-up is undone by "
                             "restoring Adam's zero initial state)" % (name, type(opt).__name__))
        for i, g in enumerate(opt.param_groups):
            if not g.get("capturable", False):
                raise ValueError("%s: optimizer param group %d needs capturable=True" % (name, i))
        if not modules:
            return
        multi_rank = dist.is_available() and dist.is_initialized()
        for name, m in model.named_modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                if m.momentum is None:
                    raise ValueError("%s: BatchNorm %r has momentum=None (a cumulative average read from "
                                     "num_batches_tracked on the host); give it a float momentum" % (type(self).__name__,
                                                                                                     name))
                if isinstance(m, nn.SyncBatchNorm) and multi_rank:
                    group = m.process_group if m.process_group is not None else dist.group.WORLD
                    if dist.get_world_size(group) > 1:
                        raise ValueError("%s: SyncBatchNorm %r synchronises over several ranks; multi-rank capture "
                                         "is not supported" % (type(self).__name__, name))

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
        return self._train(self._static)

    def _train(self, item):
        """One training step on ``item``: what a replay runs."""
        opt = self.optimizer
        opt.zero_grad(set_to_none=True)
        loss, info = ffb6d_loss(_forward(self.model, item), item, valid=item.get("valid"))
        loss.backward()
        opt.step()
        return loss.detach(), info

    def _warm_up(self, n):
        """The warm-up, then every parameter, buffer and optimizer state tensor and the CUDA generator restored."""
        model, opt = self.model, self.optimizer
        opt.zero_grad(set_to_none=True)
        dev = next(model.parameters()).device
        tracked = list(model.parameters()) + list(model.buffers())
        before = {id(t): t for t in _state_tensors(opt)}
        had_state = {p for p in opt.state if opt.state[p]}
        saved = [t.detach().clone() for t in tracked]
        saved_state = {k: t.detach().clone() for k, t in before.items()}
        rng = torch.cuda.get_rng_state(dev)
        super()._warm_up(n)
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
            raise ValueError("%s: the optimizer created state %s whose initial value is not known to be zero; only "
                             "Adam's own state can be restored after the warm-up" % (type(self).__name__, unknown))
        del saved, saved_state
        opt.zero_grad(set_to_none=True)

    def _writes(self):
        model = self.model
        return (list(model.parameters()) + list(model.buffers()) + _state_tensors(self.optimizer) +
                [p.grad for p in model.parameters() if p.grad is not None])

    # ------------------------------------------------------------------------------------------ a step
    def __call__(self, item):
        self._check(self._sync)
        self._copy_in(item)
        return self._replay()


class GraphedFrameTrainStep(GraphedTrainStep):
    """:func:`ffb6d_b200.build_ffb6d_train_item` and a :class:`GraphedTrainStep` training step of an
    :class:`~ffb6d_b200.model.FFB6D`, captured in one CUDA graph and replayed per batch: the colour jitter, both
    ``rgb_add_noise`` passes, ``add_real_back``, the depth completion (YCB), the sampling, the 22 searches and the
    point arrays, then ``zero_grad``, the forward, ``ffb6d_loss``, the backward and ``optimizer.step()``.

    :param example_batch: a batch as :func:`~ffb6d_b200.build_ffb6d_train_item` takes it.  Its CUDA tensors (the
      images, the background frames, the object tables, a per-frame ``K``) get static input buffers, as
      :class:`GraphedTrainStep`'s item does; its host values (the worker's ``jitter``, ``jittered``, ``plans``,
      ``augment``, ``apply_rgb``, and any other entry that is not a CUDA tensor) get device buffers that every call
      fills through pinned staging memory.  Later batches must have the same keys, and each entry the same kind
      (CUDA or host), shape and dtype.
    :param warmup: eager steps before the first capture, undone as :class:`GraphedTrainStep` undoes them.

    Baked in at construction: ``dataset``, ``cam_scale``, ``n_points``, ``normals`` (as
    :func:`~ffb6d_b200.build_ffb6d_train_item` takes it; with ``"device"`` batches hold no ``nrm_map``), ``meshes`` (a
    :class:`~ffb6d_b200.render.RenderMeshTable`, LineMOD with ``normals="device"``: batches then hold the render keys,
    host draws or CUDA tensors, and the flagged frames are rendered into the step's input buffers before the colour
    jitter), ``crops`` (a :class:`~ffb6d_b200.fuse_frames.FuseCropTable`, LineMOD with ``normals="device"``: batches
    then hold the fuse keys and a per-frame ``K``, and the flagged frames' crops are pasted into the step's input
    buffers after the renders) and ``K``
    (copied to the device once; with ``batch['K']`` the per-frame matrices are inputs instead).  Everything else that capture bakes in, and every rule
    that captures again, rejects or restores, is :class:`GraphedTrainStep`'s (DESIGN.md §4.20).

    ``step(batch, seed)`` checks the batch's jitter plans and noise records on the host (a bad one raises
    :class:`~ffb6d_b200._lib.FFB6DError` before anything is copied), copies the host values and ``seed`` (an int in
    [0, 2^64), or a one-element int64 / uint64 CUDA tensor) through pinned buffers without synchronising the host,
    copies the CUDA tensors into the input buffers on the current stream, and replays.  It returns ``(loss, info)``
    of :func:`ffb6d_b200.loss.ffb6d_loss`: the graph's tensors, which the next replay overwrites.  The replay equals
    ``build_ffb6d_train_item`` with that seed followed by an eager training step, bit for bit.

    Rejected with ``ValueError``: what :class:`GraphedTrainStep` rejects; an :class:`FFB6DFusionNet` (its image maps
    do not come from frames); a batch whose keys, or an entry's kind, shape, dtype or device, differ from the example.
    """

    _needs_image_branch = True
    _STAGING_SLOTS = 2

    def __init__(self, model, optimizer, example_batch, *, dataset, cam_scale, K, n_points=12800, warmup=3,
                 normals="input", meshes=None, crops=None):
        name = type(self).__name__
        self._check_model(model)
        check_train_batch(example_batch, dataset, name, normals, meshes, crops)
        self.dataset, self.cam_scale, self.n_points, self.normals = dataset, cam_scale, int(n_points), normals
        self.meshes, self.crops = meshes, crops
        self._keys = set(example_batch)
        dev = next(model.parameters()).device
        device_part = {k: v for k, v in example_batch.items() if isinstance(v, torch.Tensor) and v.is_cuda}
        host = self._host_values(example_batch, None)
        B = example_batch["rgb"].shape[0]
        self._intr = None if "K" in example_batch else ops._intrinsics_arg(K, B, dev)[0]
        # the device buffers of the host values and of the seed, and the pinned slots they are copied from in turn
        self._records = {k: torch.empty(t.shape, dtype=t.dtype, device=dev) for k, t in host.items()}
        self._seed = torch.zeros(1, dtype=torch.int64, device=dev)
        self._pinned = [dict({k: torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for k, t in host.items()},
                             _seed=torch.empty(1, dtype=torch.int64, pin_memory=True))
                        for _ in range(self._STAGING_SLOTS)]
        self._staged = [None] * self._STAGING_SLOTS
        self._slot = 0
        self._check_records(host)
        self._stage(host, 0)
        self._mirror = {k: host[k].numpy().copy() for k in ("jitter", "plans")}
        self.optimizer = optimizer
        _GraphedStep.__init__(self, model, device_part, warmup)     # GraphedTrainStep's, less the model check above

    def _host_values(self, batch, want):
        """Every entry of ``batch`` that is not a CUDA tensor, as a contiguous CPU tensor; with ``want`` (the example's
        values) each must exist and match its shape and dtype."""
        name, out = type(self).__name__, {}
        for k, v in batch.items():
            if isinstance(v, torch.Tensor) and v.is_cuda:
                if want is not None and k in want:
                    raise ValueError("%s: batch[%r] is a CUDA tensor; the step was captured with it on the host"
                                     % (name, k))
                continue
            t = torch.as_tensor(v).contiguous()
            if want is not None:
                if k not in want:
                    raise ValueError("%s: batch[%r] is on the host; the step was captured with it on the device"
                                     % (name, k))
                if t.shape != want[k].shape or t.dtype != want[k].dtype:
                    raise ValueError("%s: batch[%r] is %s %s; the step was captured for %s %s"
                                     % (name, k, tuple(t.shape), t.dtype, tuple(want[k].shape), want[k].dtype))
            out[k] = t
        missing = [k for k in TRAIN_RECORD_KEYS if k not in out]
        if missing:
            raise ValueError("%s: %s must be host values (the worker's draws), not CUDA tensors" % (name, missing))
        return out

    @staticmethod
    def _check_records(host):
        """The checks the jitter and noise entry points run on the host records, without a launch."""
        ops.color_jitter_check_plans(host["jitter"].numpy())
        plans = host["plans"].numpy()
        for p in range(plans.shape[1]):
            ops.rgb_noise_check_records(plans[:, p])

    def _stage(self, host, seed):
        """Copy the host values and the seed into their device buffers through the next pinned slot, on the current
        stream.  The slot is written once the copies that last read it have run (an event, two calls back): the
        host waits only when it is that far ahead of the stream."""
        i = self._slot
        self._slot = (i + 1) % self._STAGING_SLOTS
        if self._staged[i] is not None:
            self._staged[i].synchronize()
        pin = self._pinned[i]
        for k, t in host.items():
            pin[k].copy_(t)
            self._records[k].copy_(pin[k], non_blocking=True)
        if isinstance(seed, torch.Tensor):
            self._seed.copy_(seed.reshape(1).view(torch.int64))
        else:
            pin["_seed"][0] = seed - (1 << 64) if seed >= 1 << 63 else seed
            self._seed.copy_(pin["_seed"], non_blocking=True)
        self._staged[i] = torch.cuda.Event()
        self._staged[i].record()

    def _step(self):
        batch = dict(self._static, **self._records)
        item = _train_item(batch, self.dataset, self.cam_scale, self._intr, self.n_points, self._seed,
                           records=self._mirror, normals=self.normals, meshes=self.meshes, in_place=True,
                           crops=self.crops)
        return self._train(item)

    def __call__(self, batch, seed):
        name = type(self).__name__
        self._check(self._sync)
        self._check_keys(batch)
        check_render_batch(batch, self.dataset, name, self.meshes, self.normals)
        check_fuse_batch(batch, self.dataset, name, self.crops, self.normals)
        if isinstance(seed, torch.Tensor):
            ops._device_seed(seed, self._seed.device)
        elif isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < 1 << 64:
            raise ValueError("%s: seed must be an int in [0, 2^64) or a one-element CUDA tensor, got %r" % (name, seed))
        host = self._host_values(batch, self._records)
        self._check_records(host)
        self._copy_in({k: batch[k] for k in self._static})
        self._stage(host, seed if isinstance(seed, torch.Tensor) else int(seed))
        return self._replay()


class _GraphedEvalBase(_GraphedStep):
    """An eval-mode step: the model in eval mode, nothing a replay writes outside its own outputs.  Calling it checks
    the model, the batch's keys (when built from a flat batch) and the input buffers' shapes, copies the batch in and
    replays."""

    _wrapper_hint = "pass its .module"

    def _check(self, modules=False):
        """What cannot be captured at all: raise ``ValueError`` before any CUDA work."""
        if self.model.training:
            raise ValueError("%s: the model is in training mode; call model.eval() first, it captures eval steps only"
                             % type(self).__name__)
        self._refuse_index_check()

    def __call__(self, batch):
        self._check()
        self._check_keys(batch)
        self._copy_in(batch)
        return self._replay()


class GraphedEvalStep(_GraphedEvalBase):
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
        self._check_model(model)
        self._with_loss = isinstance(example_item, dict) and all(k in example_item for k in _LOSS_KEYS)
        super().__init__(model, example_item, warmup)

    def _step(self):
        item = self._static
        with torch.no_grad():
            out = _forward(self.model, item)
            loss = info = None
            if self._with_loss:
                loss, info = ffb6d_loss(out, item, valid=item.get("valid"))
        return out, loss, info
