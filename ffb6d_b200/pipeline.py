"""One pass of the fusion hot path over a batch of frames (the unit bench.py times).

A *pass* is what BASELINE.md §3 defines: the 22 KNN index builds of the dataset schedule
(datasets/ycb/ycb_dataset.py:269-309) followed by the 11 ``random_sample``, 11
``nearest_interpolation`` and 1 ``choose`` gathers of ``FFB6D.forward``
(models/ffb6d.py:240-312), each gather consuming the index tensor the reference feeds it and
a feature tensor of the width the reference has at that point.  The network layers between
the gathers (cuDNN convs, 1x1 fusion MLPs) are not part of the pass, so the gather inputs are
synthetic N(0,1) features resident in HBM.
"""
import torch

from . import ops
from . import schedule as S


class FusionPass:
    """Holds the device-resident feature tensors of one batch and runs passes over it.

    :param batch: frames per pass (B)
    :param n_points: sampled cloud size N0 (12288 in the reference, common.py:61)
    :param layout: ``"nchw"`` -- features are contiguous [B,C,S,1] like the reference's;
      ``"channels_last"`` -- same logical tensors in torch channels_last memory format.
    """

    def __init__(self, batch, n_points=12288, h=480, w=640, k=S.K_NEIGH, device="cuda",
                 layout="nchw", seed=0, index_dtype=torch.int32, n_streams=2, n_gather_streams=None):
        self.B, self.n_points, self.h, self.w, self.k = batch, n_points, h, w, k
        self.device = torch.device(device)
        self.layout = layout
        self.index_dtype = index_dtype
        self.streams = [torch.cuda.Stream(device=self.device) for _ in range(n_streams)] if n_streams > 1 else None
        # the gathers (HBM bound) get streams of their own: each waits only for its index tensor, so
        # it overlaps the searches (issue bound) that are still running
        self.gstreams = ([torch.cuda.Stream(device=self.device) for _ in range(n_gather_streams or n_streams)]
                         if n_streams > 1 else None)
        self.gathers = S.gather_schedule(n_points, h, w)
        g = torch.Generator(device=self.device).manual_seed(seed)
        self.features = []
        for op, key, C, Sz, Q, K in self.gathers:
            f = torch.randn((batch, C, Sz, 1), generator=g, device=self.device, dtype=torch.float32)
            if layout == "channels_last":
                f = f.contiguous(memory_format=torch.channels_last)
            elif layout != "nchw":
                raise ValueError("layout must be 'nchw' or 'channels_last'")
            self.features.append(f)
        # issue order of the searches: bytes of the gathers a search unlocks per unit of search work
        # (measured: a K = 16 query costs about 12 K = 1 queries)
        unlocked = {}
        derived = S.derived_searches(S.knn_schedule(n_points, h, w, k))   # row slices of another search
        derived.update({c: p_ for c, (p_, f_) in S.derived_image_searches(S.knn_schedule(n_points, h, w, k), h, w).items()})
        for op, key, C, Sz, Q, K in self.gathers:
            src = key.replace("cld_sub_idx", "cld_nei_idx")
            src = derived.get(src, src)
            unlocked[src] = unlocked.get(src, 0) + S.gather_alg_bytes(C, Sz, Q, K)
        self.priority = {key: unlocked.get(key, 0) / float(S.set_size(q, n_points, h, w) * (12 if kk > 1 else 1))
                         for key, s_, q, kk in S.knn_schedule(n_points, h, w, k)}
        # ... except the level-0 self search, the longest search of the pass: it needs only the level-0 grid, so it goes
        # first and the big p2r searches queue behind it (measured three times: -0.2 ... -0.6 % of the pass)
        self.priority["cld_nei_idx0"] = float("inf")
        kb, gb = S.frame_alg_bytes(n_points, h, w, k)
        self.alg_bytes_per_frame = kb + gb
        self.knn_alg_bytes_per_frame = kb
        self.gather_alg_bytes_per_frame = gb

    # -- the two halves of a pass ------------------------------------------------------
    def build_indices(self, cld, dpt_xyz, choose, timer=None, events=None):
        inputs = S.build_ffb6d_indices(cld, dpt_xyz, k=self.k, index_dtype=self.index_dtype,
                                       timer=timer, streams=self.streams, events=events, priority=self.priority)
        inputs["choose"] = choose
        return inputs

    def _gather(self, op, C, feat, idx):
        if op == "random_sample":
            return ops.random_sample(feat, idx)
        if op == "nearest_interpolation":
            return ops.nearest_interpolation(feat, idx)
        return ops.choose_gather(feat.reshape(self.B, C, self.h, self.w) if self.layout == "nchw"
                                 else feat.squeeze(3), idx)

    def kernel_of(self, i):
        """Name of the CUDA kernel the i-th gather of the schedule runs on."""
        from ._lib import lib, LAYOUT_NCS, LAYOUT_NSC
        op, key, C, Sz, Q, K = self.gathers[i]
        k = 1 if op != "random_sample" else self.k
        lay = LAYOUT_NCS if self.layout == "nchw" else LAYOUT_NSC
        return lib.ffb6d_gather_kernel_name(self.B, C, Sz, Q, k, lay).decode()

    def run_gathers(self, inputs, timer=None, events=None):
        """``events``: per-key events from :func:`build_ffb6d_indices` (side streams not joined yet):
        every gather waits for its own index tensor only; this call joins all side streams."""
        n = len(self.gathers)
        outs = [None] * n
        if self.streams is None or timer is not None:
            for i, ((op, key, C, Sz, Q, K), feat) in enumerate(zip(self.gathers, self.features)):
                idx = inputs[key]
                if timer is not None:
                    timer.start("gather:%s:%s" % (key, self.kernel_of(i)),
                                S.gather_alg_bytes(C, Sz, Q, idx.shape[-1] if op != "choose" else 1) * self.B)
                outs[i] = self._gather(op, C, feat, idx)
                if timer is not None:
                    timer.stop()
            return outs
        # the 23 gathers are independent of each other too
        main = torch.cuda.current_stream(self.device)
        capturing = torch.cuda.is_current_stream_capturing()
        order = sorted(range(n), key=lambda i: -(self.gathers[i][2] * self.gathers[i][4]))
        gs = self.gstreams if events is not None else self.streams
        for st in gs:
            st.wait_stream(main)
        for j, i in enumerate(order):
            op, key, C, Sz, Q, K = self.gathers[i]
            st = gs[j % len(gs)]
            if events is not None and key in events:
                st.wait_event(events[key])
            with torch.cuda.stream(st):
                outs[i] = self._gather(op, C, self.features[i], inputs[key])
            if not capturing:
                # produced on a search stream, read here / produced here, read on the caller's stream:
                # tell the caching allocator (inside a capture the graph's private pool keeps them alive)
                inputs[key].record_stream(st)
                outs[i].record_stream(main)
        for st in (self.streams + self.gstreams) if events is not None else gs:
            main.wait_stream(st)
        if events is not None:
            events.pop("_keepalive", None)   # every search has been joined: the grids may go
        return outs

    # -- CUDA-graph replay: the pass is ~200 small launches with static shapes ----------
    def capture(self, fn, copies=(), digest=None, prefetch=()):
        """Capture ``fn()`` (a closure over static device buffers that runs a pass and returns its
        result) into a CUDA graph and return ``replay()``.

        ``copies``: ``(dst_device, src_pinned_host)`` pairs copied at the start of the graph, on the
        main stream, before ``fn``.  ``prefetch``: pairs copied on a side stream concurrently with
        ``fn`` (inputs of the NEXT replay: double buffering).  ``digest=(f, pinned_out)``:
        ``pinned_out.copy_(f(*result))`` at the end (the D2H read of the end-to-end variant)."""
        side = torch.cuda.Stream(device=self.device)

        def body():
            main = torch.cuda.current_stream(self.device)
            for dst, src in copies:
                dst.copy_(src, non_blocking=True)
            if prefetch:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    for dst, src in prefetch:
                        dst.copy_(src, non_blocking=True)
            res = fn()
            if prefetch:
                main.wait_stream(side)
            if digest is not None:
                d = digest[0](*res)
                digest[1][: d.numel()].copy_(d, non_blocking=True)
            return res

        warm = torch.cuda.Stream(device=self.device)
        warm.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(warm):
            for _ in range(2):        # allocator + lazy one-time settings happen outside the capture
                body()
        torch.cuda.current_stream(self.device).wait_stream(warm)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            res = body()

        def replay():
            graph.replay()
            return res

        replay.graph = graph
        return replay

    def from_depth(self, depth, intr, choose):
        """depth [B,H,W] f32, intr = device (fx,fy,cx,cy) float64 [4]|[B,4], choose [B,1,N] -> pass."""
        cld, pyr = ops.backproject(depth, intr, choose)
        events = {} if self.streams is not None else None
        inputs = S.build_ffb6d_indices(cld, None, k=self.k, index_dtype=self.index_dtype, streams=self.streams,
                                       pyramid=pyr, image_hw=(self.h, self.w), events=events, priority=self.priority)
        inputs["choose"] = choose
        return inputs, self.run_gathers(inputs, events=events)

    def __call__(self, cld, dpt_xyz, choose, timer=None):
        """cld [B,N0,3] f32, dpt_xyz [B,H,W,3] f32, choose [B,1,N0] int -> (inputs dict, outputs)."""
        events = {} if (self.streams is not None and timer is None) else None
        inputs = self.build_indices(cld, dpt_xyz, choose, timer, events)
        return inputs, self.run_gathers(inputs, timer, events)


class FusionMLPs:
    """The 28 fusion 1x1 MLPs of one batch with synthetic weights and inputs (eval-mode BatchNorm
    folded into scale/shift), run through the tensor-core kernel.  BASELINE.md reports them
    separately from the KNN + gather pass."""

    def __init__(self, batch, n_points=12288, h=480, w=640, device="cuda", seed=0, prepack=True):
        self.B = batch
        self.device = torch.device(device)
        self.prepack = prepack   # weights split once at load (inference), as a deployed model would
        self.layers = S.fusion_mlp_schedule(n_points, h, w)
        g = torch.Generator(device=self.device).manual_seed(seed)
        self.args = []
        self.flops = 0
        for name, P, C1, C2, Co in self.layers:
            def rnd(*shape):
                return torch.randn(shape, generator=g, device=self.device, dtype=torch.float32)
            x1 = rnd(batch, C1, P, 1)
            x2 = rnd(batch, C2, P, 1) if C2 else None
            wgt = rnd(Co, C1 + C2) / float(C1 + C2) ** 0.5
            scale = torch.rand(Co, generator=g, device=self.device) + 0.5
            shift = rnd(Co) * 0.1
            self.args.append((x1, x2, ops.fusion_mlp_pack(wgt) if prepack else wgt, scale, shift))
            self.flops += 2 * batch * Co * (C1 + C2) * P

    def __call__(self):
        return [ops.fusion_mlp(*a) for a in self.args]


class FusionStack:
    """BASELINE configs[1], "full 4-scale fusion stack": the seven bidirectional fusion stages of
    ``FFB6D.forward`` (models/ffb6d.py:231-298) chained on this package's kernels -- per stage the set
    abstraction gather (``random_sample`` / ``nearest_interpolation`` of the point branch), ``p2r_pre`` ->
    restructured ``p2r_fuse`` (no interpolated map, :mod:`ffb6d_b200.fusion`), the image -> point gather and
    ``r2p_pre`` -> ``r2p_fuse``; then the final interpolation and the ``choose`` gather (:301-312).
    The CNN / RandLA layers between the stages are out of scope, so every stage starts from synthetic
    ``rgb_emb0`` / point features of the reference's widths; inside a stage the data flow is the reference's.
    Weights are synthetic, BatchNorm folded (inference)."""

    def __init__(self, batch, n_points=12288, h=480, w=640, k=S.K_NEIGH, device="cuda", seed=0):
        from . import fusion
        self.B, self.n_points, self.h, self.w, self.k = batch, n_points, h, w, k
        self.device = torch.device(device)
        g = torch.Generator(device=self.device).manual_seed(seed)

        def rnd(*shape):
            return torch.randn(shape, generator=g, device=self.device, dtype=torch.float32)

        def conv(cin, cout):
            return fusion.FusedConv(rnd(cout, cin) / float(cin) ** 0.5,
                                    torch.rand(cout, generator=g, device=self.device) + 0.5, rnd(cout) * 0.1)

        N = [S.set_size(("cld", i), n_points) for i in range(5)]
        self.stages, self.rgb0, self.pts, self.kind = [], [], [], []
        self.flops = 0
        dims = [(S.DS_RGB_OC[i], S.DS_RNDLA_OC[i], S.RGB_DS_SR[i], N[i], N[i + 1]) for i in range(S.N_DS_LAYERS)]
        up_in = (S.DS_RNDLA_OC[3], S.UP_RNDLA_OC[0], S.UP_RNDLA_OC[1])
        dims += [(S.UP_RGB_OC[i], S.UP_RNDLA_OC[i], S.RGB_UP_SR[i], N[S.N_DS_LAYERS - i], N[S.N_DS_LAYERS - i - 1])
                 for i in range(S.N_UP_LAYERS)]
        for j, (cr, cp, sr, n_src, n1) in enumerate(dims):
            enc = j < S.N_DS_LAYERS
            self.stages.append(fusion.FusionStage(conv(cr, cp), conv(2 * cp, cp), conv(cp, cr), conv(2 * cr, cr)))
            self.rgb0.append(rnd(batch, cr, h // sr, w // sr))
            if enc:      # f_encoder_i on N_i points, pooled to N_{i+1} by random_sample (:240)
                self.pts.append(rnd(batch, cp, n_src, 1))
            else:        # decoder: the interpolated point features (:273-275) feed the (out of scope) RandLA
                         # decoder conv; its output p_emb0 on N_lvl points is synthetic
                self.pts.append((rnd(batch, up_in[j - S.N_DS_LAYERS], n_src, 1), rnd(batch, cp, n1, 1)))
            n_pts = n1
            hw = (h // sr) * (w // sr)
            self.flops += 2 * batch * (n_pts * (cr * cp + 2 * cp * cp + cp * cr + cr * cr) + hw * cr * cr)
        self.p_last = rnd(batch, S.UP_RNDLA_OC[2], N[1], 1)       # :302-304
        self.rgb_last = rnd(batch, S.UP_RGB_OC[2], h, w)          # :309-312

    def __call__(self, inputs, restructured=True):
        outs = []
        for i in range(S.N_DS_LAYERS):
            p_emb0 = ops.random_sample(self.pts[i], inputs["cld_sub_idx%d" % i])
            outs.append(self.stages[i](self.rgb0[i], p_emb0, inputs["p2r_ds_nei_idx%d" % i],
                                       inputs["r2p_ds_nei_idx%d" % i], restructured))
        for i in range(S.N_UP_LAYERS):
            j, lvl = S.N_DS_LAYERS + i, S.N_DS_LAYERS - i - 1
            p_prev, p_emb0 = self.pts[j]
            outs.append(ops.nearest_interpolation(p_prev, inputs["cld_interp_idx%d" % lvl]))
            outs.append(self.stages[j](self.rgb0[j], p_emb0, inputs["p2r_up_nei_idx%d" % i],
                                       inputs["r2p_up_nei_idx%d" % i], restructured))
        outs.append(ops.nearest_interpolation(self.p_last, inputs["cld_interp_idx0"]))
        outs.append(ops.choose_gather(self.rgb_last, inputs["choose"]))
        return outs


class OpTimer:
    """CUDA-event pair per op on the current stream; durations are read after a synchronize.
    Events come from a pool created up front so that recording costs the CPU as little as possible."""

    def __init__(self, pool=4096):
        self.records = []          # (name, alg_bytes, start_event, stop_event)
        self._cur = None
        self._pool = [torch.cuda.Event(enable_timing=True) for _ in range(pool)]
        self._next = 0

    def _event(self):
        if self._next >= len(self._pool):
            self._pool.extend(torch.cuda.Event(enable_timing=True) for _ in range(1024))
        e = self._pool[self._next]
        self._next += 1
        return e

    def start(self, name, alg_bytes):
        e0, e1 = self._event(), self._event()
        e0.record()
        self._cur = (name, alg_bytes, e0, e1)

    def stop(self):
        name, b, e0, e1 = self._cur
        e1.record()
        self.records.append((name, b, e0, e1))
        self._cur = None

    def summary(self):
        """{name: {"ms": total, "bytes": total alg bytes, "n": launches}} (call after synchronize)."""
        out = {}
        for name, b, e0, e1 in self.records:
            d = out.setdefault(name, {"ms": 0.0, "bytes": 0, "n": 0})
            d["ms"] += e0.elapsed_time(e1)
            d["bytes"] += b
            d["n"] += 1
        return out
