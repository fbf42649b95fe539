"""The per-frame KNN / gather schedule of FFB6D, and its one-call GPU index build.

The reference builds 22 neighbour-index arrays per frame on the CPU inside the
dataset (datasets/ycb/ycb_dataset.py:269-309 == datasets/linemod/linemod_dataset.py:313-353)
and consumes them in ``FFB6D.forward`` through 22 gathers plus the ``choose``
gather (models/ffb6d.py:231-312).  This module states both schedules as data and
runs the index build on the GPU for a whole batch: xyz goes in, the same dict
keys with the same shapes and dtypes (int32) come out, already on the device.
"""
import contextlib
import os

import torch

from .ops import knn_search, KnnGrid, knn_uses_grid, subset_nn_from_knn

from .tables import (RGB_DS_SR, RGB_UP_SR, PCLD_SUB_S_R, N_DS_LAYERS, N_UP_LAYERS, K_NEIGH,  # noqa: F401
                     DS_RGB_OC, DS_RNDLA_OC, UP_RGB_OC, UP_RNDLA_OC, knn_schedule, set_size, gather_schedule,
                     fusion_mlp_schedule, knn_alg_bytes, gather_alg_bytes, frame_alg_bytes, derived_searches, derived_image_searches,
                     derived_subset_searches)


def image_pyramid(dpt_xyz, levels=(1, 2, 4, 8)):
    """``dpt_xyz [B,H,W,3]`` -> ``{sr: [B, (H//sr)*(W//sr), 3]}`` for sr in ``levels``: the
    stride-``sr`` sub-grids of the organised cloud (ycb_dataset.py:253-267)."""
    B, H, W, _ = dpt_xyz.shape
    pyr = {}
    for sr in levels:
        nh, nw = H // sr, W // sr
        pyr[sr] = dpt_xyz[:, :nh * sr:sr, :nw * sr:sr, :].reshape(B, nh * nw, 3).contiguous()
    return pyr


def build_ffb6d_indices(cld, dpt_xyz=None, k=K_NEIGH, index_dtype=torch.int32, timer=None, streams=None,
                        pyramid=None, image_hw=None, events=None, priority=None, build_streams=None):
    """All neighbour-index tensors of the FFB6D fusion stack for a batch, on the GPU.

    :param cld: ``[B, N0, 3]`` float32 CUDA, the sampled (already shuffled) cloud
    :param dpt_xyz: ``[B, H, W, 3]`` float32 CUDA, the organised cloud (zero rows at holes); or
      pass ``pyramid={2: [B,HW/4,3], 4: ..., 8: ...}`` + ``image_hw=(H, W)`` (what
      :func:`ffb6d_b200.ops.backproject` returns) and leave it None
    :param streams: optional list of side ``torch.cuda.Stream`` s to overlap the 22 searches on
    :param build_streams: optional extra side streams for the grid builds (latency-bound cluster kernels that
      co-run well); the caller joins them together with ``streams``
    :param priority: optional ``{index key: float}``; with ``streams`` the searches (and the grid
      builds they need) are issued in descending priority instead of descending size, so that the
      searches whose consumers are expensive finish first
    :param events: optional dict; with ``streams`` it receives one ``torch.cuda.Event`` per index
      key, recorded on the side stream that produced it, and the function returns WITHOUT joining
      the side streams: the caller waits per key (``stream.wait_event``) and joins ``streams``
      itself (:class:`ffb6d_b200.pipeline.FusionPass` overlaps the gathers with the remaining searches)
    :param timer: optional object with ``start(name, alg_bytes)`` / ``stop()`` called around
      every KNN call (bench.py's per-op CUDA-event timer)
    :return: dict with the reference's keys (ycb_dataset.py:283-309), each with a leading
      batch dimension: ``cld_xyz{i}`` f32 ``[B,Ni,3]``; ``cld_nei_idx{i}`` ``[B,Ni,k]``;
      ``cld_sub_idx{i}`` ``[B,Ni/4,k]`` (the first Ni/4 rows of ``cld_nei_idx{i}``, :279);
      ``cld_interp_idx{i}`` ``[B,Ni,1]``; ``r2p_ds_nei_idx{i}`` ``[B,Ni/4,k]``;
      ``p2r_ds_nei_idx{i}`` ``[B,HW,1]``; ``r2p_up_nei_idx{i}``, ``p2r_up_nei_idx{i}``.
      Index tensors are ``index_dtype`` (int32 like the datasets; pass torch.int64 to skip
      the cast ``model_fn`` does, train_ycb.py:224-232).

    "Random sampling" is the reference's: the cloud was shuffled once, every level keeps the
    first quarter of the previous one (ycb_dataset.py:233-235, 278).
    """
    if cld.dim() != 3 or cld.shape[2] != 3:
        raise ValueError("expected cld [B,N,3]")
    cld = cld.contiguous().float()
    B, n0, _ = cld.shape
    used = sorted(set(RGB_DS_SR) | set(RGB_UP_SR))          # sr=1 is never searched
    if pyramid is not None:
        if image_hw is None:
            raise ValueError("image_hw=(H, W) is required with pyramid=")
        H, W = image_hw
        sets = {("img", sr): pyramid[sr] for sr in used}
    else:
        if dpt_xyz is None or dpt_xyz.dim() != 4 or cld.shape[0] != dpt_xyz.shape[0]:
            raise ValueError("expected dpt_xyz [B,H,W,3] (or pyramid=)")
        H, W = dpt_xyz.shape[1], dpt_xyz.shape[2]
        sets = {("img", sr): p for sr, p in image_pyramid(dpt_xyz.float(), used).items()}
    n = n0
    for i in range(N_DS_LAYERS + 1):
        sets[("cld", i)] = cld if i == 0 else cld[:, :n, :].contiguous()
        if i < N_DS_LAYERS:
            n //= PCLD_SUB_S_R[i]
    inputs = {}
    calls = knn_schedule(n0, H, W, k)
    # one grid per (point set, K class) shared by all the searches into it; supports whose
    # searches are all tiny keep the tiled scan
    groups = {}
    for key, s, q, kk in calls:
        groups.setdefault((s, kk), []).append((key, q))
    # FFB6D_SUBSET_NN=1 (off by default: exact, but the pass is slower with it, DESIGN.md section 4.1): cld_interp_idx{i}
    # (nearest level-(i+1) point of every level-i point) is read off cld_nei_idx{i} -- level i+1 is a row prefix of
    # level i, so the first entry of a self-search row that is < N_{i+1} is the answer; only the rows without one
    # (0.75^K of them) are searched (ops.subset_nn_from_knn).  Applies where the search would take the grid.
    derived_sub = {c: p_ for c, p_ in derived_subset_searches(calls).items()
                   if k >= 8 and os.environ.get("FFB6D_SUBSET_NN", "0") == "1"}
    derived_sub = {c: p_ for c, p_ in derived_sub.items()
                   if any(key == c and knn_uses_grid(B, sets[s].shape[1], sets[q].shape[1], kk) for key, s, q, kk in calls)}
    gridded = [g for g, members in groups.items()
               if any(knn_uses_grid(B, sets[g[0]].shape[1], sets[q].shape[1], g[1]) for key_, q in members
                      if key_ not in derived_sub)]
    grids = {}
    main = torch.cuda.current_stream(cld.device)
    par = streams is not None and timer is None
    bstreams = list(build_streams) if (build_streams and par) else []

    def fork():
        if par:
            for st in streams + bstreams:
                st.wait_stream(main)

    def join():
        if par:
            for st in streams + bstreams:
                main.wait_stream(st)

    def on(i, pool=None):
        pool = pool or streams
        return torch.cuda.stream(pool[i % len(pool)]) if par else contextlib.nullcontext()

    # Cloud level j is the first N_j rows of the shuffled cloud (ycb_dataset.py:278), so two searches of the same
    # support with the same K whose query sets are cloud levels answer the same questions on a prefix: the
    # schedule's r2p_ds_nei_idx2/3 are the first 192 / 48 rows of r2p_ds_nei_idx1 (support img8), r2p_up_nei_idx0
    # the first rows of r2p_ds_nei_idx0 (img4), r2p_up_nei_idx1 of r2p_up_nei_idx2 (img2).  Those four searches
    # are not run; their tensors are row slices of the larger search (identical values by construction).
    derived = derived_searches(calls)
    children = {}
    for child, parent in derived.items():
        children.setdefault(parent, []).append(child)
    # Image level sr_c is every f-th pixel of every f-th row of level sr_p = sr_c / f (stride slicing of the same
    # organised cloud): a K = 1 search from img4 / img8 into a cloud level is a strided subset of the search from
    # img2 / img4 into the same level (p2r_ds_nei_idx0 of p2r_up_nei_idx2, idx1 of p2r_up_nei_idx1, idx2 of
    # p2r_up_nei_idx0): three more searches that are copied instead of run.
    derived_img = derived_image_searches(calls, H, W)
    children_img = {}
    for child, (parent, f) in derived_img.items():
        children_img.setdefault(parent, []).append((child, f))

    fork()
    # a search waits only for ITS grid, a consumer only for ITS index tensor (events, not joins)
    built = {}
    if par and priority:
        order = sorted(calls, key=lambda c: -priority.get(c[0], 0.0))
        first_use = {}
        for pos, (key, s_, q_, kk_) in enumerate(order):
            first_use.setdefault((s_, kk_), pos)
        build_order = sorted(gridded, key=lambda g: first_use.get(g, len(order)))
    else:
        order = sorted(calls, key=lambda c: -(sets[c[2]].shape[1] * c[3])) if par else calls
        build_order = sorted(gridded, key=lambda g: -sets[g[0]].shape[1])
    for i, g in enumerate(build_order):
        with on(i, bstreams or None):
            if timer is not None:
                timer.start("knn_build:%s%d:k%d" % (g[0][0], g[0][1], g[1]), 0)
            grids[g] = KnnGrid(sets[g[0]], g[1])
            if timer is not None:
                timer.stop()
            if par:
                built[g] = torch.cuda.Event()
                built[g].record()
    order = [c for c in order if c[0] not in derived and c[0] not in derived_img and c[0] not in derived_sub]
    qsize = {key: sets[q].shape[1] for key, s, q, kk in calls}
    for i, (key, s, q, kk) in enumerate(order):
        sup, qry = sets[s], sets[q]
        with on(i):
            if timer is not None:
                timer.start("knn:" + key, knn_alg_bytes(sup.shape[1], qry.shape[1], kk) * B)
            if (s, kk) in grids:
                if par:
                    torch.cuda.current_stream(cld.device).wait_event(built[(s, kk)])
                # image pyramid levels are organised: rows of W // sr pixels (a layout hint for K = 1)
                inputs[key] = grids[(s, kk)].query(qry, kk, out_dtype=index_dtype,
                                                   query_width=(W // q[1]) if q[0] == "img" else 0)
            else:
                inputs[key] = knn_search(sup, qry, kk, out_dtype=index_dtype, algo=1)
            if timer is not None:
                timer.stop()
            done = [key]
            if key.startswith("cld_nei_idx"):   # cld_sub_idx_i = the first N_{i+1} rows (ycb_dataset.py:279)
                lvl = int(key[len("cld_nei_idx"):])
                n_sub = sets[("cld", lvl + 1)].shape[1]
                inputs["cld_sub_idx%d" % lvl] = inputs[key][:, :n_sub, :].contiguous()
                done.append("cld_sub_idx%d" % lvl)
                child = "cld_interp_idx%d" % lvl
                if derived_sub.get(child) == key:
                    sub = sets[("cld", lvl + 1)]
                    if timer is not None:
                        timer.start("knn:" + child, knn_alg_bytes(sub.shape[1], qry.shape[1], 1) * B)
                    inputs[child] = subset_nn_from_knn(sub, qry, inputs[key])
                    if timer is not None:
                        timer.stop()
                    done.append(child)
            for child in children.get(key, ()):   # prefix slices instead of separate searches (see above)
                inputs[child] = inputs[key][:, :qsize[child], :].contiguous()
                done.append(child)
            for child, f in children_img.get(key, ()):   # strided pixel subsets (see above)
                hp, wp = H // q[1], W // q[1]
                inputs[child] = inputs[key].view(B, hp, wp, kk)[:, ::f, ::f, :].reshape(B, -1, kk)
                done.append(child)
            if par and events is not None:
                ev = torch.cuda.Event()
                ev.record()
                for name in done:
                    events[name] = ev
    if par and events is not None:
        # the caller joins the side streams later: the grids (allocated on one side stream, read by
        # searches on others) and the source point sets must outlive those searches, so they travel
        # with the events instead of dying with this frame
        events["_keepalive"] = (grids, sets)
    else:
        join()
    for i in range(N_DS_LAYERS):
        inputs["cld_xyz%d" % i] = sets[("cld", i)]
    return inputs


def build_ffb6d_indices_native(cld, pyramid, image_hw, k=K_NEIGH, index_dtype=torch.int32):
    """:func:`build_ffb6d_indices` through the single C entry point ``ffb6d_build_indices`` (one call,
    one stream, caller-owned buffers): what a non-Python host of the library would run.  Same keys,
    shapes, dtypes and bits as :func:`build_ffb6d_indices`.

    :param cld: ``[B, N0, 3]`` float32 CUDA; :param pyramid: ``{2: [B,HW/4,3], 4: ..., 8: ...}``
    :param image_hw: ``(H, W)`` of the full-resolution image"""
    import ctypes
    from ._lib import lib, check
    from .ops import _stream
    if cld.dim() != 3 or cld.shape[2] != 3 or not cld.is_cuda:
        raise ValueError("expected cld [B,N,3] on a CUDA device")
    cld = cld.contiguous().float()
    B, n0, _ = cld.shape
    H, W = image_hw
    img = {sr: pyramid[sr].contiguous().float() for sr in (2, 4, 8)}
    for sr in (2, 4, 8):
        if tuple(img[sr].shape) != (B, (H // sr) * (W // sr), 3):
            raise ValueError("pyramid[%d] must be [B, %d, 3]" % (sr, (H // sr) * (W // sr)))
    calls = knn_schedule(n0, H, W, k)
    inputs, ptrs = {}, (ctypes.c_void_p * len(calls))()
    for j, (key, s, q, kk) in enumerate(calls):
        inputs[key] = torch.empty((B, set_size(q, n0, H, W), kk), dtype=index_dtype, device=cld.device)
        ptrs[j] = inputs[key].data_ptr()
    nbytes = int(lib.ffb6d_build_indices_workspace_bytes(B, n0, H, W, int(k)))
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=cld.device)
    with torch.cuda.device(cld.device):
        check(lib.ffb6d_build_indices(cld.data_ptr(), img[2].data_ptr(), img[4].data_ptr(), img[8].data_ptr(), B, n0, H, W,
                                      int(k), ctypes.cast(ptrs, ctypes.c_void_p), int(index_dtype == torch.int64),
                                      ws.data_ptr(), nbytes, _stream(cld.device)))
    n = n0
    for i in range(N_DS_LAYERS):
        inputs["cld_xyz%d" % i] = cld if i == 0 else cld[:, :n, :].contiguous()
        n //= PCLD_SUB_S_R[i]
        inputs["cld_sub_idx%d" % i] = inputs["cld_nei_idx%d" % i][:, :n, :].contiguous()
    return inputs


def build_ffb6d_indices_from_depth(depth, K, choose, k=K_NEIGH, index_dtype=torch.int32, streams=None):
    """Depth map in, all index tensors out: back-projection, sampling and stride pyramids
    (datasets/ycb/ycb_dataset.py:165-176, 237, 253-267) followed by the 22 searches, everything on
    the GPU.  ``depth [B,H,W]`` float32 metres, ``K`` camera matrix, ``choose [B,1,N]`` pixel
    indices of the sampled points.  Returns the dict of :func:`build_ffb6d_indices`."""
    from .ops import backproject
    cld, pyr = backproject(depth, K, choose)
    return build_ffb6d_indices(cld, None, k=k, index_dtype=index_dtype, streams=streams, pyramid=pyr,
                               image_hw=(depth.shape[1], depth.shape[2]))


# float32(1e-6): the dataset's `msk_dp = dpt_um > 1e-6` on the completed raw depth (ycb_dataset.py:205)
MSK_DP_THRESHOLD = 1e-6


def build_ffb6d_indices_from_raw_depth(dpt_raw, cam_scale, K, n_points, seed=0, k=K_NEIGH, index_dtype=torch.int32,
                                       streams=None):
    """The depth half of ``YCB_Dataset.get_item`` on the GPU (datasets/ycb/ycb_dataset.py:204-309 without
    normals): depth completion (:func:`ffb6d_b200.ops.fill_missing`, :204), ``msk_dp`` and the sampling of
    ``n_points`` valid pixels (:205, 218-235, :func:`ffb6d_b200.ops.sample_valid_pixels` with ``seed``),
    ``dpt_m`` (:215), back-projection and the 22 searches (:func:`build_ffb6d_indices_from_depth`).

    :param dpt_raw: ``[B,H,W]`` ``torch.uint16`` CUDA, the depth PNGs' raw values
    :param cam_scale: raw units per metre (``meta['factor_depth']``); :param K: camera matrix as for
      :func:`ffb6d_b200.ops.backproject`
    :return: the dict of :func:`build_ffb6d_indices`, plus ``choose [B,1,n_points]`` int32 and
      ``dpt_map_m [B,H,W]`` float32 (the reference's ``item_dict`` key)"""
    from .ops import _fill_depth, sample_valid_pixels
    if not isinstance(dpt_raw, torch.Tensor) or dpt_raw.dim() != 3:
        raise ValueError("dpt_raw must be a [B,H,W] torch.uint16 CUDA tensor")
    filled, depth_m = _fill_depth(dpt_raw, cam_scale)
    choose = sample_valid_pixels(filled, n_points, seed=seed, min_depth=MSK_DP_THRESHOLD)
    inputs = build_ffb6d_indices_from_depth(depth_m, K, choose, k=k, index_dtype=index_dtype, streams=streams)
    inputs["choose"] = choose
    inputs["dpt_map_m"] = depth_m
    return inputs
