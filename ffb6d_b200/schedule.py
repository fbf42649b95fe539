"""The per-frame KNN / gather schedule of FFB6D, and its one-call GPU index build.

The reference builds 22 neighbour-index arrays per frame on the CPU inside the
dataset (datasets/ycb/ycb_dataset.py:269-309 == datasets/linemod/linemod_dataset.py:313-353)
and consumes them in ``FFB6D.forward`` through 22 gathers plus the ``choose``
gather (models/ffb6d.py:231-312).  This module states both schedules as data and
runs the index build on the GPU for a whole batch: xyz goes in, the same dict
keys with the same shapes and dtypes (int32) come out, already on the device.
"""
import contextlib

import torch

from .ops import knn_search, KnnGrid, knn_uses_grid

from .tables import (RGB_DS_SR, RGB_UP_SR, PCLD_SUB_S_R, N_DS_LAYERS, N_UP_LAYERS, K_NEIGH,  # noqa: F401
                     DS_RGB_OC, DS_RNDLA_OC, UP_RGB_OC, UP_RNDLA_OC, knn_schedule, set_size, gather_schedule,
                     fusion_mlp_schedule, knn_alg_bytes, gather_alg_bytes, frame_alg_bytes, derived_searches, derived_image_searches)


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
                        pyramid=None, image_hw=None, events=None, priority=None):
    """All neighbour-index tensors of the FFB6D fusion stack for a batch, on the GPU.

    :param cld: ``[B, N0, 3]`` float32 CUDA, the sampled (already shuffled) cloud
    :param dpt_xyz: ``[B, H, W, 3]`` float32 CUDA, the organised cloud (zero rows at holes); or
      pass ``pyramid={2: [B,HW/4,3], 4: ..., 8: ...}`` + ``image_hw=(H, W)`` (what
      :func:`ffb6d_b200.ops.backproject` returns) and leave it None
    :param streams: optional list of side ``torch.cuda.Stream`` s to overlap the 22 searches on
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
    gridded = [g for g, members in groups.items()
               if any(knn_uses_grid(B, sets[g[0]].shape[1], sets[q].shape[1], g[1]) for key_, q in members)]
    grids = {}
    main = torch.cuda.current_stream(cld.device)
    par = streams is not None and timer is None

    def fork():
        if par:
            for st in streams:
                st.wait_stream(main)

    def join():
        if par:
            for st in streams:
                main.wait_stream(st)

    def on(i):
        return torch.cuda.stream(streams[i % len(streams)]) if par else contextlib.nullcontext()

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
        with on(i):
            if timer is not None:
                timer.start("knn_build:%s%d:k%d" % (g[0][0], g[0][1], g[1]), 0)
            grids[g] = KnnGrid(sets[g[0]], g[1])
            if timer is not None:
                timer.stop()
            if par:
                built[g] = torch.cuda.Event()
                built[g].record()
    order = [c for c in order if c[0] not in derived and c[0] not in derived_img]
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
    from ._lib import lib, launch, workspace
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
    ws = workspace(nbytes, cld.device)
    launch(lib.ffb6d_build_indices, cld.device, cld.data_ptr(), img[2].data_ptr(), img[4].data_ptr(), img[8].data_ptr(),
           B, n0, H, W, int(k), ctypes.cast(ptrs, ctypes.c_void_p), int(index_dtype == torch.int64), ws.data_ptr(),
           nbytes)
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


# the datasets' get_item returns None below this many valid pixels and the loader draws another frame
# (ycb_dataset.py:219, linemod_dataset.py:266)
MIN_VALID_PIXELS = 400
_OBJECT_KEYS = ("RTs", "kp_3ds", "ctr_3ds", "cls_ids", "obj_cls", "obj_kps", "obj_ctr")


def check_dataset(dataset, name):
    """``ValueError`` unless ``dataset`` is ``"ycb"`` or ``"linemod"``."""
    if dataset not in ("ycb", "linemod"):
        raise ValueError("%s: dataset must be 'ycb' or 'linemod', got %r" % (name, dataset))


# where the normal map comes from: "input", the caller's nrm_map (normalSpeed's in the reference), or "device",
# depth_normal of the depth the datasets take it from (DESIGN.md §4.30)
NORMALS = ("input", "device")
# normalSpeed.depth_normal's k_size, distance_threshold, difference_threshold and point_into_surface in both datasets
# (ycb_dataset.py:208-210, linemod_dataset.py:252-254)
NORMAL_ARGS = (5, 2000, 20, False)
# YCB's millimetre map is (dpt_um / 10).astype(np.uint16) of the completed depth (ycb_dataset.py:207)
YCB_MM_DIVISOR = 10.0


def check_normals(normals, name, nrm_map=None):
    """``ValueError`` unless ``normals`` is one of ``NORMALS``, and with ``"device"`` unless ``nrm_map`` is None."""
    if not (isinstance(normals, str) and normals in NORMALS):
        raise ValueError("%s: normals must be 'input' or 'device', got %r" % (name, normals))
    if normals == "device" and nrm_map is not None:
        raise ValueError("%s: nrm_map is given with normals='device'; pass None (the normals are computed from the "
                         "depth)" % name)


def _normal_keys(batch, name, keys, normals):
    """``keys`` without ``nrm_map`` under ``normals="device"``, where a batch holding ``nrm_map`` is refused."""
    check_normals(normals, name)
    if normals == "input":
        return tuple(keys)
    if isinstance(batch, dict) and "nrm_map" in batch:
        raise ValueError("%s: the batch holds nrm_map with normals='device'; leave it out (the normals are computed "
                         "from the depth)" % name)
    return tuple(k for k in keys if k != "nrm_map")


def check_frame_batch(batch, name, keys, normals="input"):
    """``ValueError`` unless ``batch`` is a dict of CUDA tensors on one device with exactly ``keys`` and optionally
    ``K``: ``dpt`` uint16 ``[B,H,W]``, ``rgb`` uint8 ``[B,H,W,3]``, ``nrm_map`` float32 / float64 ``[B,H,W,3]``, ``K``
    float64 ``[B,3,3]`` and, when ``keys`` hold it, ``RTs [B,n_obj,3,4]``.  With ``normals="device"`` the batch must not
    hold ``nrm_map``.  Runs before any CUDA work."""
    keys = _normal_keys(batch, name, keys, normals)
    if not isinstance(batch, dict):
        raise ValueError("%s: the batch must be a dict, got %s" % (name, type(batch).__name__))
    missing = [k for k in keys if k not in batch]
    if missing:
        raise ValueError("%s: the batch lacks %s (it needs %s)" % (name, missing, list(keys)))
    known = tuple(keys) + ("K",)
    unknown = sorted(str(k) for k in batch if k not in known)
    if unknown:
        raise ValueError("%s: unknown batch keys %s (known: %s)" % (name, unknown, list(known)))
    for k, t in batch.items():
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: batch[%r] must be a tensor, got %s" % (name, k, type(t).__name__))
    dpt, rgb = batch["dpt"], batch["rgb"]
    if dpt.dtype != torch.uint16 or dpt.dim() != 3:
        raise ValueError("%s: batch['dpt'] must be uint16 [B,H,W], got %s %s" % (name, dpt.dtype, tuple(dpt.shape)))
    B, H, W = dpt.shape
    if rgb.dtype != torch.uint8 or tuple(rgb.shape) != (B, H, W, 3):
        raise ValueError("%s: batch['rgb'] must be uint8 [B,H,W,3] = %s, got %s %s"
                         % (name, (B, H, W, 3), rgb.dtype, tuple(rgb.shape)))
    nrm = batch.get("nrm_map")
    if nrm is not None and (nrm.dtype not in (torch.float32, torch.float64) or tuple(nrm.shape) != (B, H, W, 3)):
        raise ValueError("%s: batch['nrm_map'] must be float32 or float64 [B,H,W,3] = %s, got %s %s"
                         % (name, (B, H, W, 3), nrm.dtype, tuple(nrm.shape)))
    if "K" in batch and (batch["K"].dtype != torch.float64 or tuple(batch["K"].shape) != (B, 3, 3)):
        raise ValueError("%s: batch['K'] must be float64 [B,3,3] = %s, got %s %s"
                         % (name, (B, 3, 3), batch["K"].dtype, tuple(batch["K"].shape)))
    if "RTs" in keys and (batch["RTs"].dim() != 4 or batch["RTs"].shape[0] != B):
        raise ValueError("%s: batch['RTs'] must be [B,n_obj,3,4], got %s" % (name, tuple(batch["RTs"].shape)))
    for k, t in batch.items():
        if not t.is_cuda or t.device != dpt.device:
            raise ValueError("%s: batch[%r] is on %s; every tensor must be a CUDA tensor on one CUDA device (dpt: %s)"
                             % (name, k, t.device, dpt.device))


def build_ffb6d_inputs(dpt, cam_scale, K, rgb, nrm_map, n_points, seed=0, fill=True, min_valid=MIN_VALID_PIXELS,
                       k=K_NEIGH, index_dtype=torch.int32, streams=None, normals="input"):
    """The inference half of the datasets' ``get_item`` for a batch on the GPU: every key ``FFB6D.forward`` reads,
    from decoded frames that have no labels and no objects (what a deployed model sees).

    The depth handling and the sampling are :func:`build_ffb6d_item`'s (``fill=True`` YCB, ``fill=False``
    LineMOD), and :func:`ffb6d_b200.ops.point_input` builds ``cld_rgb_nrm``.  Every key returned here is bitwise
    what :func:`build_ffb6d_item` returns under it for the same arguments.  No host synchronisation; with ``K``
    given as device intrinsics (float64 ``[4]`` / ``[B,4]`` ``(fx, fy, cx, cy)`` CUDA) nothing is copied from the
    host either, and the whole call can be captured in a CUDA graph.

    :param dpt: ``[B,H,W]`` ``torch.uint16`` CUDA, the depth PNGs' raw values; :param cam_scale: raw units per metre
    :param K: camera matrix as :func:`ffb6d_b200.ops.backproject` takes it
    :param rgb: ``[B,H,W,3]`` uint8; :param nrm_map: ``[B,H,W,3]`` float32 / float64 normal map, or None with
      ``normals="device"``
    :param normals: ``"input"``: ``nrm_map`` is the normal map; ``"device"``: it is computed from the depth by
      :func:`ffb6d_b200.ops.depth_normal` with the datasets' ``normalSpeed`` arguments, from the completed depth's
      millimetre map (YCB, :func:`ffb6d_b200.ops.depth_to_mm`) or the raw depth (LineMOD)
    :return: dict with ``rgb [B,3,H,W]`` uint8, ``cld_rgb_nrm [B,9,N]``, ``choose [B,1,N]``, ``dpt_map_m [B,H,W]``,
      the tensors of :func:`build_ffb6d_indices` (``cld_xyz*`` and the index tensors) and ``valid [B]`` bool
    """
    check_normals(normals, "build_ffb6d_inputs", nrm_map)
    return _build_inputs(dpt, cam_scale, K, rgb, nrm_map, n_points, seed, fill, min_valid, k, index_dtype, streams,
                         normals=normals)[0]


def _build_inputs(dpt, cam_scale, K, rgb, nrm_map, n_points, seed, fill, min_valid, k, index_dtype, streams,
                  labels=None, obj=None, normals="input"):
    """:func:`build_ffb6d_inputs`; with ``labels`` and ``obj`` (the device object tables) ``cld_rgb_nrm`` comes
    from :func:`ffb6d_b200.ops.point_item` instead, and its targets are returned as well: ``(inputs,
    (labels_pt, kp_targ_ofst, ctr_targ_ofst) or None)``."""
    import numpy as np
    from .ops import (_fill_depth, _intrinsics_arg, sample_valid_pixels, point_input, point_item, depth_normal,
                      depth_to_mm)
    if not isinstance(dpt, torch.Tensor) or dpt.dim() != 3 or dpt.dtype != torch.uint16:
        raise ValueError("dpt must be a [B,H,W] torch.uint16 CUDA tensor")
    dev = dpt.device
    if fill:
        filled, depth_m = _fill_depth(dpt, cam_scale)
        choose, n_valid = sample_valid_pixels(filled, n_points, seed=seed, min_depth=MSK_DP_THRESHOLD,
                                              return_count=True)
    else:
        # dpt_m = dpt_mm.astype(np.float32) / cam_scale; msk_dp = dpt_mm > 1e-6 is dpt_m > 0
        cs = float(np.float32(cam_scale))
        if not (cs > 0.0 and np.isfinite(cs)):
            raise ValueError("cam_scale must be positive and finite, got %r" % (cam_scale,))
        depth_m = dpt.to(torch.float32) / torch.full((), cs, dtype=torch.float32, device=dev)
        choose, n_valid = sample_valid_pixels(depth_m, n_points, seed=seed, min_depth=0.0, return_count=True)
    intr = _intrinsics_arg(K, dpt.shape[0], dev)[0]           # one copy of a host K, shared by every use
    if normals == "device":
        # the depth the datasets give normalSpeed: YCB the completed depth (after add_real_back), LineMOD dpt_mm
        nrm_map = depth_normal(depth_to_mm(filled, YCB_MM_DIVISOR) if fill else dpt, intr, *NORMAL_ARGS)
    item = build_ffb6d_indices_from_depth(depth_m, intr, choose, k=k, index_dtype=index_dtype, streams=streams)
    targets = None
    if labels is None:
        cld_rgb_nrm = point_input(depth_m, intr, choose, rgb, nrm_map)
    else:
        cld_rgb_nrm, *targets = point_item(depth_m, intr, choose, rgb, labels, nrm_map, obj["obj_cls"],
                                           obj["obj_kps"], obj["obj_ctr"])
    item.update(rgb=rgb.permute(0, 3, 1, 2).contiguous(), cld_rgb_nrm=cld_rgb_nrm, choose=choose, dpt_map_m=depth_m,
                valid=n_valid >= int(min_valid))
    return item, targets


def build_ffb6d_item(dpt, cam_scale, K, rgb, labels, nrm_map, objects, n_points, seed=0, fill=True,
                     min_valid=MIN_VALID_PIXELS, k=K_NEIGH, index_dtype=torch.int32, streams=None, normals="input"):
    """The datasets' ``get_item`` for a batch on the GPU, from the decoded images to every ``item_dict`` key.

    ``fill=True`` is YCB (datasets/ycb/ycb_dataset.py:204-336): depth completion of the raw depth, ``msk_dp``,
    sampling, ``dpt_m`` and the 22 searches (as :func:`build_ffb6d_indices_from_raw_depth`).  ``fill=False`` is
    LineMOD (datasets/linemod/linemod_dataset.py:251-386): the raw ``dpt_mm`` as it is, with ``cam_scale`` 1000.
    Then :func:`ffb6d_b200.ops.point_item` builds ``cld_rgb_nrm``, ``labels`` and the offset targets of the
    sampled points.  The points are drawn by :func:`ffb6d_b200.ops.sample_valid_pixels` with ``seed``: the
    reference's distribution, not numpy's random stream.  This is :func:`build_ffb6d_inputs` plus the label and
    target keys.

    :param dpt: ``[B,H,W]`` ``torch.uint16`` CUDA, the depth PNGs' raw values
    :param cam_scale: raw units per metre (YCB ``meta['factor_depth']``, LineMOD 1000), used as float32
    :param K: camera matrix as :func:`ffb6d_b200.ops.backproject` takes it
    :param rgb: ``[B,H,W,3]`` uint8; :param labels: ``[B,H,W]`` uint8 label image
    :param nrm_map: ``[B,H,W,3]`` float32 / float64 normal map (computed by the caller, see INTEGRATION.md), or None
      with ``normals="device"``
    :param objects: the per-object arrays of :func:`ffb6d_b200.item.pose_gt_objects`, as a dict of ``[B,...]``
      arrays or tensors (what a DataLoader collates) or a list of B per-frame dicts
    :param min_valid: frames with fewer valid depth pixels are flagged ``valid = False``: the reference returns
      ``None`` for them and draws another frame, which a device batch cannot do, so the trainer masks them
    :return: dict with the reference's keys ``rgb [B,3,H,W]`` uint8, ``cld_rgb_nrm [B,9,N]``, ``choose [B,1,N]``,
      ``labels [B,N]``, ``rgb_labels [B,H,W]`` int32, ``dpt_map_m [B,H,W]``, ``RTs``, ``kp_targ_ofst [B,N,n_kps,3]``,
      ``ctr_targ_ofst [B,N,3]``, ``cls_ids``, ``ctr_3ds``, ``kp_3ds``, the tensors of :func:`build_ffb6d_indices`,
      and ``valid [B]`` bool
    :param normals: ``"input"`` or ``"device"``, as for :func:`build_ffb6d_inputs`
    """
    import numpy as np
    check_normals(normals, "build_ffb6d_item", nrm_map)
    if not isinstance(dpt, torch.Tensor) or dpt.dim() != 3 or dpt.dtype != torch.uint16:
        raise ValueError("dpt must be a [B,H,W] torch.uint16 CUDA tensor")
    dev = dpt.device
    if isinstance(objects, (list, tuple)):
        objects = {key: np.stack([np.asarray(o[key]) for o in objects]) for key in _OBJECT_KEYS}
    obj = {key: torch.as_tensor(objects[key]).to(dev) for key in _OBJECT_KEYS}
    item, (labels_pt, kp_targ_ofst, ctr_targ_ofst) = _build_inputs(
        dpt, cam_scale, K, rgb, nrm_map, n_points, seed, fill, min_valid, k, index_dtype, streams, labels, obj,
        normals)
    item.update(labels=labels_pt, rgb_labels=labels.to(torch.int32), RTs=obj["RTs"], kp_targ_ofst=kp_targ_ofst,
                ctr_targ_ofst=ctr_targ_ofst, cls_ids=obj["cls_ids"], ctr_3ds=obj["ctr_3ds"], kp_3ds=obj["kp_3ds"])
    return item


# the batch keys build_ffb6d_train_item reads (INTEGRATION.md, the worker / trainer split): the decoded images and the
# background frames, the worker's augmentation draws (host values), and the object tables of pose_gt_objects
TRAIN_IMAGE_KEYS = ("dpt", "rgb", "labels", "nrm_map", "back_rgb", "back_labels", "back_dpt")
TRAIN_RECORD_KEYS = ("jitter", "jittered", "plans", "augment", "apply_rgb")
TRAIN_BATCH_KEYS = TRAIN_IMAGE_KEYS + TRAIN_RECORD_KEYS + _OBJECT_KEYS


def check_train_batch(batch, dataset, name, normals="input", meshes=None, crops=None):
    """``ValueError`` unless ``dataset`` is known and ``batch`` is a dict holding every key of ``TRAIN_BATCH_KEYS``
    (without ``nrm_map``, which it must not hold, under ``normals="device"``), with ``meshes`` the render keys
    (:func:`check_render_batch`) and with ``crops`` the fuse keys (:func:`check_fuse_batch`)."""
    check_dataset(dataset, name)
    keys = _normal_keys(batch, name, TRAIN_BATCH_KEYS, normals)
    if not isinstance(batch, dict):
        raise ValueError("%s: the batch must be a dict, got %s" % (name, type(batch).__name__))
    check_render_batch(batch, dataset, name, meshes, normals)
    check_fuse_batch(batch, dataset, name, crops, normals)
    missing = [k for k in keys if k not in batch]
    if missing:
        raise ValueError("%s: the batch lacks %s" % (name, missing))


def check_render_batch(batch, dataset, name, meshes, normals):
    """The render keys of a training batch (``ffb6d_b200.render.RENDER_KEYS``), checked on the host before any CUDA
    work: with ``meshes`` (a :class:`~ffb6d_b200.render.RenderMeshTable`, LineMOD only, with ``normals="device"``)
    the batch holds all four, ``rendered [B]`` bool, ``render_mesh [B,M]`` int32, ``render_RTs [B,M,3,4]`` float32
    and ``render_label [B,M]`` uint8, host values or CUDA tensors, and host mesh indices lie in ``[-1,
    len(meshes))``; without it, none.

    ``meshes`` with ``normals="input"`` is refused: the reference takes a render's normals from the render's own
    ``dpt_mm`` (linemod_dataset.py:251-254), which exists only on the device here, so no normal map the worker sends
    can belong to a rendered frame."""
    import numpy as np
    from .render import RENDER_KEYS, RenderMeshTable, check_mesh_indices
    held = [k for k in RENDER_KEYS if k in batch]
    if meshes is None:
        if held:
            raise ValueError("%s: the batch holds the render keys %s but no meshes were given (pass meshes=, a "
                             "RenderMeshTable)" % (name, held))
        return
    if dataset == "ycb":
        raise ValueError("%s: meshes= renders LineMOD frames; YCB ships its synthetic frames and its meshes are "
                         "textured" % name)
    if not isinstance(meshes, RenderMeshTable):
        raise ValueError("%s: meshes must be a RenderMeshTable, got %s" % (name, type(meshes).__name__))
    if normals != "device":
        raise ValueError("%s: meshes= needs normals='device': a rendered frame's normals come from its own depth, "
                         "which exists only on the device, so a normal map from the batch cannot belong to it" % name)
    missing = [k for k in RENDER_KEYS if k not in batch]
    if missing:
        raise ValueError("%s: meshes were given but the batch lacks the render keys %s" % (name, missing))
    B = batch["dpt"].shape[0] if hasattr(batch.get("dpt"), "shape") else None
    M = tuple(batch["render_mesh"].shape)[1:2] if hasattr(batch["render_mesh"], "shape") else ()
    want = {"rendered": (torch.bool, (B,)), "render_mesh": (torch.int32, (B,) + M),
            "render_RTs": (torch.float32, (B,) + M + (3, 4)), "render_label": (torch.uint8, (B,) + M)}
    for k, (dtype, shape) in want.items():
        t = batch[k] if isinstance(batch[k], torch.Tensor) else torch.as_tensor(np.asarray(batch[k]))
        if t.dtype != dtype or tuple(t.shape) != shape or len(M) != 1:
            raise ValueError("%s: batch[%r] must be %s %s, got %s %s" % (name, k, dtype, shape, t.dtype,
                                                                       tuple(t.shape)))
    check_mesh_indices(meshes, batch["render_mesh"], name)


def check_fuse_batch(batch, dataset, name, crops, normals):
    """The fuse keys of a training batch (``ffb6d_b200.fuse_frames.FUSE_KEYS``), checked on the host before any CUDA
    work: with ``crops`` (a :class:`~ffb6d_b200.fuse_frames.FuseCropTable`, LineMOD only, with ``normals="device"``)
    the batch holds all four, ``fused [B]`` bool, ``fuse_crop [B,M]`` int32, ``fuse_offset [B,M,2]`` int32 and
    ``fuse_label [B,M]`` uint8, host values or CUDA tensors, and a per-frame ``K [B,3,3]`` float64 (a fused frame's
    camera is its own); host crop indices lie in ``[-1, len(crops))`` and no host frame is both ``rendered`` and
    ``fused``.  Without ``crops``, none of the fuse keys.

    ``crops`` with ``normals="input"`` is refused for the reason ``meshes`` is (:func:`check_render_batch`): a fused
    frame's normals come from its own composed ``dpt_mm`` (linemod_dataset.py:251-254), which exists only on the
    device."""
    import numpy as np
    from .fuse_frames import FUSE_KEYS, FuseCropTable, check_crop_indices
    held = [k for k in FUSE_KEYS if k in batch]
    if crops is None:
        if held:
            raise ValueError("%s: the batch holds the fuse keys %s but no crops were given (pass crops=, a "
                             "FuseCropTable)" % (name, held))
        return
    if dataset == "ycb":
        raise ValueError("%s: crops= composes LineMOD's fuse frames; YCB ships its synthetic frames" % name)
    if not isinstance(crops, FuseCropTable):
        raise ValueError("%s: crops must be a FuseCropTable, got %s" % (name, type(crops).__name__))
    if normals != "device":
        raise ValueError("%s: crops= needs normals='device': a fused frame's normals come from its own depth, which "
                         "exists only on the device, so a normal map from the batch cannot belong to it" % name)
    missing = [k for k in FUSE_KEYS if k not in batch]
    if missing:
        raise ValueError("%s: crops were given but the batch lacks the fuse keys %s" % (name, missing))
    if "K" not in batch:
        raise ValueError("%s: crops= needs a per-frame K [B,3,3] float64 in the batch: a fused frame's camera is its "
                         "own (draw_fuse_frame)" % name)
    B = batch["dpt"].shape[0] if hasattr(batch.get("dpt"), "shape") else None
    M = tuple(batch["fuse_crop"].shape)[1:2] if hasattr(batch["fuse_crop"], "shape") else ()
    want = {"fused": (torch.bool, (B,)), "fuse_crop": (torch.int32, (B,) + M),
            "fuse_offset": (torch.int32, (B,) + M + (2,)), "fuse_label": (torch.uint8, (B,) + M),
            "K": (torch.float64, (B, 3, 3))}
    host = {}
    for k, (dtype, shape) in want.items():
        t = batch[k] if isinstance(batch[k], torch.Tensor) else torch.as_tensor(np.asarray(batch[k]))
        if t.dtype != dtype or tuple(t.shape) != shape or len(M) != 1:
            raise ValueError("%s: batch[%r] must be %s %s, got %s %s" % (name, k, dtype, shape, t.dtype,
                                                                       tuple(t.shape)))
        host[k] = None if t.is_cuda else t
    check_crop_indices(crops, batch["fuse_crop"], name)
    rendered = batch.get("rendered")
    if host["fused"] is not None and rendered is not None and not (isinstance(rendered, torch.Tensor)
                                                                   and rendered.is_cuda):
        both = np.flatnonzero(host["fused"].numpy() & np.asarray(rendered, dtype=bool).reshape(-1))
        if both.size:
            raise ValueError("%s: frames %s are flagged both rendered and fused" % (name, both.tolist()))


def build_ffb6d_train_item(batch, *, dataset, cam_scale, K, n_points, seed, normals="input", meshes=None,
                           crops=None):
    """The training ``get_item`` of a collated batch on the GPU, in the reference's order: the colour jitter, the first
    ``rgb_add_noise``, ``add_real_back``, the second ``rgb_add_noise``, :func:`build_ffb6d_item` (``fill=True`` for
    YCB, ``False`` for LineMOD) and ``model_fn``'s ``rgb.float()``.  This is INTEGRATION.md's trainer composition in
    one call.

    :param batch: what the DataLoader collates from the worker's dict: CUDA tensors ``dpt``, ``rgb``, ``labels``,
      ``nrm_map``, ``back_rgb``, ``back_labels``, ``back_dpt`` and the object tables of
      :func:`ffb6d_b200.item.pose_gt_objects`; the worker's draws on the host: ``jitter [B,8]``, ``jittered [B]``,
      ``plans [B,2,REC_LEN]``, ``augment [B]``, ``apply_rgb [B]``; optionally ``K [B,3,3]`` float64, one camera
      matrix per frame (it replaces ``K``)
    :param dataset: ``"ycb"`` or ``"linemod"``; :param cam_scale: raw depth units per metre
    :param K: the camera matrix as :func:`build_ffb6d_item` takes it
    :param seed: the key of the noise draws and of the point sampling: an int, or a one-element int64 / uint64 CUDA
      tensor read on the device (the same bits as the int of the same 64 bits)
    :param normals: ``"input"``: the batch's ``nrm_map``; ``"device"``: the batch holds no ``nrm_map`` and the normals
      are computed from the composed depth (YCB: completed too), in the reference's order (:func:`build_ffb6d_item`)
    :param meshes: LineMOD only, with ``normals="device"``: a :class:`~ffb6d_b200.render.RenderMeshTable`.  The batch
      then also holds the render keys (``rendered [B]`` bool, ``render_mesh [B,M]`` int32, ``render_RTs [B,M,3,4]``
      float32, ``render_label [B,M]`` uint8, host draws or CUDA tensors), and the flagged frames' ``dpt`` / ``rgb`` /
      ``labels`` are replaced by :func:`~ffb6d_b200.render.render_rgbd` frames (``dpt_mm``) before the colour jitter,
      as the reference loads a render pickle before ``get_item``'s augmentation.  Every frame's normals are then
      computed from its composed depth, the rendered frames' from the render's.  The renders go into copies; the
      batch's tensors are not written
    :param crops: LineMOD only, with ``normals="device"``: a :class:`~ffb6d_b200.fuse_frames.FuseCropTable`.  The
      batch then also holds the fuse keys (``fused [B]`` bool, ``fuse_crop [B,M]`` int32, ``fuse_offset [B,M,2]``
      int32, ``fuse_label [B,M]`` uint8, host draws or CUDA tensors) and a per-frame ``K``, and the flagged frames'
      crops are pasted by :func:`~ffb6d_b200.fuse_frames.fuse_rgbd` over their ``dpt`` / ``rgb`` / ``labels``,
      after the renders and before the colour jitter.  A frame is rendered or fused, not both.  The pastes go into
      copies; the batch's tensors are not written
    :return: the dict of :func:`build_ffb6d_item` with ``rgb`` as float32
    """
    check_train_batch(batch, dataset, "build_ffb6d_train_item", normals, meshes, crops)
    return _train_item(batch, dataset, cam_scale, K, n_points, seed, normals=normals, meshes=meshes, crops=crops)


def _render_frames(batch, meshes, K, in_place):
    """The batch with its flagged frames' ``dpt`` / ``rgb`` / ``labels`` rendered (``dpt_mm``): into the batch's own
    tensors with ``in_place`` (a graph's input buffers), else into copies."""
    from .render import render_rgbd
    out = tuple(batch[k] if in_place else batch[k].clone(memory_format=torch.contiguous_format)
                for k in ("dpt", "rgb", "labels"))
    B, H, W = out[0].shape
    render_rgbd(meshes, batch["render_mesh"], batch["render_RTs"], batch["render_label"], K, H, W,
                active=batch["rendered"], out=out)
    return dict(batch, dpt=out[0], rgb=out[1], labels=out[2])


def _fuse_frames(batch, crops, in_place):
    """The batch with its flagged frames' crops pasted over ``dpt`` / ``rgb`` / ``labels``: into the batch's own
    tensors with ``in_place`` (a graph's input buffers, or copies the renders already made), else into copies."""
    from .fuse_frames import fuse_rgbd
    out = tuple(batch[k] if in_place else batch[k].clone(memory_format=torch.contiguous_format)
                for k in ("dpt", "rgb", "labels"))
    B, H, W = out[0].shape
    fuse_rgbd(crops, batch["fuse_crop"], batch["fuse_offset"], batch["fuse_label"], H, W, active=batch["fused"],
              out=out)
    return dict(batch, dpt=out[0], rgb=out[1], labels=out[2])


def _train_item(batch, dataset, cam_scale, K, n_points, seed, records=None, normals="input", meshes=None,
                in_place=False, crops=None):
    """:func:`build_ffb6d_train_item` on a checked batch.  ``records``: host copies of ``batch['jitter']`` and
    ``batch['plans']`` when the batch holds those on the device (a graph's input buffers); the host copies are what
    the entry points check, the device ones what the kernels read.  ``in_place``: render and paste into the batch's
    tensors."""
    import numpy as np
    from .ops import _frame_intrinsics, add_real_back, color_jitter, rgb_add_noise
    if "K" in batch:
        K = batch["K"]
        if isinstance(K, torch.Tensor) and K.is_cuda:
            K = _frame_intrinsics(K)
    if meshes is not None:
        batch = _render_frames(batch, meshes, K, in_place)
    if crops is not None:
        batch = _fuse_frames(batch, crops, in_place or meshes is not None)
    if records is None:
        jitter, plans = np.asarray(batch["jitter"]), np.asarray(batch["plans"])
        jitter_d = plans_d = None
    else:
        jitter, plans = records["jitter"], records["plans"]
        jitter_d, plans_d = batch["jitter"], batch["plans"]
    rgb = color_jitter(batch["rgb"], jitter, active=batch["jittered"], plan_dev=jitter_d)
    rgb = rgb_add_noise(rgb, plans[:, 0], seed, plan_dev=None if plans_d is None else plans_d[:, 0])
    rgb, dpt = add_real_back(rgb, batch["labels"], batch["dpt"], batch["back_rgb"], batch["back_labels"],
                             batch["back_dpt"], batch["apply_rgb"], dataset, active=batch["augment"])
    rgb = rgb_add_noise(rgb, plans[:, 1], seed, plan_dev=None if plans_d is None else plans_d[:, 1])
    item = build_ffb6d_item(dpt, cam_scale, K, rgb, batch["labels"], batch.get("nrm_map"), batch, n_points, seed=seed,
                            fill=dataset == "ycb", normals=normals)
    item["rgb"] = item["rgb"].float()
    return item
