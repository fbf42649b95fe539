"""oracle/net_oracle.py -- TEST INFRASTRUCTURE ONLY.  What tests/golden/make_ffb6d_golden.py (which runs the
reference's own ``FFB6D``) and the tests of tests/golden/ffb6d_net_cases.npz share, so that the fixture stores
nothing but digests of the reference's index tensors and its outputs: the seeded weights, the seeded inputs with
their digests, the sampled positions, and the packing of many sampled tensors into a few arrays.

* Weights: :func:`seeded_state` is ``oracle/cnn_oracle.py``'s per-key draw over the whole state dict, rounded to
  float32, so the reference in float64, the reference in float32 and a float32 model all hold the same numbers.
* The eval run's running statistics are this batch's (:func:`eval_tensors`), stored in the fixture.
* Inputs: two 120x160 frames with 4096 points (:func:`ffb6d_b200.synthetic.make_batch`), a seeded image and seeded
  training targets.  The deepest point level has 16 points per frame: K = 16 stays legal, and the batch statistics
  there are taken over 32 positions.
* Index tensors: the fixture holds the sha256 of each of the reference's 22 index tensors; :func:`oracle_indices`
  recomputes them with the exact CPU oracle and :func:`check_indices` holds them to the digests, as
  ``schedule_digest.json`` does for the full-size frames.
* Samples: tensor number ``k`` of a group is kept at ``positions(seed + k, size, n)``.
"""
import hashlib

import numpy as np

from . import cnn_oracle

SEEDS, N_POINTS, H, W = (3, 4), 4096, 120, 160
N_CLASSES, N_KPS = 22, 8
INPUT_KEYS = ("rgb", "cld_rgb_nrm", "choose", "cld", "dpt_xyz", "labels", "kp_targ_ofst", "ctr_targ_ofst")
END_POINTS = ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")
LOSSES = ("loss_rgbd_seg", "loss_kp_of", "loss_ctr_of", "loss_all")
STAGE_SAMPLES, PARAM_SAMPLES = 512, 48
STAGE_SEED, GRAD_SEED, STAT_SEED = 100, 1000, 3000


def seeded_state(shapes, seed=0):
    """``{key: float32 / int64 ndarray}`` for the ``{key: shape}`` of a whole FFB6D state dict."""
    return {k: v if v.dtype == np.int64 else v.astype(np.float32)
            for k, v in cnn_oracle.seeded_state(shapes, seed).items()}


def seeded_tensors(state_dict, seed=0):
    """:func:`seeded_state` for a torch ``state_dict()``, as float32 / int64 tensors."""
    import torch
    vals = seeded_state({k: tuple(v.shape) for k, v in state_dict.items()}, seed)
    return {k: torch.from_numpy(vals[k]) for k in state_dict}


def running_keys(state_dict):
    return sorted(k for k in state_dict if k.endswith(("running_mean", "running_var")))


def eval_tensors(state_dict, fixture, seed=0):
    """The eval run's state: :func:`seeded_tensors` with every BatchNorm's running statistics replaced by the
    fixture's ``eval/running`` (float32, all of them end to end in the order of their sorted keys): the statistics of
    this very batch, as a trained network has them for its data.  With drawn statistics the activations of the 60-layer
    network reach 1e6 and a comparison relative to their scale sees little."""
    import torch
    sd, at = seeded_tensors(state_dict, seed), 0
    flat = torch.from_numpy(np.asarray(fixture["eval/running"]))
    for k in running_keys(state_dict):
        n = sd[k].numel()
        sd[k] = flat[at:at + n].reshape(sd[k].shape).clone()
        at += n
    assert at == flat.numel()
    return sd


def make_inputs():
    """The fixture's inputs as numpy arrays (``INPUT_KEYS``): the synthetic batch, a seeded image and seeded targets
    (half of the points background, as a frame with objects has them)."""
    from ffb6d_b200.synthetic import make_batch
    batch = make_batch(list(SEEDS), n_points=N_POINTS, h=H, w=W)
    B = len(SEEDS)
    rs = np.random.RandomState(7)
    data = {k: batch[k] for k in ("cld_rgb_nrm", "choose", "cld", "dpt_xyz")}
    data["rgb"] = rs.uniform(-1.0, 1.0, (B, 3, H, W)).astype(np.float32)
    labels = rs.randint(1, N_CLASSES, (B, N_POINTS)).astype(np.int32)
    labels[rs.rand(B, N_POINTS) < 0.5] = 0
    data["labels"] = labels
    data["kp_targ_ofst"] = rs.randn(B, N_POINTS, N_KPS, 3).astype(np.float32)
    data["ctr_targ_ofst"] = rs.randn(B, N_POINTS, 3).astype(np.float32)
    return data


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def check_inputs(data, fixture):
    """Fail with the key's name if a regenerated input is not the one the fixture was made from."""
    for k in INPUT_KEYS:
        assert sha(data[k]) == str(fixture["digest/" + k]), \
            "the regenerated input %r differs from the one ffb6d_net_cases.npz was made from" % k


def oracle_indices(data):
    """The 22 index arrays ``{key: [B,Q,K] int32}`` of the batch from the exact CPU oracle (``oracle/cpu_oracle.py``),
    frame by frame as the datasets build them."""
    from ffb6d_b200.synthetic import image_pyramid_np
    from ffb6d_b200.tables import knn_schedule
    from . import cpu_oracle
    idx = {}
    for b in range(len(SEEDS)):
        sets = {("cld", i): data["cld"][b][: N_POINTS // 4 ** i] for i in range(5)}
        sets.update({("img", sr): p for sr, p in image_pyramid_np(data["dpt_xyz"][b]).items()})
        for key, s, q, k in knn_schedule(N_POINTS, H, W):
            idx.setdefault(key, []).append(cpu_oracle.knn_search(sets[s][None], sets[q][None], k)[0])
    return {k: np.stack(v) for k, v in idx.items()}


def check_indices(idx, fixture):
    """Fail with the key's name if an index array is not, bit for bit, the one the reference's compiled KNN gave
    when the fixture was made (the frames have no exact-distance ties among a query's neighbours)."""
    assert sorted("idx_sha256/" + k for k in idx) == sorted(k for k in fixture if k.startswith("idx_sha256/"))
    for k, v in idx.items():
        assert v.dtype == np.int32 and sha(v) == str(fixture["idx_sha256/" + k]), \
            "index tensor %r differs from the reference's (ffb6d_net_cases.npz)" % k


def network_inputs(data, idx, device="cpu", dtype=None, index_dtype=None):
    """The reference's input dict as torch tensors from :func:`make_inputs` and the index arrays ``{key: [B,Q,K]}``
    of the schedule (``cld_sub_idx{i}`` = the first rows of ``cld_nei_idx{i}``, ``cld_xyz{i}`` = the first rows of
    the cloud, ycb_dataset.py:278-283)."""
    import torch
    dtype = dtype or torch.float32
    index_dtype = index_dtype or torch.int32
    inp = {"rgb": torch.from_numpy(data["rgb"]).to(device, dtype),
           "cld_rgb_nrm": torch.from_numpy(data["cld_rgb_nrm"]).to(device, dtype),
           "choose": torch.from_numpy(data["choose"]).to(device, index_dtype)}
    n = N_POINTS
    for i in range(4):
        inp["cld_xyz%d" % i] = torch.from_numpy(np.ascontiguousarray(data["cld"][:, :n])).to(device, dtype)
        n //= 4
        inp["cld_sub_idx%d" % i] = torch.from_numpy(np.ascontiguousarray(idx["cld_nei_idx%d" % i][:, :n])).to(
            device, index_dtype)
    for k, v in idx.items():
        inp[k] = torch.from_numpy(v).to(device, index_dtype)
    return inp


def targets(data, device="cpu", dtype=None):
    import torch
    return {"labels": torch.from_numpy(data["labels"]).to(device),
            "kp_targ_ofst": torch.from_numpy(data["kp_targ_ofst"]).to(device, dtype or torch.float32),
            "ctr_targ_ofst": torch.from_numpy(data["ctr_targ_ofst"]).to(device, dtype or torch.float32)}


def positions(seed, size, n):
    """Sorted flat positions: all of them up to ``n``, else ``n`` drawn without replacement from ``RandomState(seed)``."""
    if size <= n:
        return np.arange(size)
    return np.sort(np.random.RandomState(seed).choice(size, n, replace=False))


def sample(a, seed, n):
    """``a`` (array or tensor, any device) at :func:`positions`, as a float64 numpy vector."""
    if hasattr(a, "detach"):
        import torch
        flat = a.detach().reshape(-1)
        pos = torch.from_numpy(positions(seed, flat.numel(), n)).to(flat.device)
        return flat[pos].double().cpu().numpy()
    flat = np.asarray(a).reshape(-1)
    return flat[positions(seed, flat.size, n)].astype(np.float64)


def pack(group, items, seed, n):
    """``items``: ``[(name, float64 array, float32 array)]`` of one group.  Stored per group: the names, the shapes
    (padded with 0 to four dimensions), the float64 norms, the sampled float64 values of all tensors end to end, and
    of the float32 run its distance from the float64 run only: the norm over the whole tensor (``err32``), and at
    the sampled positions the largest difference (``e32max``) and the norm of the differences (``e32norm``)."""
    d = [sample(b, seed + k, n) - sample(a, seed + k, n) for k, (_, a, b) in enumerate(items)]
    return {group + "/names": np.array([name for name, _, _ in items]),
            group + "/shapes": np.array([list(a.shape) + [0] * (4 - a.ndim) for _, a, _ in items], np.int64),
            group + "/norm": np.array([np.linalg.norm(a.reshape(-1)) for _, a, _ in items], np.float64),
            group + "/err32": np.array([np.linalg.norm((b.astype(np.float64) - a).reshape(-1)) for _, a, b in items],
                                       np.float64),
            group + "/e32max": np.array([np.abs(x).max() for x in d], np.float64),
            group + "/e32norm": np.array([np.linalg.norm(x) for x in d], np.float64),
            group + "/f64": np.concatenate([sample(a, seed + k, n) for k, (_, a, _) in enumerate(items)])}


def unpack(fixture, group, n):
    """``{name: dict(k, shape, norm, err32, e32max, e32norm, f64)}`` of a packed group, in stored order."""
    out, at = {}, 0
    for k, name in enumerate(fixture[group + "/names"]):
        shape = tuple(int(d) for d in fixture[group + "/shapes"][k] if d)
        cnt = min(int(np.prod(shape)), n)
        out[str(name)] = dict(k=k, shape=shape, f64=fixture[group + "/f64"][at:at + cnt],
                              **{f: float(fixture[group + "/" + f][k]) for f in ("norm", "err32", "e32max", "e32norm")})
        at += cnt
    return out
