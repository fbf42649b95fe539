"""GPU: the deterministic backward taken under torch's determinism switches.  The linear-size segment CSR against a
stable torch.sort restatement (and the counter plan) at every gather shape of a 480x640 step; the gather + max
backward without atomics against float64 by the arg-max rule of the atomic kernel; the split-ordered weight
gradient against float64; bitwise repeatability over calls and CUDA-graph replays; which kernels a training step
launches under each switch; and bit-identical training of the whole FFB6DFusionNet.  Inputs come from seeds."""
import contextlib
import re

import numpy as np
import pytest
import torch

import test_gpu_model
from test_gpu_train import close_fp32, WGRAD_CASES, WGRAD_CENTRED
from ffb6d_b200 import ops
from ffb6d_b200 import tables as T
from ffb6d_b200._lib import lib, check, LAYOUT_NCS
from ffb6d_b200.model import FFB6DFusionNet
from ffb6d_b200.schedule import build_ffb6d_indices
from ffb6d_b200.synthetic import make_batch

pytestmark = pytest.mark.gpu

GATHERS = T.gather_schedule()
N_LEVEL = [T.set_size(("cld", i)) for i in range(5)]
# the K = 1 gathers of Building_block (_gather_cm): cld_nei_idx{i} [B, N_i, 16] flattened onto the N_i points
NEIGHBOURS = [("cld_nei_idx%d" % i, N_LEVEL[i]) for i in range(4)]
_indices = {}


@contextlib.contextmanager
def switches(algorithms=False, cudnn=False):
    saved = torch.are_deterministic_algorithms_enabled(), torch.backends.cudnn.deterministic
    torch.use_deterministic_algorithms(algorithms)
    torch.backends.cudnn.deterministic = cudnn
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(saved[0])
        torch.backends.cudnn.deterministic = saved[1]


def step_indices(cuda, B=2):
    """The index tensors of ``B`` synthetic 480x640 frames, ``choose`` included."""
    if B not in _indices:
        batch = make_batch(list(range(11, 11 + B)))
        _indices[B] = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(cuda), torch.from_numpy(batch["dpt_xyz"]).to(cuda))
        _indices[B]["choose"] = torch.from_numpy(batch["choose"]).to(cuda)
    return _indices[B]


# ------------------------------------------------------------------ CSR plan
def want_csr(idx2, na):
    """offsets and entries of the CSR by a stable sort: out-of-range indices sort last and belong to no segment."""
    k = idx2.long()
    key = torch.where((k >= 0) & (k < na), k, torch.full_like(k, na))
    order = torch.sort(key, dim=1, stable=True).indices.int()
    counts = torch.stack([torch.bincount(key[b], minlength=na + 1)[:na] for b in range(key.shape[0])])
    offs = torch.cat((torch.zeros_like(counts[:, :1]), counts.cumsum(1)), 1).int()
    return offs, order


def check_csr(plan, idx2, na, what):
    off, ent = plan.csr()
    woff, went = want_csr(idx2, na)
    assert torch.equal(off, woff), what + ": offsets"
    for b in range(idx2.shape[0]):
        n = int(woff[b, -1])
        assert torch.equal(ent[b, :n], went[b, :n]), "%s: entries of frame %d" % (what, b)
    return off, ent


@pytest.mark.parametrize("g", GATHERS + [("neighbour", k, 0, n, n, 16) for k, n in NEIGHBOURS],
                         ids=["%s-%s" % (g[0], g[1]) for g in GATHERS] + [k for k, _ in NEIGHBOURS])
def test_csr_matches_stable_sort_at_step_shapes(cuda, g):
    op, key, _, S, Q, K = g
    idx = step_indices(cuda)[key]
    B = idx.shape[0]
    idx2 = idx.reshape(B, -1)
    assert idx2.shape[1] == Q * K, (key, tuple(idx.shape))
    off, ent = check_csr(ops.segment_csr(idx2, S), idx2, S, key)
    if key.startswith("p2r"):                  # the seven p2r maps: the counter plan's CSR too
        o2, e2 = ops.segment_plan(idx2, S).csr()
        assert torch.equal(off, o2)
        for b in range(B):
            assert torch.equal(ent[b, :int(off[b, -1])], e2[b, :int(off[b, -1])])


CSR_EDGES = {"one_segment": (2, 76800, 768), "na_much_larger": (2, 100, 300000), "p1": (3, 1, 7), "na1": (2, 4099, 1),
             "out_of_range_i64": (2, 5000, 300), "long_segments": (2, 50000, 20), "very_long_segments": (2, 50000, 3),
             "mid_segments_i64": (2, 60000, 1500)}


@pytest.mark.parametrize("case", list(CSR_EDGES))
def test_csr_edge_cases(cuda, case):
    B, P, na = CSR_EDGES[case]
    g = torch.Generator(device=cuda).manual_seed(len(case))
    idx = torch.randint(0, na, (B, P), generator=g, device=cuda, dtype=torch.int32)
    if case == "one_segment":
        idx.fill_(5)
    if case.endswith("i64"):
        idx = idx.long()
    if case == "out_of_range_i64":             # -1, NA and far beyond: no segment
        r = torch.rand((B, P), generator=g, device=cuda)
        idx = torch.where(r < 0.1, -1, torch.where(r < 0.2, na, torch.where(r < 0.25, na + 10 ** 10, idx)))
    check_csr(ops.segment_csr(idx, na), idx, na, case)
    grad = torch.randn((B, 9, P), generator=g, device=cuda)
    # the sum on the CSR equals the sum on the counter plan bit for bit (the same kernel on the same CSR)
    assert torch.equal(ops.segment_sum(grad, None, na, plan=ops.segment_csr(idx, na)), ops.segment_sum(grad, idx, na))


# ------------------------------------------------------------------ gather + max backward
def want_gather_bwd(f3, idx, gout):
    """float64 scatter of gout onto the arg-max neighbour: a NaN wins, else the first strict maximum; reads of
    out-of-range indices are clamped to row S-1 as in the kernels.  Returns (want, sum of |terms|, hit mask)."""
    B, Cc, S = f3.shape
    Q, K = idx.shape[1], idx.shape[2]
    ix = idx.long()
    rd = torch.where((ix >= 0) & (ix < S), ix, S - 1)
    vals = f3.gather(2, rd.reshape(B, 1, Q * K).expand(B, Cc, Q * K)).reshape(B, Cc, Q, K)
    ks = torch.arange(K, device=f3.device)
    nan = vals.isnan()
    first_nan = torch.where(nan, ks, K).amin(-1)
    m = torch.where(nan, -float("inf"), vals).amax(-1, keepdim=True)
    first_max = torch.where(vals == m, ks, K).amin(-1)
    kb = torch.where(nan.any(-1), first_nan, first_max)
    s = ix.unsqueeze(1).expand(B, Cc, Q, K).gather(3, kb.unsqueeze(-1)).squeeze(-1)        # [B, C, Q]
    ok = (s >= 0) & (s < S)
    sc = torch.where(ok, s, 0)
    g = torch.where(ok, gout.double(), 0.0)
    want = torch.zeros((B, Cc, S), dtype=torch.float64, device=f3.device).scatter_add_(2, sc, g)
    mag = torch.zeros_like(want).scatter_add_(2, sc, g.abs())
    hit = torch.zeros_like(want).scatter_add_(2, sc, ok.double()) > 0
    return want, mag, hit


def check_sum(out, want, mag, what):
    w = want.cpu().numpy()
    bound = np.maximum(np.spacing(np.abs(w).astype(np.float32)).astype(np.float64), 2.0 ** -36 * mag.cpu().numpy())
    err = np.abs(out.double().cpu().numpy() - w)
    bad = err > bound
    assert not bad.any(), "%s: %d elements out of bound, worst err %.3e" % (what, int(bad.sum()), err[bad].max())


def gather_grad(f_values, idx, gout, layout, deterministic):
    """The backward of ops.random_sample through autograd; f_values [B, C, S], stored channels-last for NSC."""
    leaf = (f_values.clone() if layout == "ncs" else f_values.transpose(1, 2).contiguous()).requires_grad_(True)
    f3 = leaf if layout == "ncs" else leaf.transpose(1, 2)
    with switches(algorithms=deterministic):
        out = ops._gather_max(f3, idx)
        out.backward(gout)
    return leaf.grad if layout == "ncs" else leaf.grad.transpose(1, 2)


def run_gather_case(f3, idx, gout, what):
    want, mag, hit = want_gather_bwd(f3.double(), idx, gout)
    for layout in ("ncs", "nsc"):
        det = gather_grad(f3, idx, gout, layout, True)
        check_sum(det, want, mag, "%s %s" % (what, layout))
        assert torch.equal(det[~hit], torch.zeros_like(det[~hit])), what + ": gradient where no arg-max lands"
        atomic = gather_grad(f3, idx, gout, layout, False)
        assert torch.equal(det != 0, atomic != 0), what + ": positions receiving gradient differ from the atomic path"
        assert torch.equal(det, gather_grad(f3, idx, gout, layout, True)), what + ": not bitwise repeatable"


RANDOM_SAMPLE = [g for g in GATHERS if g[0] == "random_sample"]


@pytest.mark.parametrize("g", RANDOM_SAMPLE, ids=[g[1] for g in RANDOM_SAMPLE])
def test_gather_max_bwd_det_at_step_shapes(cuda, g):
    _, key, Cc, S, Q, K = g
    idx = step_indices(cuda)[key]
    B = idx.shape[0]
    gen = torch.Generator(device=cuda).manual_seed(Cc + S)
    f3 = torch.randn((B, Cc, S), generator=gen, device=cuda)
    gout = torch.randn((B, Cc, Q), generator=gen, device=cuda)
    run_gather_case(f3, idx, gout, key)


@pytest.mark.parametrize("case", ["k_gt_s_duplicates", "nan_and_ties", "i64", "k1_choose"])
def test_gather_max_bwd_det_edge_cases(cuda, case):
    gen = torch.Generator(device=cuda).manual_seed(len(case) + 3)
    B, Cc, S, Q, K = {"k_gt_s_duplicates": (2, 40, 5, 300, 16), "nan_and_ties": (2, 33, 700, 500, 16),
                      "i64": (3, 70, 1000, 257, 8), "k1_choose": (2, 64, 19200, 3072, 1)}[case]
    idx = torch.randint(0, S, (B, Q, K), generator=gen, device=cuda, dtype=torch.int32)
    f3 = torch.randn((B, Cc, S), generator=gen, device=cuda)
    if case == "nan_and_ties":                 # three distinct values: ties everywhere; 1 % NaN
        f3 = torch.randint(0, 3, (B, Cc, S), generator=gen, device=cuda).float()
        f3[torch.rand((B, Cc, S), generator=gen, device=cuda) < 0.01] = float("nan")
    if case == "i64":
        idx = idx.long()
    gout = torch.randn((B, Cc, Q), generator=gen, device=cuda)
    run_gather_case(f3, idx, gout, case)


def test_nearest_interpolation_det_at_step_shapes(cuda):
    """The K = 1 gathers of a step (interp, p2r, choose, the neighbour gathers): plan choice by shape, one CSR."""
    ind = step_indices(cuda)
    cases = [(g[1], g[2], g[3], g[4]) for g in GATHERS if g[5] == 1] + [(k, 16, n, n * 16) for k, n in NEIGHBOURS]
    for key, Cc, S, Q in cases:
        idx = ind[key].reshape(ind[key].shape[0], Q, 1)
        B = idx.shape[0]
        gen = torch.Generator(device=cuda).manual_seed(S + Q)
        f3 = torch.randn((B, Cc, S), generator=gen, device=cuda)
        gout = torch.randn((B, Cc, Q), generator=gen, device=cuda)
        want, mag, _ = want_gather_bwd(f3.double(), idx, gout)
        det = gather_grad(f3, idx, gout, "ncs", True)
        check_sum(det, want, mag, key)
        assert torch.equal(det, gather_grad(f3, idx, gout, "ncs", True)), key


def test_gather_neighbour_bwd_det(cuda):
    gen = torch.Generator(device=cuda).manual_seed(7)
    idx = step_indices(cuda)["cld_nei_idx1"]
    B, N, K = idx.shape
    for D in (3, 40):
        pc = torch.randn((B, N, D), generator=gen, device=cuda, requires_grad=True)
        gout = torch.randn((B, N, K, D), generator=gen, device=cuda)
        grads = []
        for det in (True, True, False):
            pc.grad = None
            with switches(algorithms=det):
                ops.gather_neighbour(pc, idx).backward(gout)
            grads.append(pc.grad.clone())
        assert torch.equal(grads[0], grads[1])
        want = torch.zeros((B, N, D), dtype=torch.float64, device=cuda)
        mag = torch.zeros_like(want)
        ix = idx.reshape(B, -1).long()
        for b in range(B):
            want[b].index_add_(0, ix[b], gout[b].reshape(-1, D).double())
            mag[b].index_add_(0, ix[b], gout[b].reshape(-1, D).double().abs())
        check_sum(grads[0], want, mag, "gather_neighbour D=%d" % D)
        assert torch.equal(grads[0] != 0, grads[2] != 0)


# ------------------------------------------------------------------ weight gradient
def wgrad_det(dz, x1, x2, B, Co, P):
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    gw = torch.full((Co, C1 + C2), float("nan"), device=dz.device)
    nbytes = int(lib.ffb6d_fusion_mlp_wgrad_det_workspace_bytes(C1, C2, B, Co, P))
    ws = torch.full((nbytes,), 0xff, dtype=torch.uint8, device=dz.device)        # NaN partials unless overwritten
    check(lib.ffb6d_fusion_mlp_wgrad_det(dz.data_ptr(), x1.data_ptr(), C1, x2.data_ptr() if x2 is not None else None, C2,
                                         B, Co, P, ws.data_ptr(), nbytes, gw.data_ptr(), ops._stream(dz.device)))
    return gw


LAYERS = [(2, c1, c2, co, p) for _, p, c1, c2, co in T.fusion_mlp_schedule()]


@pytest.mark.parametrize("B,C1,C2,Co,P,centred",
                         [pytest.param(*c, False, id="-".join(map(str, c))) for c in LAYERS + WGRAD_CASES]
                         + [pytest.param(*c, True, id="-".join(map(str, c)) + "-centred") for c in WGRAD_CENTRED])
def test_wgrad_det_vs_float64(cuda, B, C1, C2, Co, P, centred):
    g = torch.Generator(device=cuda).manual_seed(P + Co)
    dz = torch.randn(B, Co, P, generator=g, device=cuda)
    x1 = torch.randn(B, C1, P, generator=g, device=cuda)
    x2 = torch.randn(B, C2, P, generator=g, device=cuda) if C2 else None
    if centred:
        dz = (dz.double() - dz.double().mean(dim=(0, 2), keepdim=True)).float()
        x1 += 4
        if C2:
            x2 += 4
    gw = wgrad_det(dz, x1, x2, B, Co, P)
    assert torch.equal(gw, wgrad_det(dz, x1, x2, B, Co, P)), "not bitwise repeatable"
    x = torch.cat((x1, x2), 1) if C2 else x1
    want = sum(dz[b].double() @ x[b].double().t() for b in range(B))
    ref32 = torch.einsum("bop,bcp->oc", dz, x)
    close_fp32(gw, want, ref32, "wgrad_det" + " centred" * centred, factor=8 if centred else 4)


# ------------------------------------------------------------------ graph replay
def test_deterministic_paths_replay_bitwise_in_cuda_graph(cuda):
    ind = step_indices(cuda)
    gen = torch.Generator(device=cuda).manual_seed(11)
    idx_rs = ind["r2p_up_nei_idx2"].contiguous()           # K = 16 gather + max
    B, Q, K = idx_rs.shape
    S = T.set_size(("img", 2))
    f3 = torch.randn((B, 64, S), generator=gen, device=cuda)
    g_rs = torch.randn((B, 64, Q), generator=gen, device=cuda)
    idx_ch = ind["choose"].reshape(B, -1).contiguous()
    g_ch = torch.randn((B, 64, idx_ch.shape[1]), generator=gen, device=cuda)
    idx_nb = ind["cld_nei_idx0"].contiguous()
    g_nb = torch.randn(tuple(idx_nb.shape) + (8,), generator=gen, device=cuda)
    dz = torch.randn((B, 64, 19200), generator=gen, device=cuda)
    x1 = torch.randn((B, 64, 19200), generator=gen, device=cuda)
    dz_s = torch.randn((B, 32, 49152), generator=gen, device=cuda)
    x_s = torch.randn((B, 16, 49152), generator=gen, device=cuda)

    def work():
        gf = torch.empty((B, 64, S), device=cuda)
        ops._gather_max_bwd_det(f3, idx_rs, g_rs, LAYOUT_NCS, gf)
        ch = ops.segment_sum(g_ch, None, T.set_size(("img", 1)), plan=ops.segment_csr(idx_ch, T.set_size(("img", 1))))
        n = idx_nb.shape[1]
        nbytes = int(lib.ffb6d_gather_neighbour_bwd_det_workspace_bytes(B, n, n, 16))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=cuda)
        gpc = torch.empty((B, n, 8), device=cuda)
        check(lib.ffb6d_gather_neighbour_bwd_det(g_nb.data_ptr(), idx_nb.data_ptr(), int(idx_nb.dtype == torch.int64), B, n, 8, n, 16, ws.data_ptr(), nbytes,
                                                 gpc.data_ptr(), ops._stream(cuda)))
        return [gf, ch, gpc, wgrad_det(dz, x1, None, B, 64, 19200), wgrad_det(dz_s, x_s, None, B, 32, 49152)]

    first = work()
    again = work()
    for a, b in zip(first, again):
        assert torch.equal(a, b)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        work()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = work()
    for _ in range(2):
        for o in outs:
            o.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        for o, f in zip(outs, first):
            assert torch.equal(o, f)


# ------------------------------------------------------------------ the switch, on the whole network
ATOMIC = {"gather_max_bwd_kernel", "gather1_bwd_runs_kernel", "gather_neighbour_bwd_kernel", "fusion_wgrad_kernel",
          "wgrad_small_kernel"}
DET_GATHER = {"csr_count_kernel", "csr_tile_sum_kernel", "csr_tile_scan_kernel", "csr_offsets_kernel", "csr_place_kernel",
              "csr_sort_short_kernel", "csr_sort_long_kernel", "segment_sum_masked_kernel", "gather_argmax_kernel"}
DET_WGRAD = {"fusion_wgrad_det_kernel", "wgrad_small_det_kernel", "wgrad_split_reduce_kernel"}
_small = {}


def small_setup(cuda):
    """test_gpu_model's shapes: B = 2, 120x160, 4096 points; its seeded model, inputs and image features."""
    if not _small:
        B, h, w, n_pts = 2, 120, 160, 4096
        torch.manual_seed(3)
        model = FFB6DFusionNet(n_classes=5, n_pts=n_pts, n_kps=8).to(cuda)
        g = torch.Generator().manual_seed(9)
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
                    m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                    m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                    m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                    m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
        batch = make_batch([3, 4], n_points=n_pts, h=h, w=w)
        inputs = build_ffb6d_indices(torch.from_numpy(batch["cld"]).to(cuda), torch.from_numpy(batch["dpt_xyz"]).to(cuda))
        inputs["choose"] = torch.from_numpy(batch["choose"]).to(cuda)
        inputs["cld_rgb_nrm"] = torch.from_numpy(batch["cld_rgb_nrm"]).to(cuda)
        gg = torch.Generator(device=cuda).manual_seed(1)
        rgb = [torch.randn(s, generator=gg, device=cuda) for s in FFB6DFusionNet.rgb_feature_shapes(B, h, w)]
        _small.update(sd={k: v.clone() for k, v in model.state_dict().items()}, inputs=inputs, rgb=rgb,
                      go_state=gg.get_state())
    return _small


def upstream_gradients(cuda, s, outs):
    """The output gradients test_gpu_model.py draws: the same generator, continued after the image features."""
    gg = torch.Generator(device=cuda)
    gg.set_state(s["go_state"])
    return [torch.randn(v.shape, generator=gg, device=cuda) for v in outs]


def flat(d):
    return [d[k] for k in ("pred_rgbd_segs", "pred_kp_ofs", "pred_ctr_ofs")] + list(d["fused_rgb"])


def make_model(cuda, sd, restructured):
    model = FFB6DFusionNet(n_classes=5, n_pts=4096, n_kps=8, restructured=restructured).to(cuda)
    model.load_state_dict(sd)
    return model.train()


def step(model, inputs, rgb, go):
    out = model(inputs, rgb)
    sum((v * g).sum() for v, g in zip(flat(out), go)).backward()


def kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = set()
    for ev in prof.events():
        if ev.device_type is not None and "cuda" in str(ev.device_type).lower():
            n = re.sub(r"\(.*", "", ev.name).replace("void ", "").replace("ffb6d::", "")
            names.add(re.sub(r"<.*", "", n))
    return names


@pytest.mark.parametrize("setting", ["algorithms", "cudnn", "neither"])
def test_switch_selects_backward_kernels(cuda, setting):
    s = small_setup(cuda)
    model = make_model(cuda, s["sd"], False)
    rgb = [t.clone().requires_grad_(True) for t in s["rgb"]]
    with torch.no_grad():
        go = [torch.randn_like(v) for v in flat(model(s["inputs"], rgb))]
    with switches(algorithms=setting == "algorithms", cudnn=setting == "cudnn"):
        names = kernel_names(lambda: step(model, s["inputs"], rgb, go))
    if setting == "algorithms":
        assert not names & ATOMIC, names & ATOMIC
        assert {"fusion_wgrad_det_kernel", "wgrad_small_det_kernel", "gather_argmax_kernel",
                "segment_sum_masked_kernel", "csr_place_kernel"} <= names
    elif setting == "cudnn":
        assert DET_WGRAD <= names and not names & {"fusion_wgrad_kernel", "wgrad_small_kernel"}
        assert {"gather_max_bwd_kernel", "gather1_bwd_runs_kernel"} <= names and not names & DET_GATHER
    else:
        assert ATOMIC - {"gather_neighbour_bwd_kernel"} <= names
        assert not names & (DET_GATHER | DET_WGRAD), names & (DET_GATHER | DET_WGRAD)


def train_run(cuda, s, restructured, go):
    """Under torch.use_deterministic_algorithms(True): one forward + backward (gradients, running statistics), then
    Adam steps to three in all."""
    model = make_model(cuda, s["sd"], restructured)
    rgb = [t.clone().requires_grad_(True) for t in s["rgb"]]
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    with switches(algorithms=True):
        step(model, s["inputs"], rgb, go)
        grads = {n: p.grad.clone() for n, p in model.named_parameters()}
        rgb_grads = [t.grad.clone() for t in rgb]
        stats = {n: b.clone() for n, b in model.named_buffers()}
        for i in range(3):
            if i:
                opt.zero_grad(set_to_none=True)
                step(model, s["inputs"], rgb, go)
            opt.step()
    params = {n: p.detach().clone() for n, p in model.named_parameters()}
    return grads, rgb_grads, stats, params


@pytest.mark.parametrize("restructured", [False, True], ids=["reference_order", "restructured"])
def test_whole_network_bitwise_reproducible(cuda, restructured):
    s = small_setup(cuda)
    with torch.no_grad():
        go = upstream_gradients(cuda, s, flat(make_model(cuda, s["sd"], restructured)(s["inputs"], s["rgb"])))
    a, b = train_run(cuda, s, restructured, go), train_run(cuda, s, restructured, go)
    for what, x, y in (("grad", a[0], b[0]), ("running statistics", a[2], b[2]), ("parameters after Adam", a[3], b[3])):
        for n in x:
            assert torch.equal(x[n], y[n]), "%s of %s differs between two runs" % (what, n)
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        assert torch.equal(x, y), "gradient of rgb_feats[%d] differs between two runs" % i
    # and the gradients meet tests/test_gpu_model.py's bounds against its float64 restatement
    ref = test_gpu_model.TorchRef(s["sd"], True, 8)
    ref32 = test_gpu_model.TorchRef(s["sd"], True, 8, dtype=torch.float32)
    rgb64 = [t.double().requires_grad_(True) for t in s["rgb"]]
    rgb32 = [t.clone().requires_grad_(True) for t in s["rgb"]]
    sum((v * g.double()).sum() for v, g in zip(flat(ref.forward(s["inputs"], rgb64)), go)).backward()
    sum((v * g).sum() for v, g in zip(flat(ref32.forward(s["inputs"], rgb32)), go)).backward()

    def unit(name):
        return name.rsplit(".conv.", 1)[0].rsplit(".normlayer.", 1)[0].rsplit(".bn.bn.", 1)[0].rsplit(".fc.", 1)[0]

    scale = {}
    for name in a[0]:
        scale[unit(name)] = max(scale.get(unit(name), 1e-12), ref.p[name].grad.norm().item())
    for name, gr in a[0].items():
        r, r32 = ref.p[name].grad, ref32.p[name].grad
        e_ours = (gr.double() - r).norm().item() / scale[unit(name)]
        e_t32 = (r32.double() - r).norm().item() / scale[unit(name)]
        assert e_ours <= max(4 * e_t32, 2e-3), "grad %s: error %.3e of its layer's scale (torch fp32 %.3e)" % (name, e_ours, e_t32)
    for gr, r, r32 in zip(a[1], rgb64, rgb32):
        if r.grad is not None:
            nrm = max(r.grad.norm().item(), 1e-12)
            e_ours = (gr.double() - r.grad).norm().item() / nrm
            e_t32 = (r32.grad.double() - r.grad).norm().item() / nrm
            assert e_ours <= max(4 * e_t32, 2e-3), (e_ours, e_t32)
