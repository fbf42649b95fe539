"""GPU: kernel entry points at the size limits their argument checks admit, against plain restatements.

The other suites pin every kernel at FFB6D's own shapes (480x640 frames, B <= 32, <= 1024 channels, 12288 points).
The C ABI admits far more, and between those shapes and its limits lie the usual ways a kernel goes wrong: a grid
dimension past 65535, a 32-bit loop counter or a flat offset past 2^31.  Each case below makes the dimensions it does
not test degenerate so that it stays cheap, fills every output with a NaN sentinel first, and compares with a
float64 (or exact) restatement of the operation at the first and last element, +-64 elements around flat index 2^31
and the last frame, channel and query, and over the whole output where that is cheap.

LIMITS is the table: one row per entry point that launches a kernel, with the limits its FFB6D_CHECK_ARG lines
admit, the kernel each case takes, and the test that covers it (or why there is none).  Cases that need more than
about 20 GB are not run; the cases that need several GB read torch.cuda.mem_get_info() first and skip, with the
reason, when that much is not free.
"""
import gc
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F_

from test_gpu_deterministic import check_atomic_sum, check_sum
from test_gpu_train import away_from_kink, bn_split_plan, close_elementwise, close_fp32
from ffb6d_b200 import augment as A
from ffb6d_b200._lib import lib, check, ERR_INVALID, LAYOUT_NCS, LAYOUT_NSC, MAX_K, last_error
from ffb6d_b200.ops import _stream
from oracle import aug_oracle as O

pytestmark = pytest.mark.gpu

GiB = 1 << 30
FLAT = 1 << 31
#  entry point: (limits its checks admit; kernel(s) and case(s), or why there is none)
LIMITS = {
    # gather.cu
    "ffb6d_gather_max_fwd": (
        "B < 65536, C <= 65535*8, S, Q < 2^31, 1 <= K <= 64",
        "staged, staged_v4, K=1 direct, generic direct, K-lane, NSC: test_gather_max_fwd_at_limits (B = 65535, "
        "C = 524280, K = 64, B*C*S > 2^31; staged shapes with more than 65535 channel chunks take the direct / K-lane "
        "kernels, the generic direct one at C = 524280 with grid.y = 65535).  NSC: the check admits "
        "B*Q <= 8*(2^31 - 1), what grid.x holds; test_abi.py asserts the rejection above it"),
    "ffb6d_gather_max_bwd": (
        "B, C, S, Q >= 0, 1 <= K <= 64",
        "gather1_bwd_runs_kernel, gather_max_bwd_kernel: test_gather_max_bwd_at_limits (B = 65535; B*C*S > 2^31)"),
    "ffb6d_gather_max_bwd_det": (
        "as the atomic one, ceil(C/32) <= 65535 for the sum",
        "csr_* + segment_sum_masked_kernel: test_gather_max_bwd_at_limits"),
    "ffb6d_gather_neighbour_fwd": (
        "S, D < 2^31; B, N, K >= 0",
        "gather_neighbour_kernel: test_gather_neighbour_past_2_31 (B*N*K*D > 2^31)"),
    "ffb6d_gather_neighbour_bwd": (
        "B, S, D, N, K >= 0",
        "gather_neighbour_bwd_kernel (fp64 atomics): test_gather_neighbour_past_2_31"),
    "ffb6d_gather_neighbour_bwd_det": (
        "ceil(D/32) <= 65535",
        "csr_* + segment_sum_kernel: test_gather_neighbour_past_2_31"),
    "ffb6d_relative_pos_encoding_fwd": (
        "B, N, K >= 0 (no upper bound; N >= 2^31 would need an 86 GB output)",
        "rel_pos_enc_kernel: test_rel_pos_enc_past_2_31 (B*N*K*10 > 2^31)"),
    "ffb6d_relative_pos_encoding_cm_fwd": (
        "B, N, K >= 0", "rel_pos_enc_cm_kernel: test_rel_pos_enc_past_2_31"),
    "ffb6d_att_pool_fwd": (
        "C1 >= 1, C2 >= 0, 1 <= K <= 64",
        "att_pool_kernel<16>, <0>: test_att_pool_at_limits (B = 65535; B*C*N*K > 2^31 for K = 16)"),
    "ffb6d_att_pool_bwd": (
        "C1 >= 1, C2 >= 0, 1 <= K <= 64",
        "att_pool_bwd_kernel<16>, <0>: test_att_pool_at_limits (B = 65535).  Past 2^31 it needs three 8.6 GB "
        "arrays (26 GB), not run"),
    # train.cu
    "ffb6d_bn_train_fwd": (
        "B < 65536, C <= 65535, P < 2^31, B*C < 2^31",
        "bn_stats/finalize/apply_kernel: test_bn_train_at_limits (B = 65535, C = 65535, P = 2^31 - 1 and 2^31 - 4).  "
        "B*C near 2^31 needs 17 GB plus a float64 reference of the same size, not run"),
    "ffb6d_bn_train_bwd": ("as bn_train_fwd", "bn_bwd_reduce/finalize/apply_kernel: test_bn_train_at_limits"),
    "ffb6d_bn_sync_moments": ("as bn_train_fwd", "bn_stats/moments_kernel: test_bn_sync_b65535_w65536"),
    "ffb6d_bn_sync_fwd": ("as bn_train_fwd, 1 <= W <= 65536",
                          "bn_sync_finalize/apply_kernel: test_bn_sync_b65535_w65536 (W = 65536 rows)"),
    "ffb6d_bn_sync_bwd_sums": ("as bn_train_fwd", "bn_bwd_reduce/sync_bwd_local_kernel: test_bn_sync_b65535_w65536"),
    "ffb6d_bn_sync_bwd": ("as bn_train_fwd, 1 <= W <= 65536",
                          "bn_sync_bwd_combine/bwd_apply_kernel: test_bn_sync_b65535_w65536 (W = 65536 rows)"),
    "ffb6d_act_bwd": (
        "n >= 0", "act_bwd_kernel: test_act_bwd_past_2_31 (n > 2^31; n > 2^32 needs 34 GB, not run)"),
    # psp.cu
    "ffb6d_log_softmax_bwd": (
        "B < 65536, C < 2^31, P < 2^38, C*P < 2^50",
        "log_softmax_bwd_kernel: test_log_softmax_bwd_at_limits (B = 65535; C*P > 2^31)"),
    "ffb6d_upsample_bilinear2d_bwd": (
        "every size < 2^24, B*C < 2^40, B*C*Hi*Wi and B*C*Ho*Wo < 2^50",
        "upsample_bilinear_ac_bwd_kernel: test_upsample_bilinear2d_bwd_past_2_31 (B*C*Ho*Wo > 2^31)"),
    "ffb6d_psp_pool": ("H <= 1024, W < 2^24, B*C < 2^31, B*C*50 < 2^40, H*W < 2^31",
                       "psp_pool_kernel: test_psp_pool_b65535"),
    "ffb6d_psp_pool_bwd": ("H <= 1024, W <= 16384, B*C < 2^31, B*C*50 < 2^40, H*W < 2^31", "not covered here"),
    "ffb6d_psp_bottleneck_fwd": (
        "B < 65536, Co <= 65535*128, C < 2^31, H + W <= 3072, H*W < 2^31, B*50*Co < 2^31", "not covered here"),
    "ffb6d_psp_bottleneck_bwd": ("H, W <= 1024, the shared-memory bound, B*Co < 2^31, B*50*Co < 2^40",
                                 "not covered here"),
    # augment.cu
    "ffb6d_rgb_add_noise": (
        "B < 65536, 32 <= H <= 65535*8, 32 <= W < 2^20, H*W*3 < 2^31",
        "hsv/filter/gauss/noise_kernel: test_rgb_add_noise_at_limits (H = 524280 at W = 32, B = 65535; "
        "H = 600000 is rejected before any launch)"),
    "ffb6d_add_real_back": ("as rgb_add_noise, back_label_channels 1 or 3", "not covered here"),
    "ffb6d_aug_noise_field": ("as rgb_add_noise, 0 <= stage < 4", "not covered here"),
    "ffb6d_color_jitter": ("1 <= B < 65536, 1 <= H, W < 2^20, H*W*3 < 2^31",
                           "jitter_sum/apply_kernel: test_color_jitter_b65535"),
    # segment_sum.cu
    "ffb6d_segment_plan / ffb6d_segment_sum": (
        "1 <= B < 65536, 1 <= P, NA < 2^31, plan ints per frame < 2^31; ceil(C/32) <= 65535",
        "segment_count/scan/place + segment_sum_kernel: test_segment_sum_at_limits (B = 65535; C = 65535*32)"),
    "ffb6d_segment_csr / ffb6d_segment_sum_csr": (
        "1 <= B < 65536, 1 <= P, NA < 2^31, CSR bytes per frame < 2^31; ceil(C/32) <= 65535",
        "csr_* + segment_sum_kernel: test_segment_sum_at_limits"),
    # fusion_mlp.cu
    "ffb6d_fusion_mlp_fwd_ex / _fwd_packed": (
        "B < 65536, 1 <= Co <= 65535*128, P < 2^31, C1 + C2 < 2^31; NA < 2^31 with an addend",
        "the wgmma layer: test_fusion_mlp_fwd_ex_at_limits (Co = 65535*128; B*Co*P > 2^31)"),
    "ffb6d_fusion_mlp_wgrad / _wgrad_det": (
        "B < 65536, Co <= 65535*128, C1 + C2 <= 65535*128, P < 2^31, B*P < 2^31", "not covered here"),
    "ffb6d_conv1x1_log_softmax_fwd": ("B < 65536, 1 <= Co <= 128, Ci, P < 2^31", "not covered here"),
    # the rest
    "ffb6d_focal_loss_* / ffb6d_of_l1_loss_*": (
        "1 <= B < 65536, 1 <= N < 2^31 - 128, C <= 256, B*C*N < 2^40, n_kps <= 32", "not covered here"),
    "ffb6d_point_item": ("0 <= B < 65536, H*W < 2^31, 0 <= N < 2^31, n_kps <= 32, n_obj <= 256",
                         "not covered here"),
    "ffb6d_backproject": ("0 <= B < 65536, H, W >= 8, H*W < 2^31", "not covered here"),
    "ffb6d_sample_pixels": ("0 <= B < 65536, H*W < 2^30, N < 2^30", "not covered here"),
    "ffb6d_fill_depth": ("depth_fill.cu size_ok: H <= 65535*8", "not covered here"),
    "ffb6d_lfa_att_pool_fused": ("B < 65536, N < 2^31, K = 16, Dh in {16, 32, 64}, Do <= 2 Dh", "not covered here"),
    "ffb6d_mean_shift_fit": ("G <= 64, N < 2^24", "not covered here"),
    "ffb6d_best_fit_transform": ("1 <= M <= 4096", "not covered here"),
    "ffb6d_knn_batch / _grid_build / _grid_query": ("B < 65536, S, Q < 2^31",
                                                    "grid and brute-force searches: test_knn_b65535"),
    "ffb6d_build_indices": ("B < 65536, N0 a multiple of 256, H, W multiples of 8", "not covered here"),
}

PEAK = {}


@pytest.fixture(autouse=True)
def _free_between_cases(request):
    """Every case starts with the allocator empty and records its peak allocation and wall time."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    PEAK[request.node.name] = (torch.cuda.max_memory_allocated() / GiB, time.perf_counter() - t0)
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.perf_counter()
    yield
    if PEAK:
        name, (gb, sec) = max(PEAK.items(), key=lambda kv: kv[1][0])
        print("\nsize limits: %d cases in %.1f s; largest peak allocation %.2f GB (%s, %.1f s)"
              % (len(PEAK), time.perf_counter() - t0, gb, name, sec))


def need(gb):
    free, _ = torch.cuda.mem_get_info()
    if free < gb * GiB:
        pytest.skip("needs %.1f GB of device memory, %.1f GB free" % (gb, free / GiB))


def sentinel(*shape, dtype=torch.float32, dev="cuda"):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def all_written(x):
    """No NaN sentinel left anywhere in x (scanned in slices, without a bool copy of the whole array)."""
    return not any(bool(c.isnan().any()) for c in x.reshape(-1).split(1 << 28))


def flat_samples(n, *extra):
    """Flat indices: the first and last 64 and +-64 around 2^31 and 2^32 where the array reaches them, plus
    ``extra`` ones, in range."""
    s = [np.arange(0, 64), np.arange(n - 64, n)]
    for at in (1 << 31, 1 << 32):
        if at - 64 < n:
            s.append(np.arange(at - 64, at + 64))
    s.extend(np.atleast_1d(e) for e in extra)
    s = np.unique(np.concatenate(s))
    return torch.from_numpy(s[(s >= 0) & (s < n)])


def test_limits_table_names_exported_entry_points():
    for name in LIMITS:
        for sym in name.split(" / "):
            if "*" not in sym and sym.startswith("ffb6d_"):
                assert hasattr(lib, sym), sym


# ------------------------------------------------------------------ gather + max forward
# (B, C, S, Q, K, layout, kernel, GB needed)
FWD = {
    "staged_k16_b65535": (65535, 1, 64, 4, 16, "ncs", "gather_max_ncs_staged_kernel", 0.1),
    "staged_v4_k1_b65535": (65535, 2, 16, 4, 1, "ncs", "gather1_ncs_staged_v4_kernel", 0.1),
    "staged_k1_q3_b65535": (65535, 2, 16, 3, 1, "ncs", "gather_max_ncs_staged_kernel", 0.1),
    "staged_k64_widest_c": (1, 524280, 8, 4, 64, "ncs", "gather_max_ncs_staged_kernel", 1.0),
    "staged_v4_k1_widest_c": (1, 524280, 8, 4, 1, "ncs", "gather1_ncs_staged_v4_kernel", 0.2),   # grid.y = 65535
    "klane_k16_b65535": (65535, 1, 41, 1, 16, "ncs", "gather_max_ncs_klane_kernel", 0.1),
    "klane_k32_widest_c": (1, 524280, 41, 1, 32, "ncs", "gather_max_ncs_klane_kernel", 0.3),     # grid.y = 65535
    "direct_k64_long_rows": (2, 8, 28929, 4, 64, "ncs", "gather_max_ncs_direct_kernel", 0.1),
    "direct_k5_b65535": (65535, 1, 28929, 1, 5, "ncs", "gather_max_ncs_direct_kernel", 8.0),
    # rows that stage one channel per CTA: 65536 chunks do not fit grid.y, the direct / K-lane kernels take them
    "staged_k16_wide_c_falls_back": (1, 65536, 14465, 362, 16, "ncs", "gather_max_ncs_klane_kernel", 4.5),
    "staged_k1_wide_c_falls_back": (1, 65536, 14465, 4, 1, "ncs", "gather1_ncs_direct_kernel", 4.5),
    "staged_k64_wide_c_falls_back": (1, 65536, 14465, 2, 64, "ncs", "gather_max_ncs_direct_kernel", 4.5),
    # 7 channels per staged CTA (S > 3616) would need 74897 chunks: the generic direct kernel at the widest C
    "direct_k5_widest_c": (1, 524280, 3617, 4, 5, "ncs", "gather_max_ncs_direct_kernel", 8.0),
    # the `choose` gather with B*C*S > 2^31
    "direct_k1_flat_past_2_31": (1, 74241, 28929, 4, 1, "ncs", "gather1_ncs_direct_kernel", 9.5),
    "nsc_k64_b65535": (65535, 4, 2, 1, 64, "nsc", "gather_max_nsc_kernel", 0.1),
    "nsc_odd_c_widest": (1, 524279, 2, 2, 3, "nsc", "gather_max_nsc_kernel", 0.1),
}


def gather_want(f3, idx):
    """out[b, c, q] = max_k f3[b, c, idx[b, q, k]], exactly (the features hold no NaN and no ties matter)."""
    B, Cc, _ = f3.shape
    Q, K = idx.shape[1], idx.shape[2]
    vals = f3.gather(2, idx.long().reshape(B, 1, Q * K).expand(B, Cc, Q * K))
    return vals.reshape(B, Cc, Q, K).amax(-1)


def make_idx(gen, B, S, Q, K, dev):
    idx = torch.randint(0, S, (B, Q, K), generator=gen, device=dev, dtype=torch.int32)
    idx[-1, -1, -1] = S - 1                              # the last element of the last row is read
    idx[0, 0, 0] = 0
    return idx


@pytest.mark.parametrize("case", list(FWD))
def test_gather_max_fwd_at_limits(cuda, case):
    B, C, S, Q, K, layout, kernel, gb = FWD[case]
    need(gb)
    lay = LAYOUT_NCS if layout == "ncs" else LAYOUT_NSC
    assert lib.ffb6d_gather_kernel_name(B, C, S, Q, K, lay).decode() == kernel
    g = torch.Generator(device=cuda).manual_seed(B + 7 * C + 13 * S + Q + K)
    store = torch.randn((B, C, S) if layout == "ncs" else (B, S, C), generator=g, device=cuda)
    f3 = store if layout == "ncs" else store.transpose(1, 2)
    idx = make_idx(g, B, S, Q, K, cuda)
    out = sentinel(*((B, C, Q) if layout == "ncs" else (B, Q, C)))
    check(lib.ffb6d_gather_max_fwd(store.data_ptr(), idx.data_ptr(), 0, B, C, S, Q, K, lay, out.data_ptr(),
                                   _stream(cuda)))
    got = out if layout == "ncs" else out.transpose(1, 2)
    assert torch.equal(got, gather_want(f3, idx)), case


# ------------------------------------------------------------------ gather + max backward
def bwd_pair(f3, idx, gout, K):
    """grad_feat by the atomic and by the deterministic entry point (NCS)."""
    B, C, S = f3.shape
    Q = idx.shape[1]
    dev = f3.device
    atomic = sentinel(B, C, S)
    check(lib.ffb6d_gather_max_bwd(f3.data_ptr(), idx.data_ptr(), 0, gout.data_ptr(), B, C, S, Q, K, LAYOUT_NCS,
                                   atomic.data_ptr(), _stream(dev)))
    nb = int(lib.ffb6d_gather_max_bwd_det_workspace_bytes(B, C, S, Q, K))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    det = sentinel(B, C, S)
    check(lib.ffb6d_gather_max_bwd_det(f3.data_ptr(), idx.data_ptr(), 0, gout.data_ptr(), B, C, S, Q, K, LAYOUT_NCS,
                                       ws.data_ptr(), nb, det.data_ptr(), _stream(dev)))
    return atomic, det


@pytest.mark.parametrize("B,C,S,Q,K", [(65535, 2, 64, 4, 16), (65535, 2, 16, 4, 1), (65535, 1, 3, 2, MAX_K)],
                         ids=["k16_b65535", "k1_b65535", "k64_b65535"])
def test_gather_max_bwd_at_limits(cuda, B, C, S, Q, K):
    from test_gpu_deterministic import want_gather_bwd
    g = torch.Generator(device=cuda).manual_seed(B + C + S + Q + K)
    f3 = torch.randn(B, C, S, generator=g, device=cuda)
    idx = make_idx(g, B, S, Q, K, cuda)
    gout = torch.randn(B, C, Q, generator=g, device=cuda)
    want, mag, cnt = want_gather_bwd(f3.double(), idx, gout)
    atomic, det = bwd_pair(f3, idx, gout, K)
    check_atomic_sum(atomic, want, mag, cnt, "gather_max_bwd")
    check_sum(det, want, mag, "gather_max_bwd_det")


def test_gather_k1_bwd_flat_past_2_31(cuda):
    """The `choose` gather's backward with B*C*S > 2^31 (C > 65535: the generic atomic kernel), checked over the
    channels on both sides of flat index 2^31 and the last, and for no gradient elsewhere.  (The deterministic backward's
    workspace would add 17 GB here; it is run at B = 65535 above.)"""
    B, C, S, Q = 1, 74241, 28929, 4
    assert C * S > FLAT
    need(18.0)
    g = torch.Generator(device=cuda).manual_seed(5)
    f3 = torch.empty(B, C, S, device=cuda)               # K = 1: the arg-max is the one neighbour, whatever f3 holds
    idx = torch.tensor([[[0], [S - 1], [FLAT % S], [FLAT % S]]], dtype=torch.int32, device=cuda)
    gout = torch.randn(B, C, Q, generator=g, device=cuda)
    atomic = sentinel(B, C, S)
    check(lib.ffb6d_gather_max_bwd(f3.data_ptr(), idx.data_ptr(), 0, gout.data_ptr(), B, C, S, Q, 1, LAYOUT_NCS,
                                   atomic.data_ptr(), _stream(cuda)))
    del f3
    cols = idx.long().reshape(Q)
    nonzero = sum(int(torch.count_nonzero(c)) for c in atomic.reshape(-1).split(1 << 28))
    assert all_written(atomic) and nonzero <= C * 3
    ones = torch.ones(Q, dtype=torch.float64, device=cuda)
    for c in (0, FLAT // S - 1, FLAT // S, FLAT // S + 1, C - 1):
        zero = torch.zeros(S, dtype=torch.float64, device=cuda)
        want = zero.clone().index_add_(0, cols, gout[0, c].double())
        mag = zero.clone().index_add_(0, cols, gout[0, c].double().abs())
        cnt = zero.clone().index_add_(0, cols, ones)
        check_atomic_sum(atomic[0, c], want, mag, cnt, "channel %d" % c)


# ------------------------------------------------------------------ neighbour gather, relative position encoding
def test_gather_neighbour_past_2_31(cuda):
    B, S, D, K = 2, 16, 8, 16
    N = -(-(FLAT + 1024) // (B * K * D))
    n_out = B * N * K * D
    assert n_out > FLAT
    need(n_out * 4 / GiB + 4.0)
    g = torch.Generator(device=cuda).manual_seed(7)
    pc = torch.randn(B, S, D, generator=g, device=cuda)
    idx = torch.randint(0, S, (B, N, K), generator=g, device=cuda, dtype=torch.int32)
    out = sentinel(B, N, K, D)
    check(lib.ffb6d_gather_neighbour_fwd(pc.data_ptr(), idx.data_ptr(), 0, B, S, D, N, K, out.data_ptr(),
                                         _stream(cuda)))
    assert all_written(out), "gather_neighbour_fwd: output elements never written"
    t = flat_samples(n_out).to(cuda)
    row, j = t // D, t % D
    b = row // (N * K)
    want = pc[b, idx.reshape(-1)[row].long(), j]
    assert torch.equal(out.reshape(-1)[t], want), "gather_neighbour_fwd"
    # backward with grad_out = out: source point s of frame b receives count(b, s) * pc[b, s], exactly
    cnt = torch.stack([torch.bincount(idx[bb].reshape(-1).long(), minlength=S) for bb in range(B)])      # [B, S]
    want = (cnt.double()[..., None] * pc.double()).float()
    grad = sentinel(B, S, D)
    check(lib.ffb6d_gather_neighbour_bwd(out.data_ptr(), idx.data_ptr(), 0, B, S, D, N, K, grad.data_ptr(),
                                         _stream(cuda)))
    assert torch.equal(grad, want), "gather_neighbour_bwd"
    nb = int(lib.ffb6d_gather_neighbour_bwd_det_workspace_bytes(B, S, N, K))
    ws = torch.empty(nb, dtype=torch.uint8, device=cuda)
    grad.fill_(float("nan"))
    check(lib.ffb6d_gather_neighbour_bwd_det(out.data_ptr(), idx.data_ptr(), 0, B, S, D, N, K, ws.data_ptr(), nb,
                                             grad.data_ptr(), _stream(cuda)))
    assert torch.equal(grad, want), "gather_neighbour_bwd_det"


def f32(x):
    return x.float().double()


def rel_pos_want(xyz, idx_flat, rows, N, K):
    """The ten channels at flat rows (b*N + n)*K + k, restated in float64 and rounded to float32 after every
    operation (products and sums of two floats and a square root are then rounded exactly as in fp32)."""
    bn = rows // K
    b = bn // N
    j = idx_flat[rows].long()
    c = xyz.reshape(-1, 3)[bn].double()
    nb = xyz.reshape(-1, 3)[b * N + j].double()
    d = f32(c - nb)
    ss = f32(f32(f32(d[:, 0] * d[:, 0]) + f32(d[:, 1] * d[:, 1])) + f32(d[:, 2] * d[:, 2]))
    return torch.cat([f32(ss.sqrt())[:, None], d, c, nb], 1).float()               # [len(rows), 10]


@pytest.mark.parametrize("cm", [False, True], ids=["nk10", "channel_major"])
def test_rel_pos_enc_past_2_31(cuda, cm):
    B, K = 1, 64
    N = -(-(FLAT + 512) // (10 * K))
    rows_total = B * N * K
    assert rows_total * 10 > FLAT
    need(rows_total * 44 / GiB + 0.5)
    g = torch.Generator(device=cuda).manual_seed(11)
    xyz = torch.randn(B, N, 3, generator=g, device=cuda)
    idx = torch.randint(0, N, (B, N, K), generator=g, device=cuda, dtype=torch.int32)
    idx[-1, -1, -1] = N - 1
    out = sentinel(rows_total * 10)
    fn = lib.ffb6d_relative_pos_encoding_cm_fwd if cm else lib.ffb6d_relative_pos_encoding_fwd
    check(fn(xyz.data_ptr(), idx.data_ptr(), 0, B, N, K, out.data_ptr(), _stream(cuda)))
    assert all_written(out), "output elements never written"
    plane = N * K
    # rows whose outputs lie around flat 2^31 in either layout, and the first and last rows
    rows = flat_samples(rows_total, np.arange(FLAT // 10 - 8, FLAT // 10 + 8),
                        np.arange(FLAT % plane - 64, FLAT % plane + 64)).to(cuda)
    want = rel_pos_want(xyz, idx.reshape(-1), rows, N, K)
    if cm:
        got = out.reshape(B, 10, plane)[0][:, rows].t()
    else:
        got = out.reshape(rows_total, 10)[rows]
    assert torch.equal(got, want)


# ------------------------------------------------------------------ attentive pooling
def att_pool_want(f, a):
    s = torch.softmax(a.double(), -1)
    return (f.double() * s).sum(-1), s


@pytest.mark.parametrize("K", [16, MAX_K])
def test_att_pool_at_limits(cuda, K):
    """B = 65535 forward and backward with two inputs; for K = 16, a forward whose f / att reach past flat 2^31."""
    B, C1, C2, N = 65535, 1, 2, 1
    g = torch.Generator(device=cuda).manual_seed(K)
    f1, f2 = torch.randn(B, C1, N, K, generator=g, device=cuda), torch.randn(B, C2, N, K, generator=g, device=cuda)
    att = torch.randn(B, C1 + C2, N, K, generator=g, device=cuda)
    gout = torch.randn(B, C1 + C2, N, generator=g, device=cuda)
    f = torch.cat([f1, f2], 1)
    want, s = att_pool_want(f, att)
    out = sentinel(B, C1 + C2, N)
    check(lib.ffb6d_att_pool_fwd(f1.data_ptr(), C1, f2.data_ptr(), C2, att.data_ptr(), B, N, K, out.data_ptr(),
                                 _stream(cuda)))
    close_fp32(out, want, None, "att_pool_fwd B=65535")
    gf1, gf2, gatt = sentinel(B, C1, N, K), sentinel(B, C2, N, K), sentinel(B, C1 + C2, N, K)
    check(lib.ffb6d_att_pool_bwd(f1.data_ptr(), C1, f2.data_ptr(), C2, att.data_ptr(), gout.data_ptr(), B, N, K,
                                 gf1.data_ptr(), gf2.data_ptr(), gatt.data_ptr(), _stream(cuda)))
    gg = gout.double()[..., None]
    close_fp32(torch.cat([gf1, gf2], 1), gg * s, None, "att_pool_bwd grad_f B=65535")
    close_fp32(gatt, s * gg * (f.double() - want[..., None]), None, "att_pool_bwd grad_att B=65535")
    if K != 16:
        return
    del f1, f2, att, gout, f, want, s, out, gf1, gf2, gatt
    torch.cuda.empty_cache()
    Nb = FLAT // K + 64                                   # f1 = att [1, 1, Nb, 16]: flat index past 2^31
    need(Nb * K * 4 / GiB + Nb * 4 / GiB + 0.5)
    x = torch.randn(1, 1, Nb, K, generator=g, device=cuda)
    out = sentinel(1, 1, Nb)
    check(lib.ffb6d_att_pool_fwd(x.data_ptr(), 1, None, 0, x.data_ptr(), 1, Nb, K, out.data_ptr(), _stream(cuda)))
    assert all_written(out), "att_pool_fwd: output elements never written"
    n = flat_samples(Nb, np.arange(FLAT // K - 8, FLAT // K + 8)).to(cuda)
    xs = x[0, 0, n]
    close_fp32(out[0, 0, n], att_pool_want(xs, xs)[0], None, "att_pool_fwd past 2^31")


# ------------------------------------------------------------------ training BatchNorm and activation backward
def test_act_bwd_past_2_31(cuda):
    n = FLAT + 4096
    need(2 * n * 4 / GiB + 0.5)
    g = torch.Generator(device=cuda).manual_seed(3)
    z = torch.randn(n, generator=g, device=cuda)          # also the upstream gradient
    dz = sentinel(n)
    check(lib.ffb6d_act_bwd(z.data_ptr(), z.data_ptr(), n, 2, 0.2, dz.data_ptr(), _stream(cuda)))
    assert all_written(dz), "act_bwd: output elements never written"
    t = flat_samples(n).to(cuda)
    zt = z[t]
    want = torch.where(zt > 0, zt, (zt.double() * float(np.float32(0.2))).float())
    assert torch.equal(dz[t], want)


def chunked_sums(fn, z, chunk=1 << 25):
    """Float64 sums of fn(z chunk) over a flat z, one chunk at a time."""
    acc = None
    for i in range(0, z.numel(), chunk):
        v = fn(z[i:i + chunk].double())
        acc = v if acc is None else [a + b for a, b in zip(acc, v)]
    return [float(a) for a in acc]


def bn_run(cuda, z, B, C, P, gamma, beta, rm, rv, act, slope, eps, momentum):
    nb = int(lib.ffb6d_bn_workspace_bytes(C, P))
    ws = torch.empty(nb, dtype=torch.uint8, device=cuda)
    stats = torch.empty(C, 4, device=cuda)
    y = sentinel(B, C, P)
    check(lib.ffb6d_bn_train_fwd(z.data_ptr(), B, C, P, gamma.data_ptr(), beta.data_ptr(), eps, momentum,
                                 rm.data_ptr(), rv.data_ptr(), act, slope, stats.data_ptr(), y.data_ptr(), ws.data_ptr(),
                                 nb, _stream(cuda)))
    return y, stats, ws, nb


@pytest.mark.parametrize("B,C,P", [(65535, 1, 5), (1, 65535, 5), (1, 1, FLAT - 1), (1, 1, FLAT - 4)],
                         ids=["b65535", "c65535", "p_2_31_minus_1_scalar", "p_2_31_minus_4_vec"])
def test_bn_train_at_limits(cuda, B, C, P):
    """Forward and backward of the batch-statistics BatchNorm with LeakyReLU.  At P near 2^31 the row loops run
    to within one stride of 2^31; the values are small integers, so the sums are exact in any order and the
    statistics are known exactly; the pre-activations stay 0.25 from the kink."""
    eps, momentum, act, slope = 1e-5, 0.1, 2, 0.2
    if P < 1024:
        g = torch.Generator(device=cuda).manual_seed(B + C)
        z = torch.randn(B, C, P, generator=g, device=cuda)
        gy = torch.randn(B, C, P, generator=g, device=cuda)
        gamma = 1 + 0.5 * torch.randn(C, generator=g, device=cuda)
        beta = 0.5 * torch.randn(C, generator=g, device=cuda)
        rm, rv = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
        z64 = z.double().requires_grad_(True)
        gam64, bet64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        rm64, rv64 = rm.double(), rv.double()
        pre64 = F_.batch_norm(z64, rm64, rv64, gam64, bet64, True, momentum, eps)
        y64 = F_.leaky_relu(pre64, slope)
        gy = away_from_kink(gy, pre64, act)
        gz64, gg64, gb64 = torch.autograd.grad(y64, (z64, gam64, bet64), gy.double())
        y, stats, ws, nb = bn_run(cuda, z, B, C, P, gamma, beta, rm, rv, act, slope, eps, momentum)
        # 1e-4: a thread sums up to B = 65535 values of a channel in fp32 (measured 1.2e-5 of scale on y)
        close_fp32(y, y64, None, "bn_train_fwd y", tol=1e-4)
        # the running statistics inherit the fp32 round-off of those sums: (B - 1) 2^-24 sum |terms| per thread
        n = B * P
        d = (z - z[:1, :, :1]).double()
        ma, mq = d.abs().sum((0, 2)) / n, (d * d).sum((0, 2)) / n
        off = (d.sum((0, 2)) / n).abs()
        ulps = (B - 1) * 2.0 ** -24
        close_fp32(rm, rm64, None, "running_mean", inherent=float((momentum * ulps * ma).max()), why="fp32 sums")
        close_fp32(rv, rv64, None, "running_var", inherent=float((momentum * ulps * (mq + 2 * off * ma) * n / (n - 1)).max()),
                   why="fp32 sums")
        dz, ggam, gbet = sentinel(B, C, P), sentinel(C), sentinel(C)
        check(lib.ffb6d_bn_train_bwd(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, C, P, act, slope,
                                     ggam.data_ptr(), gbet.data_ptr(), dz.data_ptr(), ws.data_ptr(), nb, _stream(cuda)))
        close_fp32(dz, gz64, None, "bn_train_bwd grad_z", tol=1e-4)
        close_fp32(ggam, gg64, None, "grad_gamma", tol=1e-4)
        close_fp32(gbet, gb64, None, "grad_beta", tol=1e-4)
        return
    n = B * C * P
    need(2 * n * 4 / GiB + 1.5)
    g = torch.Generator(device=cuda).manual_seed(P)
    z = torch.randint(-3, 4, (B, C, P), generator=g, device=cuda, dtype=torch.float32)   # also the upstream gradient
    gamma, beta = torch.ones(C, device=cuda), torch.full((C,), 0.25, device=cuda)
    rm, rv = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
    zc = [z[:, c].reshape(-1) for c in range(C)]
    sums = [chunked_sums(lambda v: (v.sum(), (v * v).sum()), zz) for zz in zc]
    m = B * P
    mean = torch.tensor([s[0] / m for s in sums], dtype=torch.float64, device=cuda)
    var = torch.tensor([s[1] / m for s in sums], dtype=torch.float64, device=cuda) - mean * mean
    invstd = 1 / (var + eps).sqrt()
    # the sums of the backward: g' = leaky'(pre) * z and g' * xhat
    bsum = []
    for c in range(C):
        mu, inv = float(mean[c]), float(invstd[c])

        def terms(v):
            xh = (v - mu) * inv
            gp = torch.where(xh + 0.25 > 0, v, v * slope)
            return gp.sum(), (gp * xh).sum(), gp.abs().sum(), (gp * xh).abs().sum()
        bsum.append(chunked_sums(terms, zc[c]))
    del zc

    y, stats, ws, nb = bn_run(cuda, z, B, C, P, gamma, beta, rm, rv, act, slope, eps, momentum)
    assert all_written(y), "bn_train_fwd: output elements never written"
    close_fp32(stats[:, 0], mean, None, "mean")
    close_fp32(stats[:, 1], invstd, None, "invstd")
    close_fp32(rm, momentum * mean, None, "running_mean")
    close_fp32(rv, (1 - momentum) + momentum * var * m / (m - 1), None, "running_var")
    t = flat_samples(P).to(cuda)
    for c in range(C):
        for b in (0, B - 1):
            pre = (z[b, c, t].double() - mean[c]) * invstd[c] + 0.25
            close_fp32(y[b, c, t], torch.where(pre > 0, pre, pre * slope), None, "y[%d, %d]" % (b, c))
    dz = y
    del y
    dz.fill_(float("nan"))
    ggam, gbet = sentinel(C), sentinel(C)
    check(lib.ffb6d_bn_train_bwd(z.data_ptr(), z.data_ptr(), stats.data_ptr(), B, C, P, act, slope, ggam.data_ptr(),
                                 gbet.data_ptr(), dz.data_ptr(), ws.data_ptr(), nb, _stream(cuda)))
    assert all_written(dz), "bn_train_bwd: output elements never written"
    # grad_beta / grad_gamma are fp32 sums of chunk/256 terms per thread (then fp64): within (terms - 1) 2^-24
    # sum |terms| of float64, plus the final rounding
    terms = bn_split_plan(C, P, torch.cuda.get_device_properties(cuda).multi_processor_count)[0] * B // 256
    for c in range(C):
        sb, sg, mag_b, mag_g = bsum[c]
        assert abs(float(gbet[c]) - sb) <= (terms - 1) * 2.0 ** -24 * mag_b + abs(sb) * 2.0 ** -23, ("grad_beta", c)
        assert abs(float(ggam[c]) - sg) <= (terms - 1) * 2.0 ** -24 * mag_g + abs(sg) * 2.0 ** -23, ("grad_gamma", c)
        for b in (0, B - 1):
            v = z[b, c, t].double()
            xh = (v - mean[c]) * invstd[c]
            gp = torch.where(xh + 0.25 > 0, v, v * slope)
            want = invstd[c] * (gp - sb / m - xh * sg / m)
            # the two sums' fp32 round-off above, carried through dz = invstd (g' - sum g' / m - xhat sum g' xhat / m)
            carried = float((invstd[c] * (terms - 1) * 2.0 ** -24 * (mag_b + xh.abs() * mag_g) / m).max())
            close_fp32(dz[b, c, t], want, None, "grad_z[%d, %d]" % (b, c), inherent=carried,
                       why="the fp32 per-thread sums' bound")


# ------------------------------------------------------------------ log_softmax backward
@pytest.mark.parametrize("B,C,P", [(65535, 3, 5), (1, 2, FLAT // 2 + 64)], ids=["b65535", "cp_past_2_31"])
def test_log_softmax_bwd_at_limits(cuda, B, C, P):
    n = B * C * P
    need(2 * n * 4 / GiB + 0.5)
    g = torch.Generator(device=cuda).manual_seed(C)
    out = -torch.rand(B, C, P, generator=g, device=cuda) * 3      # also the upstream gradient
    gin = sentinel(B, C, P)
    check(lib.ffb6d_log_softmax_bwd(out.data_ptr(), out.data_ptr(), B, C, P, gin.data_ptr(), _stream(cuda)))
    assert all_written(gin), "log_softmax_bwd: output elements never written"
    p = flat_samples(P, np.arange(FLAT - P - 64, FLAT - P + 64)).to(cuda)
    for b in {0, B - 1}:
        o = out[b][:, p].double()
        s = o.sum(0, keepdim=True)
        want = o - o.exp() * s
        close_elementwise(gin[b][:, p], want, 2.0 ** -21 * (o.abs() + o.exp() * o.abs().sum(0, keepdim=True)),
                          "log_softmax_bwd frame %d" % b)


# ------------------------------------------------------------------ augmentation
def filter_record(seed=0):
    """A YCB record with the HSV stage, the sharpen, a motion blur and the Gaussian blur on and the noise stages off."""
    rs = np.random.RandomState(seed)
    for _ in range(10000):
        r = A.draw_rgb_noise(rs, "ycb")
        if r[A.I_HSV] and r[A.I_SHARPEN] and r[A.I_MOTION_A] >= 3 and r[A.I_GAUSS_K]:
            r[A.I_NOISE] = r[A.I_FINAL] = 0
            return r
    raise AssertionError("no record with every filter stage")


def add_noise_call(cuda, rgb, plans, out, work):
    B, H, W, _ = rgb.shape
    dev_plan = torch.from_numpy(plans).to(cuda)
    return lib.ffb6d_rgb_add_noise(rgb.data_ptr(), B, H, W, plans.ctypes.data, dev_plan.data_ptr(), 1, None,
                                   out.data_ptr(), work.data_ptr(), _stream(cuda))


def test_rgb_add_noise_at_limits(cuda):
    """The tallest image the filters' grid takes (65535 tiles of 8 rows) at the narrowest W, checked against the
    numpy restatement on three windows (rows within the filters' reach of a window edge are not compared), and one
    row more, which is rejected before anything is written."""
    rec = filter_record()
    reach = 1 + int(rec[A.I_MOTION_A]) // 2 + int(rec[A.I_GAUSS_K]) // 2
    W = 32
    for H in (65535 * 8, 600000):
        g = torch.Generator(device=cuda).manual_seed(H)
        rgb = torch.randint(0, 256, (1, H, W, 3), generator=g, device=cuda, dtype=torch.uint8)
        out = torch.full_like(rgb, 0xAB)
        work = torch.empty_like(rgb)
        plans = rec[None].copy()
        rc = add_noise_call(cuda, rgb, plans, out, work)
        if H > 65535 * 8:
            assert rc == ERR_INVALID and "H <= 524280" in last_error()
            torch.cuda.synchronize()
            assert bool((out == 0xAB).all()), "rejected call wrote its output"
            continue
        check(rc)
        img = rgb[0].cpu().numpy()
        got = out[0].cpu().numpy()
        for lo, hi in ((0, 160), (H // 2 - 80, H // 2 + 80), (H - 160, H)):
            want = O.rgb_add_noise(img[lo:hi], rec)
            keep = slice(0 if lo == 0 else reach, (hi - lo) if hi == H else (hi - lo) - reach)
            assert np.array_equal(got[lo:hi][keep], want[keep]), (lo, hi)


def test_rgb_add_noise_b65535(cuda):
    B, H, W = 65535, 32, 32
    rec = filter_record(1)
    g = torch.Generator(device=cuda).manual_seed(B)
    rgb = torch.randint(0, 256, (B, H, W, 3), generator=g, device=cuda, dtype=torch.uint8)
    out, work = torch.full_like(rgb, 0xAB), torch.empty_like(rgb)
    check(add_noise_call(cuda, rgb, np.repeat(rec[None], B, 0), out, work))
    for b in (0, 1, B // 2, B - 2, B - 1):
        assert np.array_equal(out[b].cpu().numpy(), O.rgb_add_noise(rgb[b].cpu().numpy(), rec)), b


# ------------------------------------------------------------------ PSP head and upsampling
def test_upsample_bilinear2d_bwd_past_2_31(cuda):
    """grad_out [1, C, 64, 64] with more than 2^31 elements into grad_in [1, C, 3, 3], against torch's autograd of
    align_corners=True upsampling in float64 on the channels around flat 2^31 and the first and last."""
    Hi = Wi = 3
    Ho = Wo = 64
    C = -(-(FLAT + 4096) // (Ho * Wo))
    need(C * Ho * Wo * 4 / GiB + 0.5)
    g = torch.Generator(device=cuda).manual_seed(13)
    go = torch.randn(1, C, Ho, Wo, generator=g, device=cuda)
    gi = sentinel(1, C, Hi, Wi)
    check(lib.ffb6d_upsample_bilinear2d_bwd(go.data_ptr(), 1, C, Hi, Wi, Ho, Wo, gi.data_ptr(), _stream(cuda)))
    assert all_written(gi)
    chans = [0, FLAT // (Ho * Wo) - 1, FLAT // (Ho * Wo), C - 1]
    x = torch.zeros(1, len(chans), Hi, Wi, dtype=torch.float64, device=cuda, requires_grad=True)
    y = F_.interpolate(x, size=(Ho, Wo), mode="bilinear", align_corners=True)
    want, = torch.autograd.grad(y, x, go[:, chans].double())
    close_fp32(gi[:, chans], want, None, "upsample_bilinear2d_bwd")


def test_psp_pool_b65535(cuda):
    B, C, H, W = 65535, 1, 6, 7
    g = torch.Generator(device=cuda).manual_seed(B)
    x = torch.randn(B, C, H, W, generator=g, device=cuda)
    out = sentinel(50 * B * C)
    check(lib.ffb6d_psp_pool(x.data_ptr(), B, C, H, W, out.data_ptr(), _stream(cuda)))
    want = torch.cat([F_.adaptive_avg_pool2d(x.double(), s).reshape(-1) for s in (1, 2, 3, 6)])
    close_fp32(out, want, None, "psp_pool")


# ------------------------------------------------------------------ BatchNorm over ranks
def test_bn_sync_b65535_w65536(cuda):
    """The synchronised BatchNorm with B = 65535 frames and W = 65536 gathered rows, all this rank's own: the combined
    statistics are this batch's (n times W values), so y, grad_z and this rank's grad_gamma / grad_beta are the
    single-batch BatchNorm's, and the global count is exactly W B P."""
    B, C, P, W = 65535, 2, 5, 65536
    eps, momentum, act, slope = 1e-5, 0.1, 2, 0.2
    g = torch.Generator(device=cuda).manual_seed(W)
    z = torch.randn(B, C, P, generator=g, device=cuda)
    gy = torch.randn(B, C, P, generator=g, device=cuda)
    gamma = 1 + 0.5 * torch.randn(C, generator=g, device=cuda)
    beta = 0.5 * torch.randn(C, generator=g, device=cuda)
    z64 = z.double().requires_grad_(True)
    gam64, bet64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    pre64 = F_.batch_norm(z64, None, None, gam64, bet64, True, momentum, eps)
    y64 = F_.leaky_relu(pre64, slope)
    gy = away_from_kink(gy, pre64, act)
    gz64, gg64, gb64 = torch.autograd.grad(y64, (z64, gam64, bet64), gy.double())

    nb = int(lib.ffb6d_bn_workspace_bytes(C, P))
    ws = torch.empty(nb, dtype=torch.uint8, device=cuda)
    st = _stream(cuda)
    moments = torch.empty(2 * C + 1, dtype=torch.float64, device=cuda)
    check(lib.ffb6d_bn_sync_moments(z.data_ptr(), B, C, P, moments.data_ptr(), ws.data_ptr(), nb, st))
    gathered = moments.repeat(W, 1)
    stats, count, y = torch.empty(C, 4, device=cuda), torch.empty(1, dtype=torch.float64, device=cuda), sentinel(B, C, P)
    rm, rv = torch.zeros(C, device=cuda), torch.ones(C, device=cuda)
    check(lib.ffb6d_bn_sync_fwd(z.data_ptr(), B, C, P, gathered.data_ptr(), W, gamma.data_ptr(), beta.data_ptr(), eps,
                                momentum, rm.data_ptr(), rv.data_ptr(), act, slope, stats.data_ptr(), count.data_ptr(),
                                y.data_ptr(), st))
    assert float(count) == W * B * P
    # 1e-4: a thread sums B = 65535 values of a channel in fp32
    close_fp32(y, y64.detach(), None, "bn_sync_fwd y", tol=1e-4)
    sums = torch.empty(2 * C, dtype=torch.float64, device=cuda)
    ggam, gbet, dz = sentinel(C), sentinel(C), sentinel(B, C, P)
    check(lib.ffb6d_bn_sync_bwd_sums(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, C, P, act, slope, sums.data_ptr(),
                                     ggam.data_ptr(), gbet.data_ptr(), ws.data_ptr(), nb, st))
    close_fp32(ggam, gg64, None, "grad_gamma", tol=1e-4)
    close_fp32(gbet, gb64, None, "grad_beta", tol=1e-4)
    gathered = sums.repeat(W, 1)
    check(lib.ffb6d_bn_sync_bwd(z.data_ptr(), gy.data_ptr(), stats.data_ptr(), B, C, P, gathered.data_ptr(), W,
                                count.data_ptr(), act, slope, dz.data_ptr(), ws.data_ptr(), nb, st))
    close_fp32(dz, gz64, None, "bn_sync_bwd grad_z", tol=1e-4)


# ------------------------------------------------------------------ colour jitter
def test_color_jitter_b65535(cuda):
    from ffb6d_b200 import ops
    from oracle import jitter_oracle as J
    B, H, W = 65535, 2, 3
    g = torch.Generator(device=cuda).manual_seed(B)
    rgb = torch.randint(0, 256, (B, H, W, 3), generator=g, device=cuda, dtype=torch.uint8)
    plan = np.asarray(A.draw_color_jitter(B, torch.Generator().manual_seed(5)), np.float64)
    out = ops.color_jitter(rgb, plan)
    for b in (0, 1, B // 2, B - 2, B - 1):
        assert np.array_equal(out[b].cpu().numpy(), J.color_jitter(rgb[b].cpu().numpy(), plan[b])), b


# ------------------------------------------------------------------ segment sums
def segment_want(grad, idx, na):
    """float64 out[b, c, s] = sum of grad[b, c, p] over idx[b, p] == s, and the sum of |terms|."""
    B, C, P = grad.shape
    ok = (idx >= 0) & (idx < na)
    s = torch.where(ok, idx.long(), 0)[:, None, :].expand(B, C, P)
    g = torch.where(ok[:, None, :], grad.double(), 0.0)
    want = torch.zeros(B, C, na, dtype=torch.float64, device=grad.device).scatter_add_(2, s, g)
    return want, torch.zeros_like(want).scatter_add_(2, s, g.abs())


@pytest.mark.parametrize("B,C,P,NA", [(65535, 3, 5, 4), (1, 65535 * 32, 3, 2)], ids=["b65535", "widest_c"])
def test_segment_sum_at_limits(cuda, B, C, P, NA):
    from ffb6d_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(B + C)
    idx = torch.randint(-1, NA + 1, (B, P), generator=g, device=cuda, dtype=torch.int32)    # -1, NA: no segment
    idx[-1, -1] = NA - 1
    grad = torch.randn(B, C, P, generator=g, device=cuda)
    want, mag = segment_want(grad, idx, NA)
    for name, plan in (("counter plan", ops.segment_plan(idx, NA)), ("csr", ops.segment_csr(idx, NA))):
        check_sum(ops.segment_sum(grad, None, NA, plan=plan), want, mag, name)


# ------------------------------------------------------------------ fusion layer
@pytest.mark.parametrize("B,C1,Co,P", [(1, 1, 65535 * 128, 4), (1, 4, 128, (FLAT + 8192) // 128)],
                         ids=["widest_co", "out_past_2_31"])
def test_fusion_mlp_fwd_ex_at_limits(cuda, B, C1, Co, P):
    n = B * Co * P
    need(n * 4 / GiB + 3.0)
    g = torch.Generator(device=cuda).manual_seed(Co + P)
    x = torch.randn(B, C1, P, generator=g, device=cuda)
    w = torch.randn(Co, C1, generator=g, device=cuda)
    scale = 1 + 0.1 * torch.randn(Co, generator=g, device=cuda)
    shift = 0.1 * torch.randn(Co, generator=g, device=cuda)
    out = sentinel(B, Co, P)
    nb = int(lib.ffb6d_fusion_mlp_pack_bytes(Co, C1))
    packed = torch.empty(nb, dtype=torch.uint8, device=cuda)
    check(lib.ffb6d_fusion_mlp_pack(w.data_ptr(), Co, C1, packed.data_ptr(), nb, _stream(cuda)))
    check(lib.ffb6d_fusion_mlp_fwd_ex(x.data_ptr(), C1, None, 0, packed.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                      B, Co, P, 1, 0.0, None, None, 0, 0, LAYOUT_NCS, out.data_ptr(), _stream(cuda)))
    assert all_written(out)
    t = flat_samples(n, n - P + np.arange(64)).to(cuda)               # + the start of the last channel
    b, co, p = t // (Co * P), (t // P) % Co, t % P
    pre = (w.double()[co] * x.double()[b, :, p]).sum(1)
    want = torch.relu(scale.double()[co] * pre + shift.double()[co])
    close_fp32(out.reshape(-1)[t], want, None, "fusion_mlp_fwd")


# ------------------------------------------------------------------ KNN
@pytest.mark.parametrize("algo", [1, 2], ids=["brute", "grid"])
def test_knn_b65535(cuda, algo):
    from ffb6d_b200 import ops
    from oracle import cpu_oracle as CO
    B, S, Q, K = 65535, 8, 3, 4
    rs = np.random.RandomState(algo)
    sup = rs.rand(B, S, 3).astype(np.float32)
    qry = rs.rand(B, Q, 3).astype(np.float32)
    got = ops.knn_search(torch.from_numpy(sup).to(cuda), torch.from_numpy(qry).to(cuda), K, algo=algo).cpu().numpy()
    for b in (0, 1, B // 2, B - 1):
        assert np.array_equal(got[b], CO.knn_search(sup[b][None], qry[b][None], K)[0]), b
