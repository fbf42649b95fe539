// schedule.cu -- the whole per-batch index build of FFB6D behind ONE C call.
//
// Reference: the 22 DP.knn_search calls of datasets/ycb/ycb_dataset.py:269-309 (== datasets/linemod/
// linemod_dataset.py:313-353), executed per frame on the CPU inside Dataset.__getitem__.  Here: all of
// them for a batch, on the caller's stream, into caller-provided buffers -- the native twin of
// ffb6d_b200.schedule.build_ffb6d_indices for hosts that are not Python (and a single node for a
// caller's CUDA graph).  Point sets: cld level i = the first N0 / 4^i points of every frame ("random
// sampling" of the reference is a slice of the shuffled cloud, :233-235, 278); image level sr = the
// stride-sr sub-grid of the organised cloud (:253-267), passed in by the caller (ffb6d_backproject
// produces them).  One grid per (support set, K class) is built and shared by its searches, like the
// Python scheduler does; supports whose searches are all small use the tiled all-pairs scan.
#include "common.cuh"
#include "knn_common.cuh"

#include <algorithm>

namespace ffb6d {

// reference literals (ycb_dataset.py:269-271, 298)
static const int kDsSr[4] = {4, 8, 8, 8};
static const int kUpSr[3] = {4, 2, 2};

struct Call {
    int sup_kind, sup_id;   // kind 0: cld level, 1: image stride
    int qry_kind, qry_id;
    int K;
};

// the reference's call order; `out[i]` of ffb6d_build_indices is call i
static void make_calls(int K, Call (&c)[22])
{
    int n = 0;
    for (int i = 0; i < 4; ++i) {
        c[n++] = {0, i, 0, i, K};                // cld_nei_idx{i}
        c[n++] = {0, i + 1, 0, i, 1};            // cld_interp_idx{i}
        c[n++] = {1, kDsSr[i], 0, i + 1, K};     // r2p_ds_nei_idx{i}
        c[n++] = {0, i + 1, 1, kDsSr[i], 1};     // p2r_ds_nei_idx{i}
    }
    for (int i = 0; i < 3; ++i) {
        const int lvl = 3 - i;
        c[n++] = {1, kUpSr[i], 0, lvl, K};       // r2p_up_nei_idx{i}
        c[n++] = {0, lvl, 1, kUpSr[i], 1};       // p2r_up_nei_idx{i}
    }
}

struct Sizes {
    int64_t cld[5];   // N0 / 4^i
    int64_t img[9];   // by stride (2, 4, 8 used)
};

static Sizes make_sizes(int64_t N0, int64_t H, int64_t W)
{
    Sizes s{};
    s.cld[0] = N0;
    for (int i = 1; i < 5; ++i) s.cld[i] = s.cld[i - 1] / 4;
    for (int sr : {2, 4, 8}) s.img[sr] = (H / sr) * (W / sr);
    return s;
}

static int64_t size_of(const Sizes &z, int kind, int id) { return kind == 0 ? z.cld[id] : z.img[id]; }

// rows of a search from image level sr_c = every f-th pixel of every f-th image row of the search from level sr_c / f
// (4-byte words: `words` per index row)
__global__ void __launch_bounds__(256)
strided_pixels_copy_kernel(const unsigned *__restrict__ in, unsigned *__restrict__ out, int Hc, int Wc, int Hp, int Wp, int f,
                           int words, long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int wd = (int)(t % words);
    long long px = t / words;
    const int c = (int)(px % Wc);
    px /= Wc;
    const int r = (int)(px % Hc);
    const long long b = px / Hc;
    out[t] = __ldg(in + (((b * Hp + (long long)r * f) * Wp + (long long)c * f) * words + wd));
}

struct Plan {
    size_t levels_off[5];   // contiguous copies of cld levels 1..4
    size_t grid_off, scratch_off, total;
};

static Plan make_plan(int64_t B, const Sizes &z, int K)
{
    Plan p{};
    size_t off = 0;
    for (int i = 1; i < 5; ++i) {
        p.levels_off[i] = off;
        off = align_up(off + (size_t)B * (size_t)z.cld[i] * 3 * sizeof(float), 256);
    }
    Call calls[22];
    make_calls(K, calls);
    size_t grid = 0, scratch = 0;
    for (const Call &c : calls) {
        const int64_t S = size_of(z, c.sup_kind, c.sup_id), Q = size_of(z, c.qry_kind, c.qry_id);
        if (S > 0) grid = std::max(grid, knn_grid_store_bytes(B, S));
        if (Q > 0) scratch = std::max(scratch, knn_grid_query_bytes(B, Q));
    }
    p.grid_off = off;
    off = align_up(off + grid, 256);
    p.scratch_off = off;
    off = align_up(off + scratch, 256);
    p.total = off;
    return p;
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" size_t ffb6d_build_indices_workspace_bytes(int64_t B, int64_t N0, int64_t H, int64_t W, int K)
{
    if (B <= 0 || N0 < 256 || H < 8 || W < 8 || K < 1 || K > FFB6D_MAX_K) return 0;
    return make_plan(B, make_sizes(N0, H, W), K).total;
}

extern "C" int ffb6d_build_indices(const float *cld, const float *img2, const float *img4, const float *img8, int64_t B,
                                   int64_t N0, int64_t H, int64_t W, int K, void *const *out, int idx_is_i64,
                                   void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && B < 65536, "build_indices: bad batch size");
    FFB6D_CHECK_ARG(N0 >= 256 && N0 % 256 == 0 && N0 < (1ll << 31), "build_indices: N0=%lld must be a positive multiple of 256",
                    (long long)N0);
    FFB6D_CHECK_ARG(H >= 8 && W >= 8 && H % 8 == 0 && W % 8 == 0, "build_indices: H, W must be multiples of 8");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "build_indices: K=%d outside [1,%d]", K, FFB6D_MAX_K);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(cld && img2 && img4 && img8 && out && workspace, "build_indices: null pointer");
    for (int i = 0; i < 22; ++i) FFB6D_CHECK_ARG(out[i], "build_indices: out[%d] is null", i);
    const Sizes z = make_sizes(N0, H, W);
    const Plan plan = make_plan(B, z, K);
    if (workspace_bytes < plan.total) {
        set_error("build_indices: workspace of %zu bytes required, %zu given", plan.total, workspace_bytes);
        return FFB6D_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    // contiguous [B, N_i, 3] copies of the cloud levels (a level is the first N_i rows of every frame)
    const float *level[5] = {cld, nullptr, nullptr, nullptr, nullptr};
    for (int i = 1; i < 5; ++i) {
        float *dst = (float *)(ws + plan.levels_off[i]);
        FFB6D_CUDA(cudaMemcpy2DAsync(dst, (size_t)z.cld[i] * 12, cld, (size_t)N0 * 12, (size_t)z.cld[i] * 12, (size_t)B,
                                     cudaMemcpyDeviceToDevice, st));
        level[i] = dst;
    }
    auto set_ptr = [&](int kind, int id) -> const float * {
        if (kind == 0) return level[id];
        return id == 2 ? img2 : (id == 4 ? img4 : img8);
    };
    Call calls[22];
    make_calls(K, calls);
    bool done[22] = {};
    // Cloud level j is a row prefix of level i < j: a search of the same support with the same K whose queries are a
    // deeper cloud level is a row slice of the shallower one (r2p_ds_nei_idx2/3 of idx1, r2p_up_nei_idx0 of
    // r2p_ds_nei_idx0, r2p_up_nei_idx1 of idx2): those four are copied, not searched.
    int parent[22];
    for (int i = 0; i < 22; ++i) {
        parent[i] = -1;
        if (calls[i].qry_kind != 0) continue;
        for (int j = 0; j < 22; ++j)
            if (j != i && calls[j].qry_kind == 0 && calls[j].sup_kind == calls[i].sup_kind && calls[j].sup_id == calls[i].sup_id &&
                calls[j].K == calls[i].K && calls[j].qry_id < calls[i].qry_id &&
                (parent[i] < 0 || calls[j].qry_id < calls[parent[i]].qry_id))
                parent[i] = j;
    }
    // Image level sr_c is every (sr_c / sr_p)-th pixel of every (sr_c / sr_p)-th row of level sr_p: K = 1 searches from
    // img4 / img8 into a cloud level are strided subsets of the search from img2 / img4 into the same level
    // (p2r_ds_nei_idx0 of p2r_up_nei_idx2, idx1 of p2r_up_nei_idx1, idx2 of p2r_up_nei_idx0): copied, not searched.
    int stride_f[22];
    for (int i = 0; i < 22; ++i) {
        stride_f[i] = 0;
        if (calls[i].qry_kind != 1 || H % calls[i].qry_id != 0 || W % calls[i].qry_id != 0) continue;
        for (int j = 0; j < 22; ++j)
            if (j != i && calls[j].qry_kind == 1 && calls[j].sup_kind == calls[i].sup_kind && calls[j].sup_id == calls[i].sup_id &&
                calls[j].K == calls[i].K && calls[j].qry_id < calls[i].qry_id && calls[i].qry_id % calls[j].qry_id == 0 &&
                (parent[i] < 0 || calls[j].qry_id < calls[parent[i]].qry_id)) {
                parent[i] = j;
                stride_f[i] = calls[i].qry_id / calls[j].qry_id;
            }
    }
    void *grid = ws + plan.grid_off, *scratch = ws + plan.scratch_off;
    for (int i = 0; i < 22; ++i) {
        if (done[i]) continue;
        // all searches into the same support with the same K class share one grid
        const Call &c = calls[i];
        const int64_t S = size_of(z, c.sup_kind, c.sup_id);
        const float *sup = set_ptr(c.sup_kind, c.sup_id);
        bool use_grid = false;
        for (int j = i; j < 22; ++j)
            if (calls[j].sup_kind == c.sup_kind && calls[j].sup_id == c.sup_id && calls[j].K == c.K)
                use_grid = use_grid || knn_grid_workspace_bytes(B, S, size_of(z, calls[j].qry_kind, calls[j].qry_id), c.K) > 0;
        if (use_grid) {
            const int rc = knn_grid_build(sup, B, S, c.K, grid, knn_grid_store_bytes(B, S), st);
            if (rc != FFB6D_OK) return rc;
        }
        for (int j = i; j < 22; ++j) {
            const Call &d = calls[j];
            if (done[j] || d.sup_kind != c.sup_kind || d.sup_id != c.sup_id || d.K != c.K) continue;
            if (parent[j] >= 0) continue;   // a row slice of another search: copied below
            const int64_t Q = size_of(z, d.qry_kind, d.qry_id);
            const float *qry = set_ptr(d.qry_kind, d.qry_id);
            int rc;
            if (use_grid)
                rc = knn_grid_query(sup, qry, B, S, Q, d.K, out[j], idx_is_i64, grid, knn_grid_store_bytes(B, S), scratch,
                                    knn_grid_query_bytes(B, Q), st, d.qry_kind == 1 ? W / d.qry_id : 0);
            else
                rc = knn_brute_launch(sup, qry, B, S, Q, d.K, out[j], idx_is_i64, st);
            if (rc != FFB6D_OK) return rc;
            done[j] = true;
        }
    }
    const size_t esz = idx_is_i64 ? 8 : 4;
    for (int i = 0; i < 22; ++i) {
        if (parent[i] < 0) continue;
        const int64_t Qc = size_of(z, calls[i].qry_kind, calls[i].qry_id), Qp = size_of(z, calls[parent[i]].qry_kind, calls[parent[i]].qry_id);
        const size_t row = (size_t)calls[i].K * esz;
        if (stride_f[i] > 0) {
            const int sc = calls[i].qry_id, sp = calls[parent[i]].qry_id, words = (int)(row / 4);
            const long long total = (long long)B * Qc * words;
            strided_pixels_copy_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(
                (const unsigned *)out[parent[i]], (unsigned *)out[i], (int)(H / sc), (int)(W / sc), (int)(H / sp), (int)(W / sp),
                stride_f[i], words, total);
            FFB6D_LAUNCH_OK("strided_pixels_copy_kernel");
            continue;
        }
        FFB6D_CUDA(cudaMemcpy2DAsync(out[i], (size_t)Qc * row, out[parent[i]], (size_t)Qp * row, (size_t)Qc * row, (size_t)B,
                                     cudaMemcpyDeviceToDevice, st));
    }
    return FFB6D_OK;
}
