// knn_grid.cu -- exact KNN through a uniform grid over the support cloud (sm_90a).
//
// The reference answers every query with a KD-tree descent (NN/nanoflann.hpp:1350-1408).
// On the GPU the same *result* -- the K support points with the smallest reference-arithmetic
// fp32 distance, ordered by (distance, index) -- is produced by binning the support into a
// uniform grid and scanning only the cells around each query:
//
//   A-D. build  : ONE kernel, a cluster of 8 CTAs per batch item (grid_build_kernel): bounding box,
//                 an ESTIMATE of the K-th neighbour distance from 32 sample points scanned against
//                 a strided subsample -> cell edge h and grid dims; counting sort of the points
//                 into cells (one atomic per point, prefix sum of the cell counters, points
//                 (x,y,z,index) written cell-contiguous as float4)
//   E. search   : one thread per query scans the (2r+1)^3 block of cells around it, r = 1..RMAX
//                 (each ring adds only its shell of cells), keeping a sorted top-K in registers; a row of cells along x is one contiguous
//                 range of the sorted array, read four points at a time.  The search stops as
//                 soon as the K-th distance is provably smaller than the distance to anything
//                 outside the block.
//   F. overflow : queries that cannot be certified within RMAX rings (far from the support: the
//                 (0,0,0) hole pixels of the organised cloud, K > S, ...) are answered by a tiled
//                 scan of the whole support.  Far queries that are equal to the first
//                 far query of their batch item (all hole pixels are) are not searched again:
//   G. dup copy : they receive a copy of that query's result row.
//
// Exactness: candidates are evaluated with the reference arithmetic (common.cuh ref_sqdist) and
// ranked by the total order (distance, index), so the result does not depend on the order in
// which cells or points are visited, nor on h or the estimate; the stop test is conservative
// (see `slack`).  HBM traffic per call is ~ the algorithmic 12S + 12Q + 4QK plus the 16S sorted
// copy and the cell table; everything else stays in L1/L2.
#include "common.cuh"
#include "knn_common.cuh"

#include <algorithm>
#include <cooperative_groups.h>
#include <math.h>
#include <stdlib.h>

namespace ffb6d {

constexpr int RMAX = 4;                 // widest block: 9x9x9 cells
constexpr int N_SAMPLES = 32;           // sample points of the K-th-distance estimate
constexpr int BUILD_CTAS = 8;           // thread-block cluster that builds one batch item's grid
constexpr int BUILD_THREADS = 512;
constexpr int BUILD_WARPS = BUILD_THREADS / 32;
constexpr int BUILD_GT = BUILD_CTAS * BUILD_THREADS;   // threads per batch item
static_assert(N_SAMPLES == BUILD_CTAS * 4 && BUILD_WARPS == 16, "4 samples per CTA, 4 warps per sample");

struct __align__(16) GridParams {
    float lo[3];
    float h;        // cell edge
    float inv_h;    // 0 when the grid is a single cell along every axis
    float slack;    // absolute safety margin of the stop test
    int n[3];       // cells per axis
    int ncells;
    float hi[3];
    int pad[3];
};
static_assert(sizeof(GridParams) == 64, "GridParams layout");

// per batch item, per query call: who could not be certified by the grid
struct __align__(16) QueryState {
    int ovf_count;  // queries handed to the overflow pass (front of the ovf list)
    int dup_count;  // far queries equal to rep_q (back of the ovf list)
    int rep_q;      // 1 + first far query of this item, 0 if none
    int pad;        // CTAs of the overflow kernel that have finished (last one copies the duplicate rows)
};

// The grid of one support batch: written by knn_grid_build, read-only afterwards, so any
// number of query calls (on any stream ordered after the build) can share it.
struct GridStore {
    GridParams *params;   // [B]
    int *cursor;          // [B][maxc]  counts -> inclusive prefix = END offset of every cell
    int *rank;            // [B][S]     arrival rank of a point inside its cell (build scratch)
    float4 *sorted;       // [B][S]     (x, y, z, original index), cell-contiguous
    size_t maxc;
    size_t bytes;
};

// scratch of one query call
struct QueryScratch {
    QueryState *state;    // [B]
    int *ovf;             // [B][Q]
    size_t bytes;
};

static size_t max_cells_for(int64_t S)
{
    size_t m = (size_t)S * 8;   // 32 cells per point measured slower (more empty rows to look up)
    if (m < 4096) m = 4096;
    if (m > ((size_t)1 << 22)) m = (size_t)1 << 22;
    return (m + 4095) / 4096 * 4096;   // 16-byte aligned rows
}

static GridStore carve_grid(void *base, int64_t B, int64_t S)
{
    GridStore w;
    w.maxc = max_cells_for(S);
    size_t off = 0;
    char *p = (char *)base;
    auto take = [&](size_t bytes) {
        char *r = p + off;
        off = align_up(off + bytes, 256);
        return r;
    };
    w.params = (GridParams *)take((size_t)B * sizeof(GridParams));
    w.cursor = (int *)take((size_t)B * w.maxc * sizeof(int));
    w.rank = (int *)take((size_t)B * (size_t)S * sizeof(int));
    w.sorted = (float4 *)take((size_t)B * (size_t)S * sizeof(float4));
    w.bytes = off;
    return w;
}

static QueryScratch carve_query(void *base, int64_t B, int64_t Q)
{
    QueryScratch w;
    size_t off = 0;
    char *p = (char *)base;
    w.state = (QueryState *)(p + off);
    off = align_up(off + (size_t)B * sizeof(QueryState), 256);
    w.ovf = (int *)(p + off);
    off = align_up(off + (size_t)B * (size_t)Q * sizeof(int), 256);
    w.bytes = off;
    return w;
}

size_t knn_grid_store_bytes(int64_t B, int64_t S) { return carve_grid(nullptr, B, S).bytes; }
size_t knn_grid_query_bytes(int64_t B, int64_t Q) { return carve_query(nullptr, B, Q).bytes; }

// The grid pays off once the all-pairs scan is big enough to dwarf its launches.
static bool grid_worthwhile(int64_t B, int64_t S, int64_t Q, int K)
{
    (void)B;
    (void)K;
    return S >= 512 && (double)S * (double)Q >= 2.0e5;
}

size_t knn_grid_workspace_bytes(int64_t B, int64_t S, int64_t Q, int K)
{
    if (!grid_worthwhile(B, S, Q, K)) return 0;
    return knn_grid_store_bytes(B, S) + knn_grid_query_bytes(B, Q);
}

__device__ __forceinline__ int cell_of(float p, float lo, float inv_h, int n)
{
    const int c = (int)floorf((p - lo) * inv_h);
    return min(max(c, 0), n - 1);
}

// ------------------------------------------------------------------ A-D. grid build: ONE kernel
// A thread-block cluster of 8 CTAs (4096 threads) builds the grid of one batch item; the phases
// are separated by hardware cluster barriers and exchange their small results through distributed
// shared memory, so the whole build is a single launch (it was five):
//   1. partial bounding box per CTA; the K-th-neighbour-distance ESTIMATE: 32 sample points, four
//      per CTA, four warps per sample, each warp scanning a quarter of a strided subsample of the
//      support (k' points of the subsample stand for k'*stride >= K points of the cloud)
//   2. rank 0 gathers the 8 boxes and 32 estimates over DSMEM, picks the quantile, derives the
//      cell edge h and the grid dims, publishes the parameters
//   3. the cell counters that exist are zeroed
//   4. count: one atomic per point; the value it returns is the point's arrival rank inside its
//      cell, kept for step 6 (no second round of atomics); per-CTA totals of the 8 scan slices
//   5. inclusive prefix sum of the counters (cell -> END offset): every CTA scans one slice, its
//      warps own contiguous runs (coalesced 512-byte steps, shuffles only, no CTA barrier inside)
//   6. scatter: point -> sorted[end(cell-1) + rank] as float4 (x, y, z, original index)
// The order of the points inside a cell depends on the atomics' arrival order; search results do
// not (candidates are ranked by the total order (distance, index)).
__global__ void __cluster_dims__(BUILD_CTAS, 1, 1) __launch_bounds__(BUILD_THREADS)
grid_build_kernel(const float *__restrict__ support, int S, int K, int maxc, float cell_scale, int quantile,
                  GridParams *__restrict__ params, int *__restrict__ cursor_all, int *__restrict__ rank_all,
                  float4 *__restrict__ sorted_all)
{
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int crank = (int)cluster.block_rank();
    const int b = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int gtid = crank * BUILD_THREADS + tid;
    const float *sup = support + (size_t)b * S * 3;
    int *cur = cursor_all + (size_t)b * maxc;
    int *rnk = rank_all + (size_t)b * S;
    float4 *sorted = sorted_all + (size_t)b * S;
    const float INF = __int_as_float(0x7f800000);

    __shared__ float s_red[6][BUILD_WARPS];
    __shared__ float s_box[6];              // this CTA's partial bounding box
    __shared__ float s_cand[4][4][4];       // [sample of this CTA][warp of the sample][k']
    __shared__ float s_est[4];              // this CTA's four estimates
    __shared__ float s_all[N_SAMPLES];      // rank 0: all estimates
    __shared__ float s_pick;
    __shared__ GridParams s_P;              // rank 0 publishes, everybody copies
    __shared__ int s_tot[BUILD_CTAS];       // points this CTA counted into each scan slice
    __shared__ int s_wsum[BUILD_WARPS];
    __shared__ int s_base;

    // ---- 1a. partial bounding box
    {
        float mn[3] = {INF, INF, INF}, mx[3] = {-INF, -INF, -INF};
        for (int s = gtid; s < S; s += BUILD_GT) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const float v = __ldg(sup + (size_t)s * 3 + a);
                mn[a] = fminf(mn[a], v);
                mx[a] = fmaxf(mx[a], v);
            }
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
                mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
            }
            if (lane == 0) {
                s_red[a][wid] = mn[a];
                s_red[3 + a][wid] = mx[a];
            }
        }
        if (tid < BUILD_CTAS) s_tot[tid] = 0;
        __syncthreads();
        if (wid == 0) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                float u = lane < BUILD_WARPS ? s_red[a][lane] : INF, v = lane < BUILD_WARPS ? s_red[3 + a][lane] : -INF;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    u = fminf(u, __shfl_xor_sync(0xffffffffu, u, o));
                    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
                }
                if (lane == 0) {
                    s_box[a] = u;
                    s_box[3 + a] = v;
                }
            }
        }
    }
    // ---- 1b. estimate of the K-th neighbour distance (does not need the box)
    {
        const int stride = max((S + 4095) / 4096, (K + 3) / 4);
        const int kk = max(1, (K + stride - 1) / stride);          // <= 4
        const int smp = crank * 4 + (wid >> 2), w4 = wid & 3;
        const int me = (int)((((long long)smp * S) / N_SAMPLES + S / (2 * N_SAMPLES)) % max(S, 1));
        float out[4] = {INF, INF, INF, INF};
        if (S > 1) {
            const float qx = __ldg(sup + (size_t)me * 3), qy = __ldg(sup + (size_t)me * 3 + 1),
                        qz = __ldg(sup + (size_t)me * 3 + 2);
            TopK<4> t4;
            t4.init();
            const int nsub = (S + stride - 1) / stride;              // subsample = points 0, stride, 2*stride, ...
            for (int i0 = w4 * 32 + lane; i0 < nsub; i0 += 4 * 128) {   // 12 loads in flight
                float px[4], py[4], pz[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int s = min((i0 + u * 128) * stride, S - 1);
                    px[u] = __ldg(sup + (size_t)s * 3);
                    py[u] = __ldg(sup + (size_t)s * 3 + 1);
                    pz[u] = __ldg(sup + (size_t)s * 3 + 2);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int i = i0 + u * 128, s = i * stride;
                    const float d = ref_sqdist(qx, qy, qz, px[u], py[u], pz[u]);
                    if (i < nsub && s != me && d < t4.worst()) t4.push_ordered(d, s);
                }
            }
#pragma unroll
            for (int round = 0; round < 4; ++round) {   // pop this warp's minimum kk (<= 4) times
                if (round >= kk) break;
                float m = t4.d[0];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
                const unsigned who = __ballot_sync(0xffffffffu, t4.d[0] == m);
                if (lane == __ffs(who) - 1) {
                    t4.d[0] = t4.d[1];
                    t4.d[1] = t4.d[2];
                    t4.d[2] = t4.d[3];
                    t4.d[3] = INF;
                }
                out[round] = m;
            }
        }
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j) s_cand[wid >> 2][w4][j] = out[j];
        }
        __syncthreads();
        if (wid < 4) {   // the kk-th smallest of the sample's 16 candidates
            const float mine = lane < 16 ? s_cand[wid][lane >> 2][lane & 3] : INF;
            int rank = 0;
            for (int j = 0; j < 16; ++j) {
                const float o = __shfl_sync(0xffffffffu, mine, j);
                rank += (o < mine || (o == mine && j < lane)) ? 1 : 0;
            }
            // kk*stride-th neighbour measured; scale to the K-th assuming a 2-D sheet
            if (lane < 16 && rank == kk - 1) {
                const float r = (S > 1) ? sqrtf(mine) * sqrtf((float)K / (float)(kk * stride)) : 0.f;
                s_est[wid] = (r == r && r < INF) ? r : 0.f;
            }
        }
    }
    cluster.sync();
    // ---- 2. rank 0: full box, quantile of the estimates, grid parameters
    if (crank == 0) {
        if (wid == 0) {
            s_all[lane] = cluster.map_shared_rank(s_est, lane >> 2)[lane & 3];
            if (lane < 6) {
                float v = (lane < 3) ? INF : -INF;
                for (int c = 0; c < BUILD_CTAS; ++c) {
                    const float o = cluster.map_shared_rank(s_box, c)[lane];
                    v = (lane < 3) ? fminf(v, o) : fmaxf(v, o);
                }
                s_red[lane][0] = v;
            }
            __syncwarp();
            // the `quantile`-th smallest of the 32 estimates (hole pixels give zeros: they rank first)
            const float mine = s_all[lane];
            int rank = 0;
            for (int j = 0; j < N_SAMPLES; ++j) {
                const float o = s_all[j];
                rank += (o < mine || (o == mine && j < lane)) ? 1 : 0;
            }
            if (rank == quantile) s_pick = mine;
            __syncwarp();
            if (lane == 0) {
                float mn[3], mx[3];
                for (int a = 0; a < 3; ++a) {
                    mn[a] = s_red[a][0];
                    mx[a] = s_red[3 + a][0];
                }
                const float r_est = s_pick;
                GridParams P;
                float L[3], scale = 0.f;
                bool finite = true;
                for (int a = 0; a < 3; ++a) {
                    L[a] = mx[a] - mn[a];
                    finite = finite && isfinite(L[a]) && isfinite(mn[a]);
                    scale = fmaxf(scale, fmaxf(fabsf(mn[a]), fabsf(mx[a])));
                    P.lo[a] = mn[a];
                    P.hi[a] = mx[a];
                }
                const float l1 = fmaxf(L[0], fmaxf(L[1], L[2]));
                const float l3 = fminf(L[0], fminf(L[1], L[2]));
                const float l2 = L[0] + L[1] + L[2] - l1 - l3;
                float h = cell_scale * r_est;
                if (!(h > 0.f)) h = sqrtf((float)K * l1 * l2 / (float)max(S, 1));   // geometric fallback
                if (!(h > 0.f)) h = l1 * (float)K / (float)max(S, 1);               // points on a line
                int n[3] = {1, 1, 1};
                if (finite && h > 0.f && l1 > 0.f) {
                    for (int it = 0; it < 200; ++it) {
                        double prod = 1.0;
                        for (int a = 0; a < 3; ++a) {
                            const float f = floorf(L[a] / h);
                            n[a] = (f >= 4.0e6f) ? 4000000 : (int)f + 1;
                            prod *= (double)n[a];
                        }
                        if (prod <= (double)maxc) break;
                        h *= 1.2f;
                        if (it == 199) n[0] = n[1] = n[2] = 1;
                    }
                }
                const bool single = (n[0] == 1 && n[1] == 1 && n[2] == 1);
                P.h = single ? INF : h;
                P.inv_h = single ? 0.f : 1.0f / h;
                P.slack = 1e-5f * (scale + l1) + 1e-30f;
                P.n[0] = n[0];
                P.n[1] = n[1];
                P.n[2] = n[2];
                P.ncells = n[0] * n[1] * n[2];
                for (int a = 0; a < 3; ++a) P.pad[a] = 0;
                s_P = P;
                params[b] = P;
            }
        }
    }
    cluster.sync();
    if (crank != 0 && tid < 16)   // one 64-byte DSMEM read per CTA
        reinterpret_cast<float *>(&s_P)[tid] = reinterpret_cast<const float *>(cluster.map_shared_rank(&s_P, 0))[tid];
    __syncthreads();
    const GridParams P = s_P;
    const int ncells = P.ncells;
    // scan slices: 8 equal runs of cells, a multiple of 128 cells each (whole 512-byte warp steps)
    const int slice = ((ncells + BUILD_CTAS * 128 - 1) / (BUILD_CTAS * 128)) * 128;
    // ---- 3. zero the counters that exist
    {
        int4 *c4 = reinterpret_cast<int4 *>(cur);
        const int n4 = min((ncells + 3) / 4, maxc / 4);
        for (int i = gtid; i < n4; i += BUILD_GT) c4[i] = make_int4(0, 0, 0, 0);
    }
    cluster.sync();
    // ---- 4. count (the returned value is the point's rank inside its cell)
    {
        int acc = 0;   // lane j < 8: points this warp put into slice j
        const int iters = (S + BUILD_GT - 1) / BUILD_GT;
        for (int it = 0; it < iters; ++it) {
            const int s = it * BUILD_GT + gtid;
            int sl = -1;
            if (s < S) {
                const float *p = sup + (size_t)s * 3;
                const int cx = cell_of(__ldg(p), P.lo[0], P.inv_h, P.n[0]);
                const int cy = cell_of(__ldg(p + 1), P.lo[1], P.inv_h, P.n[1]);
                const int cz = cell_of(__ldg(p + 2), P.lo[2], P.inv_h, P.n[2]);
                const int cell = (cz * P.n[1] + cy) * P.n[0] + cx;
                rnk[s] = atomicAdd(cur + cell, 1);
                sl = cell / slice;
            }
#pragma unroll
            for (int j = 0; j < BUILD_CTAS; ++j) {
                const int v = __popc(__ballot_sync(0xffffffffu, sl == j));
                if (lane == j) acc += v;
            }
        }
        if (lane < BUILD_CTAS && acc) atomicAdd(&s_tot[lane], acc);
    }
    cluster.sync();
    // ---- 5. inclusive prefix sum of slice `crank`
    {
        if (wid == 0) {   // points in the slices before mine, summed over the 8 CTAs' tallies
            int t = 0;
            if (lane < BUILD_CTAS)
                for (int c = 0; c < BUILD_CTAS; ++c) t += cluster.map_shared_rank(s_tot, c)[lane];
            int before = (lane < crank) ? t : 0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
            if (lane == 0) s_base = before;
        }
        const int lo = crank * slice, hi = min(ncells, lo + slice);
        // warp w owns the contiguous run [wlo, whi) of the slice, a multiple of 128 cells long
        const int run = ((slice / 128 + BUILD_WARPS - 1) / BUILD_WARPS) * 128;
        const int wlo = min(hi, lo + wid * run), whi = min(hi, wlo + run);
        int tot = 0;
        for (int i = wlo + 4 * lane; i < whi; i += 128) {   // pass 1: total of the run (whi may cut a lane's int4)
            const int4 v = *reinterpret_cast<const int4 *>(cur + i);
            tot += v.x + (i + 1 < whi ? v.y : 0) + (i + 2 < whi ? v.z : 0) + (i + 3 < whi ? v.w : 0);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
        if (lane == 0) s_wsum[wid] = tot;
        __syncthreads();
        int carry = s_base;
        for (int w = 0; w < wid; ++w) carry += s_wsum[w];
        for (int i0 = wlo; i0 < whi; i0 += 128) {           // pass 2: scan, coalesced 512-byte steps
            const int i = i0 + 4 * lane;
            int4 v = make_int4(0, 0, 0, 0);
            if (i < whi) {
                v = *reinterpret_cast<const int4 *>(cur + i);
                if (i + 1 >= whi) v.y = 0;
                if (i + 2 >= whi) v.z = 0;
                if (i + 3 >= whi) v.w = 0;
            }
            const int t = v.x + v.y + v.z + v.w;
            int incl = t;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += u;
            }
            const int start = carry + incl - t;
            if (i < whi) {
                int4 e;
                e.x = start + v.x;
                e.y = e.x + v.y;
                e.z = e.y + v.z;
                e.w = e.z + v.w;
                if (i + 3 < whi) {
                    *reinterpret_cast<int4 *>(cur + i) = e;
                } else {
                    cur[i] = e.x;
                    if (i + 1 < whi) cur[i + 1] = e.y;
                    if (i + 2 < whi) cur[i + 2] = e.z;
                }
            }
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    cluster.sync();
    // ---- 6. scatter
    for (int s = gtid; s < S; s += BUILD_GT) {
        const float *p = sup + (size_t)s * 3;
        const float x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
        const int cx = cell_of(x, P.lo[0], P.inv_h, P.n[0]);
        const int cy = cell_of(y, P.lo[1], P.inv_h, P.n[1]);
        const int cz = cell_of(z, P.lo[2], P.inv_h, P.n[2]);
        const int cell = (cz * P.n[1] + cy) * P.n[0] + cx;
        const int pos = (cell > 0 ? cur[cell - 1] : 0) + rnk[s];
        sorted[pos] = make_float4(x, y, z, __int_as_float(s));
    }
    // after this kernel cursor[c] is the END of cell c; its start is cursor[c-1] (0 for c == 0)
}

// (dz, dy) offsets of the cell rows of a block, nearest first: nested by Chebyshev ring (entries
// [0,9) ring <= 1, [0,25) ring <= 2, [0,49) ring <= 3, [0,81) ring <= 4), Euclid-sorted inside a ring.
// Scanning rows centre-out makes the K-th distance tight early, so later rows are mostly pruned
// by their minimum possible distance.
__constant__ signed char kRowOrder[81][2] = {{0,0}, {-1,0}, {0,-1}, {0,1}, {1,0}, {-1,-1}, {-1,1}, {1,-1}, {1,1}, {-2,0}, {0,-2}, {0,2}, {2,0}, {-2,-1}, {-2,1}, {-1,-2}, {-1,2}, {1,-2}, {1,2}, {2,-1}, {2,1}, {-2,-2}, {-2,2}, {2,-2}, {2,2}, {-3,0}, {0,-3}, {0,3}, {3,0}, {-3,-1}, {-3,1}, {-1,-3}, {-1,3}, {1,-3}, {1,3}, {3,-1}, {3,1}, {-3,-2}, {-3,2}, {-2,-3}, {-2,3}, {2,-3}, {2,3}, {3,-2}, {3,2}, {-3,-3}, {-3,3}, {3,-3}, {3,3}, {-4,0}, {0,-4}, {0,4}, {4,0}, {-4,-1}, {-4,1}, {-1,-4}, {-1,4}, {1,-4}, {1,4}, {4,-1}, {4,1}, {-4,-2}, {-4,2}, {-2,-4}, {-2,4}, {2,-4}, {2,4}, {4,-2}, {4,2}, {-4,-3}, {-4,3}, {-3,-4}, {-3,4}, {3,-4}, {3,4}, {4,-3}, {4,3}, {-4,-4}, {-4,4}, {4,-4}, {4,4}};

// squared distance from coordinate q to the slab [lo + c*h, lo + (c+1)*h], shrunk by the safety slack
__device__ __forceinline__ float slab_dist2(float q, float lo, float h, int c, float slack)
{
    const float a = lo + (float)c * h, b = lo + (float)(c + 1) * h;
    const float d = fmaxf(fmaxf(a - q, q - b) - slack, 0.f);
    return d * d;
}

// ------------------------------------------------------------------ E. search
// One query, one thread: scan the (2r+1)^3 block of cells around the query, r = 1..RMAX (each ring
// adds only its shell), keeping a sorted top-K in registers.  Returns true when the K-th distance is
// provably smaller than the distance to anything outside the scanned block.
template <int KCAP>
__device__ __forceinline__ bool thread_search(float qx, float qy, float qz, int K, const GridParams &Ps,
                                              const int *__restrict__ cell_end, const float4 *__restrict__ sorted,
                                              TopK<KCAP> &top)
{
    const int nx = Ps.n[0], ny = Ps.n[1], nz = Ps.n[2];
    const float h = Ps.h, slack = Ps.slack;
    const int cx = cell_of(qx, Ps.lo[0], Ps.inv_h, nx);
    const int cy = cell_of(qy, Ps.lo[1], Ps.inv_h, ny);
    const int cz = cell_of(qz, Ps.lo[2], Ps.inv_h, nz);
    const float INF = __int_as_float(0x7f800000);
    // a query further than RMAX cells outside the support's box cannot be certified by any block
    const float out = fmaxf(fmaxf(fmaxf(Ps.lo[0] - qx, qx - Ps.hi[0]), fmaxf(Ps.lo[1] - qy, qy - Ps.hi[1])),
                            fmaxf(Ps.lo[2] - qz, qz - Ps.hi[2]));
    bool done = false;
    auto scan_range = [&](int beg, int end) {
        for (int p = beg; p < end; p += 4) {   // four loads in flight per thread
            float4 c[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) c[u] = __ldg(sorted + min(p + u, end - 1));
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float d = ref_sqdist(qx, qy, qz, c[u].x, c[u].y, c[u].z);
                const int id = __float_as_int(c[u].w);
                if (p + u < end && top.accepts(d, id)) top.push_any(d, id);
            }
        }
    };
    auto cells = [&](int row, int a, int b2) {   // points of cells [a, b2] of one x-row
        const int beg = (row + a > 0) ? __ldg(cell_end + row + a - 1) : 0;
        scan_range(beg, __ldg(cell_end + row + b2));
    };
    const int r_first = (out > (float)RMAX * h) ? RMAX + 1 : 1;
    int px0 = 1, px1 = 0, py0 = 1, py1 = 0, pz0 = 1, pz1 = 0;   // block already scanned (empty)
    for (int r = r_first; r <= RMAX && !done; ++r) {
        const int x0 = max(cx - r, 0), x1 = min(cx + r, nx - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, ny - 1);
        const int z0 = max(cz - r, 0), z1 = min(cz + r, nz - 1);
        const int e0 = (2 * r - 1) * (2 * r - 1) * (r > r_first ? 1 : 0);   // rows of the inner block are done
        const int e1 = (2 * r + 1) * (2 * r + 1);
        // new x-cells of the rows already visited (ring growth)
        if (r > r_first) {
            for (int e = 0; e < e0; ++e) {
                const int z = cz + kRowOrder[e][0], y = cy + kRowOrder[e][1];
                if (z < pz0 || z > pz1 || y < py0 || y > py1) continue;
                const int row = (z * ny + y) * nx;
                if (x0 < px0) cells(row, x0, px0 - 1);
                if (x1 > px1) cells(row, px1 + 1, x1);
            }
        }
        for (int e = e0; e < e1; ++e) {   // centre-out
            const int z = cz + kRowOrder[e][0], y = cy + kRowOrder[e][1];
            if (z < z0 || z > z1 || y < y0 || y > y1) continue;
            // skip rows that cannot hold anything closer than the current K-th best
            const float dmin2 = slab_dist2(qy, Ps.lo[1], h, y, slack) + slab_dist2(qz, Ps.lo[2], h, z, slack);
            if (dmin2 > top.kth(K)) continue;
            cells((z * ny + y) * nx, x0, x1);
        }
        px0 = x0; px1 = x1; py0 = y0; py1 = y1; pz0 = z0; pz1 = z1;
        // distance from the query to the nearest face of the block that still has cells behind it
        float m = INF;
        if (x0 > 0) m = fminf(m, qx - (Ps.lo[0] + (float)x0 * h));
        if (x1 < nx - 1) m = fminf(m, (Ps.lo[0] + (float)(x1 + 1) * h) - qx);
        if (y0 > 0) m = fminf(m, qy - (Ps.lo[1] + (float)y0 * h));
        if (y1 < ny - 1) m = fminf(m, (Ps.lo[1] + (float)(y1 + 1) * h) - qy);
        if (z0 > 0) m = fminf(m, qz - (Ps.lo[2] + (float)z0 * h));
        if (z1 < nz - 1) m = fminf(m, (Ps.lo[2] + (float)(z1 + 1) * h) - qz);
        if (m == INF) {
            done = true;   // the block is the whole grid
        } else {
            const float ms = m - slack;
            const float kth = top.kth(K);   // +inf while fewer than K candidates were seen
            done = ms > 0.f && kth <= ms * ms * (1.0f - 1e-5f);
        }
    }
    return done;
}

// Not certified: hand the query over to the full scan, unless it is bit-identical to the item's first
// far query (then it only needs a copy of that query's row).  Called by any subset of a warp's lanes.
__device__ __forceinline__ void register_overflow(const float *__restrict__ query, int Q, int b, int q, float qx, float qy,
                                                  float qz, QueryState *state_all, int *__restrict__ ovf_all)
{
    QueryState *Pw = state_all + b;
    int rep = *(volatile int *)&Pw->rep_q;            // stored as q+1 so that all-zero means 'none'
    if (rep == 0) rep = atomicCAS(&Pw->rep_q, 0, q + 1);
    rep -= 1;
    bool dup = false;
    if (rep != -1 && rep != q) {
        const float *rp = query + ((size_t)b * Q + rep) * 3;
        // float equality: -0.0 == +0.0 (hole pixels carry either sign) and their distances to
        // every support point are bit-identical; NaN never compares equal
        dup = (__ldg(rp) == qx) && (__ldg(rp + 1) == qy) && (__ldg(rp + 2) == qz);
    }
    // one atomic per group of lanes that got here together (hole pixels are spread over all warps)
    if (dup) {
        auto g = cooperative_groups::coalesced_threads();
        int base = 0;
        if (g.thread_rank() == 0) base = atomicAdd(&Pw->dup_count, (int)g.size());
        const int slot = g.shfl(base, 0) + (int)g.thread_rank();
        ovf_all[(size_t)b * Q + (Q - 1 - slot)] = q;
    } else {
        auto g = cooperative_groups::coalesced_threads();
        int base = 0;
        if (g.thread_rank() == 0) base = atomicAdd(&Pw->ovf_count, (int)g.size());
        const int slot = g.shfl(base, 0) + (int)g.thread_rank();
        ovf_all[(size_t)b * Q + slot] = q;
    }
}

template <int KCAP, typename IdxT, bool SELF>
__global__ void __launch_bounds__(128)
grid_search_kernel(const float *__restrict__ query, int S, int Q, int K,
                   const GridParams *__restrict__ params_all, const int *__restrict__ cursor_all,
                   size_t cursor_stride, const float4 *__restrict__ sorted_all,
                   IdxT *__restrict__ idx_out, QueryState *state_all, int *__restrict__ ovf_all)
{
    const int b = blockIdx.y;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= Q) return;
    const GridParams Ps = params_all[b];   // 64 B, same address for the whole CTA: L1 broadcast
    const int *cell_end = cursor_all + (size_t)b * cursor_stride;
    const float4 *sorted = sorted_all + (size_t)b * S;
    float qx, qy, qz;
    int q;   // row of the output this thread produces
    if (SELF) {  // queries are the support itself: walk them in cell order (coherent warps)
        const float4 me = sorted[t];
        qx = me.x;
        qy = me.y;
        qz = me.z;
        q = __float_as_int(me.w);
    } else {
        const float *qp = query + ((size_t)b * Q + t) * 3;
        qx = __ldg(qp);
        qy = __ldg(qp + 1);
        qz = __ldg(qp + 2);
        q = t;
    }
    TopK<KCAP> top;
    top.init();
    if (thread_search<KCAP>(qx, qy, qz, K, Ps, cell_end, sorted, top)) {
        IdxT *o = idx_out + ((size_t)b * Q + q) * K;
#pragma unroll
        for (int j = 0; j < KCAP; ++j)
            if (j < K) o[j] = (IdxT)top.i[j];
        return;
    }
    register_overflow(query, Q, b, q, qx, qy, qz, state_all, ovf_all);
}

// ------------------------------------------------------------------ E'. search, one WARP per query
// For 2 <= K <= 32.  The sorted top list lives across the lanes (lane j holds the j-th best) as
// one 64-bit key per entry, (distance bits << 32) | index: squared distances are non-negative so
// their bit patterns order like unsigned integers and ONE unsigned compare implements the total
// order (distance, index).  The cell rows of the block are looked up by the lanes in parallel
// (centre-out, rows that cannot beat the current K-th distance are skipped), their point ranges
// are flattened with a warp prefix sum so every batch of 32 candidates keeps all lanes busy (one
// coalesced 512-byte read), and candidates enter the list either one by one (shift-insert through
// shuffles) or, when many qualify, by a bitonic sort + merge.  When the block has to grow, only
// the new shell is scanned (new rows, and the new end cells of the old rows) and the list is
// kept.  Compared with one thread per query this removes the divergence between neighbouring
// queries and gives the small searches of the schedule (48 ... 3072 queries per frame) 32x more
// parallelism.
typedef unsigned long long key_t64;

__device__ __forceinline__ key_t64 make_key(float d, int i)
{
    return ((key_t64)__float_as_uint(d) << 32) | (unsigned)i;
}
__device__ __forceinline__ float key_dist(key_t64 k) { return __uint_as_float((unsigned)(k >> 32)); }

constexpr key_t64 KEY_EMPTY = 0x7f80000000000000ull;     // (+inf, index 0): what an unfilled slot reports
constexpr key_t64 KEY_INVALID = 0x7f8000007fffffffull;   // (+inf, INT_MAX): a lane without a candidate

__device__ __forceinline__ void warp_minmax(key_t64 &k, int j, bool keep_min)
{
    const key_t64 o = __shfl_xor_sync(0xffffffffu, k, j);
    if ((o < k) == keep_min) k = o;
}

// ascending bitonic sort of one key per lane
__device__ __forceinline__ void warp_sort(key_t64 &k, int lane)
{
#pragma unroll
    for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
        for (int j = kk >> 1; j > 0; j >>= 1) {
            const bool up = (lane & kk) == 0;
            warp_minmax(k, j, ((lane & j) == 0) == up);
        }
    }
}

// Offer one batch (one candidate key per lane, KEY_INVALID where none) to the lane-distributed
// sorted list `mine`; only candidates below the current K-th entry can matter.
__device__ __forceinline__ void warp_list_offer(key_t64 &mine, key_t64 cand, int K, int lane, bool &list_empty)
{
    const unsigned FULL = 0xffffffffu;
    if (list_empty) {   // first batch: sort it straight into the list
        warp_sort(cand, lane);
        mine = (cand < KEY_EMPTY) ? cand : KEY_EMPTY;
        list_empty = false;
        return;
    }
    const key_t64 thr = __shfl_sync(FULL, mine, K - 1);
    unsigned mask = __ballot_sync(FULL, cand < thr);
    if (__popc(mask) > 12) {
        // many newcomers: sort the batch, keep the 32 smallest of list U batch
        warp_sort(cand, lane);
        const key_t64 rev = __shfl_sync(FULL, cand, 31 - lane);
        if (rev < mine) mine = rev;
#pragma unroll
        for (int jj = 16; jj > 0; jj >>= 1) warp_minmax(mine, jj, (lane & jj) == 0);
        if (mine > KEY_EMPTY) mine = KEY_EMPTY;
    } else {
        while (mask) {   // shift-insert one candidate
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            const key_t64 x = __shfl_sync(FULL, cand, src);
            const key_t64 pred = __shfl_up_sync(FULL, mine, 1);
            if (x < mine) mine = (lane > 0 && x < pred) ? pred : x;   // mine sorts after x: shift or take x
        }
    }
}

// ------------------------------------------------------------------ E0. K = 1, ORGANISED queries: one warp per 8x4 pixel tile
// The p2r searches of the schedule ask for the nearest cloud point of every pixel of an image pyramid
// level (ycb_dataset.py:291-293, 305-308): 94 % of all K = 1 queries.  Neighbouring pixels are
// neighbouring points, so the 32 queries of an 8 x 4 pixel tile share ONE candidate set: the cells of
// the bounding box of their own cells, grown by one cell.  All lanes walk the same candidate list
// (warp-uniform addresses: one shared-memory broadcast per candidate, no divergence -- the thread-per-query
// kernel runs at 14.5 of 32 lanes active) and certify their own result against the distance to the box faces.
// The few lanes that cannot be certified (near depth discontinuities, box too large) are finished by the
// per-thread ring search; hole pixels (far outside the support) are marked and filled afterwards (below).

// Far queries of an ORGANISED K = 1 search (the hole pixels of an image level: ~10 % of the queries, all at the
// origin).  register_overflow() costs every tile a same-address atomicAdd on the item's dup counter -- 2400 warps
// per frame queue on one L2 atomic unit, half of the tile kernel's stall samples (ncu source page) -- and leaves the
// copies to the last CTA of the overflow pass.  Here a far query that equals the item's representative only writes
// the sentinel -1 into its result slot (no atomic, no list); grid_far_fill_kernel replaces the sentinels with the
// representative's answer after the overflow pass.  The representative itself and far queries that differ from it
// (rare) take the list path as before.
template <typename IdxT>
__device__ __forceinline__ void register_far_k1(const float *__restrict__ query, int Q, int b, int q, float qx, float qy,
                                                float qz, QueryState *state_all, int *__restrict__ ovf_all,
                                                IdxT *__restrict__ idx_out)
{
    QueryState *Pw = state_all + b;
    int rep = *(volatile int *)&Pw->rep_q;            // stored as q+1 so that all-zero means 'none'
    if (rep == 0) rep = atomicCAS(&Pw->rep_q, 0, q + 1);
    rep -= 1;
    bool dup = false;
    if (rep != -1 && rep != q) {
        const float *rp = query + ((size_t)b * Q + rep) * 3;
        dup = (__ldg(rp) == qx) && (__ldg(rp + 1) == qy) && (__ldg(rp + 2) == qz);
    }
    if (dup) {
        idx_out[(size_t)b * Q + q] = (IdxT)-1;
    } else {
        auto g = cooperative_groups::coalesced_threads();
        int base = 0;
        if (g.thread_rank() == 0) base = atomicAdd(&Pw->ovf_count, (int)g.size());
        const int slot = g.shfl(base, 0) + (int)g.thread_rank();
        ovf_all[(size_t)b * Q + slot] = q;
    }
}

// after the overflow pass: every sentinel of an item becomes the representative's (now final) answer
template <typename IdxT>
__global__ void __launch_bounds__(256)
grid_far_fill_kernel(int Q, const QueryState *__restrict__ state_all, IdxT *__restrict__ idx_out)
{
    const int b = blockIdx.y;
    const int rep = state_all[b].rep_q - 1;
    if (rep < 0) return;
    IdxT *o = idx_out + (size_t)b * Q;
    const IdxT v = o[rep];
    for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < Q; q += gridDim.x * blockDim.x)
        if (o[q] == (IdxT)-1) o[q] = v;
}

// The tile kernel.  Issue path kept lean (the first version spent two thirds of its ~1300 warp instructions per tile
// outside the distance arithmetic: 93 SASS instructions per 4 candidates in the walk, a third of them uniform-datapath
// bound checks; 190 for a staging round that always ran four binary-search sub-batches; integer divisions):
//   * the staged list is padded to a multiple of four with sentinel candidates at +inf (their key sorts after
//     every real candidate), so the walk has no per-candidate bound checks and its LDS.128 use immediate offsets
//     (109 instructions per 8 candidates);
//   * best-so-far is ONE 64-bit key (distance bits << 32 | index): the total order is a single unsigned compare;
//   * staging runs only as many 32-candidate sub-batches as there are candidates;
//   * tile and row coordinates come from exact float reciprocals instead of integer divisions when the tile count
//     allows it ((i + 0.5) * (1 / n) truncates to i / n whenever i + n < 2^22; `exact_div` selects the division).
// NW = warps (tiles) per CTA; one-warp CTAs need no CTA barrier around the retry list (measured 2.805 / 2.813 /
// 2.831 ms per pass for NW = 1 / 2 / 8).
template <typename IdxT, int NW>
__global__ void __launch_bounds__(NW * 32, 1024 / (NW * 32))
grid_search_k1_tile_kernel(const float *__restrict__ query, int S, int Q, int qw, int qh, int tiles_x, int n_tiles, int exact_div,
                            const GridParams *__restrict__ params_all, const int *__restrict__ cursor_all,
                            size_t cursor_stride, const float4 *__restrict__ sorted_all,
                            IdxT *__restrict__ idx_out, QueryState *state_all, int *__restrict__ ovf_all)
{
    constexpr int TW = 8, TH = 4;               // tile = 8 x 4 pixels
    constexpr int MAX_ROWS = 32, MAX_X = 8;     // widest shared box: 32 cell rows of up to 8 cells
    constexpr int TILE_CAND = 128;              // candidates staged per round and warp
    __shared__ float4 s_cand[NW][TILE_CAND];
    __shared__ int s_list[NW * 32];
    __shared__ int s_count;
    const unsigned FULL = 0xffffffffu;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int tile = blockIdx.x * NW + wid;
    const GridParams Ps = params_all[b];
    const int *cell_end = cursor_all + (size_t)b * cursor_stride;
    const float4 *sorted = sorted_all + (size_t)b * S;
    const float INF = __int_as_float(0x7f800000);
    if (threadIdx.x == 0) s_count = 0;
    if (NW > 1) __syncthreads();
    else __syncwarp();

    const int trow = exact_div ? tile / tiles_x : (int)(((float)tile + 0.5f) * (1.0f / (float)tiles_x));   // == tile / tiles_x
    const int px = (tile - trow * tiles_x) * TW + (lane & (TW - 1)), py = trow * TH + (lane >> 3);
    const bool inimg = tile < n_tiles && px < qw && py < qh;
    const int q = inimg ? py * qw + px : 0;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (inimg) {
        const float *qp = query + ((size_t)b * Q + q) * 3;
        qx = __ldg(qp);
        qy = __ldg(qp + 1);
        qz = __ldg(qp + 2);
    }
    const int nx = Ps.n[0], ny = Ps.n[1], nz = Ps.n[2];
    const float h = Ps.h, slack = Ps.slack;
    const float out = fmaxf(fmaxf(fmaxf(Ps.lo[0] - qx, qx - Ps.hi[0]), fmaxf(Ps.lo[1] - qy, qy - Ps.hi[1])),
                            fmaxf(Ps.lo[2] - qz, qz - Ps.hi[2]));
    // state: 0 answered, 1 finish with the ring search, 2 overflow (far from the support), 3 no query
    int state = !inimg ? 3 : ((out > (float)RMAX * h || !(qx == qx && qy == qy && qz == qz)) ? 2 : 1);
    const bool part = state == 1;
    const int cx = cell_of(qx, Ps.lo[0], Ps.inv_h, nx);
    const int cy = cell_of(qy, Ps.lo[1], Ps.inv_h, ny);
    const int cz = cell_of(qz, Ps.lo[2], Ps.inv_h, nz);
    const int big = 0x3fffffff;
    int X0 = __reduce_min_sync(FULL, part ? cx : big), X1 = __reduce_max_sync(FULL, part ? cx : -1);
    int Y0 = __reduce_min_sync(FULL, part ? cy : big), Y1 = __reduce_max_sync(FULL, part ? cy : -1);
    int Z0 = __reduce_min_sync(FULL, part ? cz : big), Z1 = __reduce_max_sync(FULL, part ? cz : -1);
    if (X1 >= 0) {   // warp-uniform: somebody takes part
        X0 = max(X0 - 1, 0); X1 = min(X1 + 1, nx - 1);
        Y0 = max(Y0 - 1, 0); Y1 = min(Y1 + 1, ny - 1);
        Z0 = max(Z0 - 1, 0); Z1 = min(Z1 + 1, nz - 1);
        const int by = Y1 - Y0 + 1, nrows = by * (Z1 - Z0 + 1);
        if (nrows <= MAX_ROWS && X1 - X0 + 1 <= MAX_X) {
            int beg = 0, end = 0;
            if (lane < nrows) {   // lane r looks up cell row r of the box
                const int rz = (int)(((float)lane + 0.5f) * (1.0f / (float)by));   // == lane / by (lane, by <= 32)
                const int row = ((Z0 + rz) * ny + (Y0 + lane - rz * by)) * nx;
                beg = (row + X0 > 0) ? __ldg(cell_end + row + X0 - 1) : 0;
                end = __ldg(cell_end + row + X1);
            }
            const int cnt = end - beg;
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(FULL, incl, o);
                if (lane >= o) incl += u;
            }
            const int total = __shfl_sync(FULL, incl, 31);
            const int excl = incl - cnt;
            float4 *stage = s_cand[wid];
            key_t64 best = KEY_EMPTY;   // (+inf, 0)
            for (int c0 = 0; c0 < total; c0 += TILE_CAND) {
                const int n = min(TILE_CAND, total - c0);
                const int n4 = (n + 3) & ~3;
                __syncwarp();
                for (int u0 = 0; u0 < n4; u0 += 32) {   // warp-uniform trip count
                    const int j = c0 + u0 + lane;
                    int seg = 0;   // number of rows whose inclusive count is <= j
#pragma unroll
                    for (int step = 16; step > 0; step >>= 1) {
                        const int v = __shfl_sync(FULL, incl, seg + step - 1);
                        if (v <= j) seg += step;
                    }
                    const int sb = __shfl_sync(FULL, beg, seg & 31), se = __shfl_sync(FULL, excl, seg & 31);
                    float4 c = make_float4(INF, INF, INF, __int_as_float(0x7fffffff));   // sentinel: sorts last
                    if (j < total) c = __ldg(sorted + sb + (j - se));
                    if (u0 + lane < n4) stage[u0 + lane] = c;
                }
                __syncwarp();
                for (int p = 0; p < n4; p += 4) {
                    float4 c[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) c[u] = stage[p + u];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const key_t64 k = make_key(ref_sqdist(qx, qy, qz, c[u].x, c[u].y, c[u].z), __float_as_int(c[u].w));
                        best = k < best ? k : best;
                    }
                }
            }
            if (part) {
                const float bd = key_dist(best);
                // distance to the nearest face of the box that still has cells behind it
                float m = INF;
                if (X0 > 0) m = fminf(m, qx - (Ps.lo[0] + (float)X0 * h));
                if (X1 < nx - 1) m = fminf(m, (Ps.lo[0] + (float)(X1 + 1) * h) - qx);
                if (Y0 > 0) m = fminf(m, qy - (Ps.lo[1] + (float)Y0 * h));
                if (Y1 < ny - 1) m = fminf(m, (Ps.lo[1] + (float)(Y1 + 1) * h) - qy);
                if (Z0 > 0) m = fminf(m, qz - (Ps.lo[2] + (float)Z0 * h));
                if (Z1 < nz - 1) m = fminf(m, (Ps.lo[2] + (float)(Z1 + 1) * h) - qz);
                const float ms = m - slack;
                const bool ok = (m == INF) ? (bd < INF || S == 0) : (ms > 0.f && bd <= ms * ms * (1.0f - 1e-5f));
                if (ok) {
                    idx_out[(size_t)b * Q + q] = (IdxT)(unsigned)(best & 0xffffffffu);
                    state = 0;
                }
            }
        }
    }
    // ---- the uncertified queries of the CTA, compacted, finished by the per-thread ring search
    if (state == 1) s_list[atomicAdd(&s_count, 1)] = q;
    if (NW > 1) __syncthreads();   // a CTA of one warp holds no other warp back while a lane finishes its ring search
    else __syncwarp();
    const int n_retry = s_count;
    int q2 = -1;
    float rx = 0.f, ry = 0.f, rz = 0.f;
    bool retry_failed = false;
    if ((int)threadIdx.x < n_retry) {
        q2 = s_list[threadIdx.x];
        const float *qp = query + ((size_t)b * Q + q2) * 3;
        rx = __ldg(qp);
        ry = __ldg(qp + 1);
        rz = __ldg(qp + 2);
        TopK<1> top;
        top.init();
        if (thread_search<1>(rx, ry, rz, 1, Ps, cell_end, sorted, top))
            idx_out[(size_t)b * Q + q2] = (IdxT)top.i[0];
        else
            retry_failed = true;
    }
    if (retry_failed) register_overflow(query, Q, b, q2, rx, ry, rz, state_all, ovf_all);
    if (state == 2) register_far_k1<IdxT>(query, Q, b, q, qx, qy, qz, state_all, ovf_all, idx_out);
}

// ------------------------------------------------------------------ E'. (continued) the warp-per-query kernel
template <typename IdxT, bool SELF>
__global__ void __launch_bounds__(256, 5)
grid_search_warp_kernel(const float *__restrict__ query, int S, int Q, int K,
                        const GridParams *__restrict__ params_all, const int *__restrict__ cursor_all,
                        size_t cursor_stride, const float4 *__restrict__ sorted_all,
                        IdxT *__restrict__ idx_out, QueryState *state_all, int *__restrict__ ovf_all)
{
    const unsigned FULL = 0xffffffffu;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= Q) return;   // warp-uniform
    const GridParams Ps = params_all[b];
    const int *cell_end = cursor_all + (size_t)b * cursor_stride;
    const float4 *sorted = sorted_all + (size_t)b * S;
    float qx, qy, qz;
    int q;
    if (SELF) {
        const float4 me = __ldg(sorted + t);
        qx = me.x;
        qy = me.y;
        qz = me.z;
        q = __float_as_int(me.w);
    } else {
        const float *qp = query + ((size_t)b * Q + t) * 3;
        qx = __ldg(qp);
        qy = __ldg(qp + 1);
        qz = __ldg(qp + 2);
        q = t;
    }
    const int nx = Ps.n[0], ny = Ps.n[1], nz = Ps.n[2];
    const float h = Ps.h, slack = Ps.slack;
    const int cx = cell_of(qx, Ps.lo[0], Ps.inv_h, nx);
    const int cy = cell_of(qy, Ps.lo[1], Ps.inv_h, ny);
    const int cz = cell_of(qz, Ps.lo[2], Ps.inv_h, nz);
    const float INF = __int_as_float(0x7f800000);
    const float out = fmaxf(fmaxf(fmaxf(Ps.lo[0] - qx, qx - Ps.hi[0]), fmaxf(Ps.lo[1] - qy, qy - Ps.hi[1])),
                            fmaxf(Ps.lo[2] - qz, qz - Ps.hi[2]));

    auto margin = [&](int r) {   // distance to the nearest face of block r that has cells behind it
        float m = INF;
        if (cx - r > 0) m = fminf(m, qx - (Ps.lo[0] + (float)(cx - r) * h));
        if (cx + r < nx - 1) m = fminf(m, (Ps.lo[0] + (float)(cx + r + 1) * h) - qx);
        if (cy - r > 0) m = fminf(m, qy - (Ps.lo[1] + (float)(cy - r) * h));
        if (cy + r < ny - 1) m = fminf(m, (Ps.lo[1] + (float)(cy + r + 1) * h) - qy);
        if (cz - r > 0) m = fminf(m, qz - (Ps.lo[2] + (float)(cz - r) * h));
        if (cz + r < nz - 1) m = fminf(m, (Ps.lo[2] + (float)(cz + r + 1) * h) - qz);
        return m;
    };

    key_t64 mine = KEY_EMPTY;   // lane j: j-th best so far
    bool list_empty = true;
    bool done = false;
    int r = (out > (float)RMAX * h) ? RMAX + 1 : 1;
    int e_prev = 0;                  // rows [0, e_prev) of the table were scanned over cells [px0, px1]
    int px0 = 0, px1 = -1;
    while (r <= RMAX) {
        const int x0 = max(cx - r, 0), x1 = min(cx + r, nx - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, ny - 1);
        const int z0 = max(cz - r, 0), z1 = min(cz + r, nz - 1);
        const int e_end = (2 * r + 1) * (2 * r + 1);
        // segments: two per old row (its new end cells), one per new row (all its cells)
        const int nseg = 2 * e_prev + (e_end - e_prev);
        for (int s0 = 0; s0 < nseg; s0 += 32) {
            const float kth_now = key_dist(__shfl_sync(FULL, mine, K - 1));   // +inf until K were seen
            const int sidx = s0 + lane;
            int beg = 0, end = 0;
            if (sidx < nseg) {
                const bool old = sidx < 2 * e_prev;
                const int e = old ? (sidx >> 1) : (sidx - e_prev);
                const int z = cz + kRowOrder[e][0], y = cy + kRowOrder[e][1];
                int a = x0, c = x1;   // cell range of this segment
                if (old) {
                    if (sidx & 1) a = px1 + 1;   // right end
                    else c = px0 - 1;            // left end
                }
                if (z >= z0 && z <= z1 && y >= y0 && y <= y1 && a <= c) {
                    // rows that cannot hold anything closer than the current K-th best are skipped
                    const float dmin2 = slab_dist2(qy, Ps.lo[1], h, y, slack) + slab_dist2(qz, Ps.lo[2], h, z, slack);
                    if (!(dmin2 > kth_now)) {
                        const int row = (z * ny + y) * nx;
                        beg = (row + a > 0) ? __ldg(cell_end + row + a - 1) : 0;
                        end = __ldg(cell_end + row + c);
                    }
                }
            }
            const int cnt = end - beg;
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(FULL, incl, o);
                if (lane >= o) incl += u;
            }
            const int total = __shfl_sync(FULL, incl, 31);
            const int excl = incl - cnt;
            for (int j0 = 0; j0 < total; j0 += 32) {
                const int j = j0 + lane;
                int seg = 0;   // number of segments whose inclusive count is <= j
#pragma unroll
                for (int step = 16; step > 0; step >>= 1) {
                    const int v = __shfl_sync(FULL, incl, seg + step - 1);
                    if (v <= j) seg += step;
                }
                const int sb = __shfl_sync(FULL, beg, seg);
                const int se = __shfl_sync(FULL, excl, seg);
                key_t64 cand = KEY_INVALID;
                if (j < total) {
                    const float4 c = __ldg(sorted + sb + (j - se));
                    cand = make_key(ref_sqdist(qx, qy, qz, c.x, c.y, c.z), __float_as_int(c.w));
                }
                warp_list_offer(mine, cand, K, lane, list_empty);
            }
        }
        e_prev = e_end;
        px0 = x0;
        px1 = x1;
        const float m = margin(r);
        const float kth = key_dist(__shfl_sync(FULL, mine, K - 1));
        if (m == INF) {
            done = true;
            break;
        }
        const float ms = m - slack;
        if (ms > 0.f && kth <= ms * ms * (1.0f - 1e-5f)) {
            done = true;
            break;
        }
        // next ring: the K-th distance found so far bounds the true one, so jump to the first
        // block whose margin covers it
        int rn = r + 1;
        if (kth < INF) {
            const float need = sqrtf(kth) * (1.0f + 1e-4f) + slack;
            while (rn <= RMAX && margin(rn) < need) ++rn;
        }
        r = rn;
    }
    if (done) {
        if (lane < K) idx_out[((size_t)b * Q + q) * K + lane] = (IdxT)(unsigned)(mine & 0xffffffffu);
        return;
    }
    if (lane == 0) {
        QueryState *Pw = state_all + b;
        const int rep = atomicCAS(&Pw->rep_q, 0, q + 1) - 1;   // stored as q+1: all-zero state = 'none'
        bool dup = false;
        if (rep != -1 && rep != q) {
            const float *rp = query + ((size_t)b * Q + rep) * 3;
            dup = (__ldg(rp) == qx) && (__ldg(rp + 1) == qy) && (__ldg(rp + 2) == qz);
        }
        if (dup) {
            const int slot = atomicAdd(&Pw->dup_count, 1);
            ovf_all[(size_t)b * Q + (Q - 1 - slot)] = q;
        } else {
            const int slot = atomicAdd(&Pw->ovf_count, 1);
            ovf_all[(size_t)b * Q + slot] = q;
        }
    }
}

// ------------------------------------------------------------------ E''. search, HALF a warp per query (K <= 16)
// Same algorithm as grid_search_warp_kernel with the sorted list spread over the 16 lanes of a
// half-warp, so one warp answers two neighbouring queries at once: the control flow (segment set-up,
// prefix sums, binary searches, the ring logic) is issued once for both -- the warp-per-query kernel
// spends ~750 warp instructions per query, nine tenths of it such bookkeeping (ncu source page), so
// sharing it nearly halves the cost per query.  Everything that differs between the two queries is
// carried per lane group (ring, scanned block, done flag) and the loops run while EITHER group has
// work; a group that is finished keeps executing with empty segments.
template <int W>
__device__ __forceinline__ void group_minmax(key_t64 &k, int j, bool keep_min)
{
    const key_t64 o = __shfl_xor_sync(0xffffffffu, k, j, W);
    if ((o < k) == keep_min) k = o;
}

template <int W>
__device__ __forceinline__ void group_sort(key_t64 &k, int sub)   // ascending bitonic sort inside a group of W lanes
{
#pragma unroll
    for (int kk = 2; kk <= W; kk <<= 1) {
#pragma unroll
        for (int j = kk >> 1; j > 0; j >>= 1) {
            const bool up = (sub & kk) == 0;
            group_minmax<W>(k, j, ((sub & j) == 0) == up);
        }
    }
}

template <typename IdxT, bool SELF, int W>
__global__ void __launch_bounds__(256, 5)
grid_search_group_kernel(const float *__restrict__ query, int S, int Q, int K,
                         const GridParams *__restrict__ params_all, const int *__restrict__ cursor_all,
                         size_t cursor_stride, const float4 *__restrict__ sorted_all,
                         IdxT *__restrict__ idx_out, QueryState *state_all, int *__restrict__ ovf_all)
{
    constexpr int G = 32 / W;                       // queries per warp
    const unsigned FULL = 0xffffffffu;
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, sub = lane & (W - 1), grp = lane / W;
    const int t = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * G + grp;
    if ((blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * G >= Q) return;   // warp-uniform
    const bool valid = t < Q;                       // the last warp may hold fewer than G queries
    const int tq = valid ? t : Q - 1;
    const GridParams Ps = params_all[b];
    const int *cell_end = cursor_all + (size_t)b * cursor_stride;
    const float4 *sorted = sorted_all + (size_t)b * S;
    float qx, qy, qz;
    int q;
    if (SELF) {
        const float4 me = __ldg(sorted + tq);
        qx = me.x;
        qy = me.y;
        qz = me.z;
        q = __float_as_int(me.w);
    } else {
        const float *qp = query + ((size_t)b * Q + tq) * 3;
        qx = __ldg(qp);
        qy = __ldg(qp + 1);
        qz = __ldg(qp + 2);
        q = tq;
    }
    const int nx = Ps.n[0], ny = Ps.n[1], nz = Ps.n[2];
    const float h = Ps.h, slack = Ps.slack;
    const int cx = cell_of(qx, Ps.lo[0], Ps.inv_h, nx);
    const int cy = cell_of(qy, Ps.lo[1], Ps.inv_h, ny);
    const int cz = cell_of(qz, Ps.lo[2], Ps.inv_h, nz);
    const float INF = __int_as_float(0x7f800000);
    const float out = fmaxf(fmaxf(fmaxf(Ps.lo[0] - qx, qx - Ps.hi[0]), fmaxf(Ps.lo[1] - qy, qy - Ps.hi[1])),
                            fmaxf(Ps.lo[2] - qz, qz - Ps.hi[2]));
    auto margin = [&](int r) {   // distance to the nearest face of block r that has cells behind it
        float m = INF;
        if (cx - r > 0) m = fminf(m, qx - (Ps.lo[0] + (float)(cx - r) * h));
        if (cx + r < nx - 1) m = fminf(m, (Ps.lo[0] + (float)(cx + r + 1) * h) - qx);
        if (cy - r > 0) m = fminf(m, qy - (Ps.lo[1] + (float)(cy - r) * h));
        if (cy + r < ny - 1) m = fminf(m, (Ps.lo[1] + (float)(cy + r + 1) * h) - qy);
        if (cz - r > 0) m = fminf(m, qz - (Ps.lo[2] + (float)(cz - r) * h));
        if (cz + r < nz - 1) m = fminf(m, (Ps.lo[2] + (float)(cz + r + 1) * h) - qz);
        return m;
    };

    key_t64 mine = KEY_EMPTY;        // lane sub of a group: its sub-th best so far
    bool done = false;               // group-uniform
    int r = (out > (float)RMAX * h) ? RMAX + 1 : 1;
    bool active = valid && r <= RMAX;   // group-uniform: this group still scans rings
    int e_prev = 0, px0 = 0, px1 = -1;
    while (__any_sync(FULL, active)) {
        const int x0 = max(cx - r, 0), x1 = min(cx + r, nx - 1);
        const int y0 = max(cy - r, 0), y1 = min(cy + r, ny - 1);
        const int z0 = max(cz - r, 0), z1 = min(cz + r, nz - 1);
        const int e_end = (2 * r + 1) * (2 * r + 1);
        // segments: two per old row (its new end cells), one per new row (all its cells)
        const int nseg = active ? 2 * e_prev + (e_end - e_prev) : 0;
        for (int s0 = 0; __any_sync(FULL, s0 < nseg); s0 += W) {
            const float kth_now = key_dist(__shfl_sync(FULL, mine, K - 1, W));   // +inf until K were seen
            const int sidx = s0 + sub;
            int beg = 0, end = 0;
            if (sidx < nseg) {
                const bool old = sidx < 2 * e_prev;
                const int e = old ? (sidx >> 1) : (sidx - e_prev);
                const int z = cz + kRowOrder[e][0], y = cy + kRowOrder[e][1];
                int a = x0, c = x1;   // cell range of this segment
                if (old) {
                    if (sidx & 1) a = px1 + 1;   // right end
                    else c = px0 - 1;            // left end
                }
                if (z >= z0 && z <= z1 && y >= y0 && y <= y1 && a <= c) {
                    // rows that cannot hold anything closer than the current K-th best are skipped
                    const float dmin2 = slab_dist2(qy, Ps.lo[1], h, y, slack) + slab_dist2(qz, Ps.lo[2], h, z, slack);
                    if (!(dmin2 > kth_now)) {
                        const int row = (z * ny + y) * nx;
                        beg = (row + a > 0) ? __ldg(cell_end + row + a - 1) : 0;
                        end = __ldg(cell_end + row + c);
                    }
                }
            }
            const int cnt = end - beg;
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < W; o <<= 1) {
                const int u = __shfl_up_sync(FULL, incl, o, W);
                if (sub >= o) incl += u;
            }
            const int total = __shfl_sync(FULL, incl, W - 1, W);
            const int excl = incl - cnt;
            for (int j0 = 0; __any_sync(FULL, j0 < total); j0 += W) {
                const int j = j0 + sub;
                int seg = 0;   // number of segments of my group whose inclusive count is <= j
#pragma unroll
                for (int step = W / 2; step > 0; step >>= 1) {
                    const int v = __shfl_sync(FULL, incl, seg + step - 1, W);
                    if (v <= j) seg += step;
                }
                const int sb = __shfl_sync(FULL, beg, seg, W);
                const int se = __shfl_sync(FULL, excl, seg, W);
                key_t64 cand = KEY_INVALID;
                if (j < total) {
                    const float4 c = __ldg(sorted + sb + (j - se));
                    cand = make_key(ref_sqdist(qx, qy, qz, c.x, c.y, c.z), __float_as_int(c.w));
                }
                // ---- offer the batch to the group's list; only candidates below its K-th entry matter
                const key_t64 thr = __shfl_sync(FULL, mine, K - 1, W);
                const unsigned ball = __ballot_sync(FULL, cand < thr);
                unsigned mask = (W == 32) ? ball : ((ball >> (W * grp)) & ((1u << W) - 1u));
                if (__any_sync(FULL, __popc(mask) > (3 * W) / 8)) {
                    // many newcomers somewhere in the warp: sort the batch, keep the W smallest of list U batch
                    group_sort<W>(cand, sub);
                    const key_t64 rev = __shfl_sync(FULL, cand, W - 1 - sub, W);
                    if (rev < mine) mine = rev;
#pragma unroll
                    for (int jj = W / 2; jj > 0; jj >>= 1) group_minmax<W>(mine, jj, (sub & jj) == 0);
                    if (mine > KEY_EMPTY) mine = KEY_EMPTY;
                } else {
                    while (__any_sync(FULL, mask != 0)) {   // shift-insert one candidate per group
                        const int src = mask ? __ffs(mask) - 1 : 0;
                        key_t64 x = __shfl_sync(FULL, cand, src, W);
                        if (!mask) x = KEY_INVALID;         // this group has nothing left: a no-op insert
                        mask &= mask - 1;
                        const key_t64 pred = __shfl_up_sync(FULL, mine, 1, W);
                        if (x < mine) mine = (sub > 0 && x < pred) ? pred : x;   // mine sorts after x: shift or take x
                    }
                }
            }
        }
        const float kth = key_dist(__shfl_sync(FULL, mine, K - 1, W));   // all lanes: shuffles stay warp-uniform
        if (active) {
            e_prev = e_end;
            px0 = x0;
            px1 = x1;
            const float m = margin(r);
            if (m == INF) {
                done = true;
                active = false;
            } else {
                const float ms = m - slack;
                if (ms > 0.f && kth <= ms * ms * (1.0f - 1e-5f)) {
                    done = true;
                    active = false;
                } else {
                    // next ring: the K-th distance found so far bounds the true one, so jump to the
                    // first block whose margin covers it
                    int rn = r + 1;
                    if (kth < INF) {
                        const float need = sqrtf(kth) * (1.0f + 1e-4f) + slack;
                        while (rn <= RMAX && margin(rn) < need) ++rn;
                    }
                    r = rn;
                    active = r <= RMAX;
                }
            }
        }
    }
    if (!valid) return;
    if (done) {
        if (sub < K) idx_out[((size_t)b * Q + q) * K + sub] = (IdxT)(unsigned)(mine & 0xffffffffu);
        return;
    }
    if (sub == 0) {
        QueryState *Pw = state_all + b;
        const int rep = atomicCAS(&Pw->rep_q, 0, q + 1) - 1;   // stored as q+1: all-zero state = 'none'
        bool dup = false;
        if (rep != -1 && rep != q) {
            const float *rp = query + ((size_t)b * Q + rep) * 3;
            dup = (__ldg(rp) == qx) && (__ldg(rp + 1) == qy) && (__ldg(rp + 2) == qz);
        }
        if (dup) {
            const int slot = atomicAdd(&Pw->dup_count, 1);
            ovf_all[(size_t)b * Q + (Q - 1 - slot)] = q;
        } else {
            const int slot = atomicAdd(&Pw->ovf_count, 1);
            ovf_all[(size_t)b * Q + slot] = q;
        }
    }
}

// ------------------------------------------------------------------ F. overflow: tiled full scan
template <int KCAP, int THREADS, int TILE, typename IdxT>
__global__ void __launch_bounds__(THREADS)
grid_overflow_kernel(const float *__restrict__ support, const float *__restrict__ query, int S,
                     int Q, int K, const QueryState *__restrict__ state_all,
                     const int *__restrict__ ovf_all, IdxT *__restrict__ idx_out)
{
    const int b = blockIdx.y;
    const int count = state_all[b].ovf_count;
    __shared__ float4 tile[TILE];
    const float *sup = support + (size_t)b * S * 3;
    for (int first = blockIdx.x * THREADS; first < count; first += gridDim.x * THREADS) {  // CTA-uniform
        const int t = first + threadIdx.x;
        const bool active = t < count;
        int q = 0;
        float qx = 0.f, qy = 0.f, qz = 0.f;
        if (active) {
            q = ovf_all[(size_t)b * Q + t];
            const float *qp = query + ((size_t)b * Q + q) * 3;
            qx = __ldg(qp);
            qy = __ldg(qp + 1);
            qz = __ldg(qp + 2);
        }
        TopK<KCAP> top;
        top.init();
        for (int s0 = 0; s0 < S; s0 += TILE) {
            const int n = min(TILE, S - s0);
            __syncthreads();
            const float *src = sup + (size_t)s0 * 3;
            for (int i = threadIdx.x; i < 3 * n; i += THREADS)
                reinterpret_cast<float *>(tile)[(i / 3) * 4 + (i % 3)] = __ldg(src + i);
            __syncthreads();
            if (active) {
#pragma unroll 4
                for (int i = 0; i < n; ++i) {
                    const float4 p = tile[i];
                    const float d = ref_sqdist(qx, qy, qz, p.x, p.y, p.z);
                    if (d < top.worst()) top.push_ordered(d, s0 + i);
                }
            }
        }
        if (active) {
            IdxT *o = idx_out + ((size_t)b * Q + q) * K;
#pragma unroll
            for (int j = 0; j < KCAP; ++j)
                if (j < K) o[j] = (IdxT)top.i[j];
        }
    }
}

// ------------------------------------------------------------------ F'. overflow + duplicate rows, one CTA per query (K <= 32)
// Same full scan, but the eight warps of a CTA split the support, each building the lane-distributed
// sorted list of grid_search_warp_kernel; warp 0 merges the eight lists.  A handful of far queries
// (typically one per frame once duplicates are folded) no longer costs a serial walk over the whole
// support.  The last CTA of a batch item to finish then copies the representative's row to the
// queries that were equal to it (fused: no separate launch).
template <typename IdxT>
__global__ void __launch_bounds__(256)
grid_overflow_warp_kernel(const float *__restrict__ support, const float *__restrict__ query, int S,
                          int Q, int K, QueryState *state_all, const int *__restrict__ ovf_all,
                          IdxT *__restrict__ idx_out)
{
    __shared__ key_t64 lists[8][32];
    __shared__ int last_flag;
    const int b = blockIdx.y;
    const int count = state_all[b].ovf_count;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const float *sup = support + (size_t)b * S * 3;
    for (int t = blockIdx.x; t < count; t += gridDim.x) {   // CTA-uniform
        const int q = ovf_all[(size_t)b * Q + t];
        const float *qp = query + ((size_t)b * Q + q) * 3;
        const float qx = __ldg(qp), qy = __ldg(qp + 1), qz = __ldg(qp + 2);
        key_t64 mine = KEY_EMPTY;
        bool list_empty = true;
        for (int s0 = wid * 32; s0 < S; s0 += 8 * 32) {
            const int sI = s0 + lane;
            key_t64 cand = KEY_INVALID;
            if (sI < S)
                cand = make_key(ref_sqdist(qx, qy, qz, __ldg(sup + (size_t)sI * 3), __ldg(sup + (size_t)sI * 3 + 1),
                                           __ldg(sup + (size_t)sI * 3 + 2)), sI);
            warp_list_offer(mine, cand, K, lane, list_empty);
        }
        lists[wid][lane] = mine;
        __syncthreads();
        if (wid == 0) {
            list_empty = false;
            for (int w = 1; w < 8; ++w) warp_list_offer(mine, lists[w][lane], K, lane, list_empty);
            if (lane < K) idx_out[((size_t)b * Q + q) * K + lane] = (IdxT)(unsigned)(mine & 0xffffffffu);
        }
        __syncthreads();
    }
    // ---- rows of the queries equal to the representative far query: done by the last CTA of this item
    const int dups = state_all[b].dup_count;
    if (dups == 0) return;   // CTA-uniform
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last_flag = (atomicAdd(&state_all[b].pad, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (!last_flag) return;
    __threadfence();
    const int rep = state_all[b].rep_q - 1;
    const IdxT *src = idx_out + ((size_t)b * Q + rep) * K;
    for (int t = threadIdx.x; t < dups * K; t += blockDim.x) {
        const int q = ovf_all[(size_t)b * Q + (Q - 1 - t / K)];
        idx_out[((size_t)b * Q + q) * K + t % K] = __ldcg(src + t % K);
    }
}

// ------------------------------------------------------------------ G. rows of duplicate far queries
template <typename IdxT>
__global__ void __launch_bounds__(256)
grid_dup_copy_kernel(int Q, int K, const QueryState *__restrict__ state_all,
                     const int *__restrict__ ovf_all, IdxT *__restrict__ idx_out)
{
    const int b = blockIdx.y;
    const int count = state_all[b].dup_count;
    const int rep = state_all[b].rep_q - 1;
    if (count == 0) return;
    const IdxT *src = idx_out + ((size_t)b * Q + rep) * K;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < count * K; t += gridDim.x * blockDim.x) {
        const int q = ovf_all[(size_t)b * Q + (Q - 1 - t / K)];
        idx_out[((size_t)b * Q + q) * K + t % K] = src[t % K];
    }
}

// ------------------------------------------------------------------ H. nearest point of a row-PREFIX subset, read off a self search
// The schedule asks, per cloud level i, for the nearest level-(i+1) point of every level-i point (cld_interp_idx{i},
// ycb_dataset.py:280-282).  Level i+1 is the first N_{i+1} rows of level i (:278) and the K-neighbour self search of
// level i (cld_nei_idx{i}) has just been computed: its rows are sorted by the total order (distance, index) over ALL
// level-i points, so the first entry of a row with index < N_{i+1} IS the nearest subset point under the same total
// order -- every subset point that is not in the row sorts after the row's last entry.  Only rows without such an
// entry (0.75^16 = 1 % of the queries when the subset is a random quarter) need a search: they go to the full-scan
// pass (one CTA per query).  No grid is needed.
template <typename IdxT>
__global__ void __launch_bounds__(256)
subset_nn_from_knn_kernel(const IdxT *__restrict__ knn, int Q, int KL, int S, IdxT *__restrict__ idx_out,
                          QueryState *state_all, int *__restrict__ ovf_all)
{
    const int b = blockIdx.y;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    const IdxT *row = knn + ((size_t)b * Q + q) * KL;
    const int kl = min(KL, Q);   // a level smaller than KL leaves (+inf, 0) fillers behind its Q real entries
    for (int j = 0; j < kl; ++j) {
        const IdxT v = __ldg(row + j);
        if (v >= 0 && v < (IdxT)S) {
            idx_out[(size_t)b * Q + q] = v;
            return;
        }
    }
    auto g = cooperative_groups::coalesced_threads();
    int base = 0;
    if (g.thread_rank() == 0) base = atomicAdd(&state_all[b].ovf_count, (int)g.size());
    ovf_all[(size_t)b * Q + g.shfl(base, 0) + (int)g.thread_rank()] = q;
}

// support = the first S rows of `query` in every batch item ([B,S,3] contiguous copy), knn = the exact K-neighbour
// self search of `query` ([B,Q,KL], rows sorted by (distance, index)); idx_out [B,Q,1]
int knn_subset_nn_from_knn(const float *support, const float *query, int64_t B, int64_t S, int64_t Q, const void *knn,
                           int KL, void *idx_out, int idx_is_i64, void *scratch, size_t scratch_bytes, cudaStream_t st)
{
    QueryScratch qs = carve_query(scratch, B, Q);
    if (!scratch || scratch_bytes < qs.bytes) {
        set_error("knn subset search: %zu bytes of scratch required, %zu given", qs.bytes, scratch_bytes);
        return FFB6D_ERR_WORKSPACE;
    }
    FFB6D_CUDA(cudaMemsetAsync(qs.state, 0, (size_t)B * sizeof(QueryState), st));
    dim3 grid((unsigned)ceil_div(Q, 256), (unsigned)B);
    const int64_t per_item = std::max<int64_t>(1, 4 * num_sms() / B);
    dim3 ogrid((unsigned)std::min<int64_t>(Q, per_item), (unsigned)B);
    if (idx_is_i64) {
        subset_nn_from_knn_kernel<long long><<<grid, 256, 0, st>>>((const long long *)knn, (int)Q, KL, (int)S,
                                                                   (long long *)idx_out, qs.state, qs.ovf);
        FFB6D_LAUNCH_OK("subset_nn_from_knn_kernel");
        grid_overflow_warp_kernel<long long><<<ogrid, 256, 0, st>>>(support, query, (int)S, (int)Q, 1, qs.state, qs.ovf,
                                                                    (long long *)idx_out);
    } else {
        subset_nn_from_knn_kernel<int><<<grid, 256, 0, st>>>((const int *)knn, (int)Q, KL, (int)S, (int *)idx_out, qs.state,
                                                             qs.ovf);
        FFB6D_LAUNCH_OK("subset_nn_from_knn_kernel");
        grid_overflow_warp_kernel<int><<<ogrid, 256, 0, st>>>(support, query, (int)S, (int)Q, 1, qs.state, qs.ovf,
                                                              (int *)idx_out);
    }
    FFB6D_LAUNCH_OK("grid_overflow_warp_kernel");
    return FFB6D_OK;
}

// ------------------------------------------------------------------ host
// cell-size knobs: defaults from the environment (read once, common.cuh Env), overridable by
// ffb6d_knn_grid_tune* (tools/tune_grid.py); results never depend on them
static bool g_force_thread_search = false;
static float g_cell_scale = 1.0f;
static float g_cell_scale_k1 = 2.5f;   // grids built for K = 1 searches (measured optimum 2 ... 2.8)
static int g_quantile = 17;
static std::atomic<bool> g_env_read{false};

static void read_env()
{
    if (g_env_read.load(std::memory_order_acquire)) return;
    const Env &e = env();
    if (e.grid_scale > 0.f) g_cell_scale = e.grid_scale;
    if (e.grid_scale_k1 > 0.f) g_cell_scale_k1 = e.grid_scale_k1;
    g_force_thread_search = e.grid_thread_search;
    g_quantile = e.grid_quantile;
    g_env_read.store(true, std::memory_order_release);
}

void knn_grid_tune(float cell_scale, int quantile)
{
    read_env();
    if (cell_scale > 0.f) g_cell_scale = cell_scale;
    if (quantile >= 0) g_quantile = std::min(31, quantile);
}

void knn_grid_tune_k1(float cell_scale_k1)
{
    read_env();
    if (cell_scale_k1 > 0.f) g_cell_scale_k1 = cell_scale_k1;
}

template <int KCAP, typename IdxT>
static int launch_search(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                         int K, void *idx_out, const GridStore &w, const QueryScratch &qs, int64_t query_width,
                         cudaStream_t st)
{
    const bool self = (support == query) && (S == Q);
    const bool warp = K >= 2 && K <= 32 && !g_force_thread_search;
    FFB6D_CUDA(cudaMemsetAsync(qs.state, 0, (size_t)B * sizeof(QueryState), st));
    const bool organised = K == 1 && !self && query_width >= 8 && Q % query_width == 0 && Q / query_width >= 4 &&
                           !g_force_thread_search;
    bool far_sentinels = false;
    if (organised) {   // queries are an image: one warp per 8x4 pixel tile
        const int64_t tiles_x = ceil_div(query_width, 8), tiles = tiles_x * ceil_div(Q / query_width, 4);
        far_sentinels = true;
        grid_search_k1_tile_kernel<IdxT, 1><<<dim3((unsigned)tiles, (unsigned)B), 32, 0, st>>>(
            query, (int)S, (int)Q, (int)query_width, (int)(Q / query_width), (int)tiles_x, (int)tiles,
            (int)(tiles + tiles_x >= 4000000), w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
    } else if (warp && K <= 16) {   // half a warp per query
        dim3 ggrid((unsigned)ceil_div(Q, 16), (unsigned)B);
        if (self)
            grid_search_group_kernel<IdxT, true, 16><<<ggrid, 256, 0, st>>>(
                query, (int)S, (int)Q, K, w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
        else
            grid_search_group_kernel<IdxT, false, 16><<<ggrid, 256, 0, st>>>(
                query, (int)S, (int)Q, K, w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
    } else if (warp) {
        dim3 wgrid((unsigned)ceil_div(Q, 8), (unsigned)B);
        if (self)
            grid_search_warp_kernel<IdxT, true><<<wgrid, 256, 0, st>>>(
                query, (int)S, (int)Q, K, w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
        else
            grid_search_warp_kernel<IdxT, false><<<wgrid, 256, 0, st>>>(
                query, (int)S, (int)Q, K, w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
    } else {
        dim3 grid((unsigned)ceil_div(Q, 128), (unsigned)B);
        if (self)
            grid_search_kernel<KCAP, IdxT, true><<<grid, 128, 0, st>>>(
                query, (int)S, (int)Q, K, w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
        else
            grid_search_kernel<KCAP, IdxT, false><<<grid, 128, 0, st>>>(
                query, (int)S, (int)Q, K, w.params, w.cursor, w.maxc, w.sorted, (IdxT *)idx_out, qs.state, qs.ovf);
    }
    FFB6D_LAUNCH_OK("grid_search_kernel");
    const int64_t per_item = std::max<int64_t>(1, 4 * num_sms() / B);
    if (K <= 32) {
        dim3 ogrid((unsigned)std::min<int64_t>(Q, per_item), (unsigned)B);
        grid_overflow_warp_kernel<IdxT><<<ogrid, 256, 0, st>>>(support, query, (int)S, (int)Q, K, qs.state,
                                                               qs.ovf, (IdxT *)idx_out);
        FFB6D_LAUNCH_OK("grid_overflow_warp_kernel");
        if (far_sentinels) {   // the lean tile kernel marked the duplicates of the far representative with -1
            dim3 fgrid((unsigned)std::min<int64_t>(ceil_div(Q, 1024), 64), (unsigned)B);
            grid_far_fill_kernel<IdxT><<<fgrid, 256, 0, st>>>((int)Q, qs.state, (IdxT *)idx_out);
            FFB6D_LAUNCH_OK("grid_far_fill_kernel");
        }
    } else {
        constexpr int OT = (KCAP >= 32) ? 64 : 128;
        dim3 ogrid((unsigned)std::min<int64_t>(ceil_div(Q, OT), per_item), (unsigned)B);
        grid_overflow_kernel<KCAP, OT, 1024, IdxT><<<ogrid, OT, 0, st>>>(
            support, query, (int)S, (int)Q, K, qs.state, qs.ovf, (IdxT *)idx_out);
        FFB6D_LAUNCH_OK("grid_overflow_kernel");
        dim3 dgrid((unsigned)std::min<int64_t>(ceil_div(Q * K, 256), per_item), (unsigned)B);
        grid_dup_copy_kernel<IdxT><<<dgrid, 256, 0, st>>>((int)Q, K, qs.state, qs.ovf, (IdxT *)idx_out);
        FFB6D_LAUNCH_OK("grid_dup_copy_kernel");
    }
    return FFB6D_OK;
}

template <typename IdxT>
static int launch_search_k(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                           int K, void *idx_out, const GridStore &w, const QueryScratch &qs, int64_t query_width,
                           cudaStream_t st)
{
    if (K == 1) return launch_search<1, IdxT>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
    if (K <= 4) return launch_search<4, IdxT>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
    if (K <= 8) return launch_search<8, IdxT>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
    if (K <= 16) return launch_search<16, IdxT>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
    if (K <= 32) return launch_search<32, IdxT>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
    return launch_search<64, IdxT>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
}

// Build the grid of `support` for searches of about K neighbours (K only tunes the cell size).
int knn_grid_build(const float *support, int64_t B, int64_t S, int K, void *grid_mem,
                   size_t grid_bytes, cudaStream_t st)
{
    read_env();
    GridStore w = carve_grid(grid_mem, B, S);
    if (!grid_mem || grid_bytes < w.bytes) {
        set_error("knn grid build: %zu bytes of grid storage required, %zu given", w.bytes, grid_bytes);
        return FFB6D_ERR_WORKSPACE;
    }
    // one launch: a cluster of 8 CTAs per batch item (cluster dims are a compile-time attribute of the kernel)
    grid_build_kernel<<<dim3(BUILD_CTAS, (unsigned)B), BUILD_THREADS, 0, st>>>(
        support, (int)S, K, (int)w.maxc, K == 1 ? g_cell_scale_k1 : g_cell_scale, g_quantile, w.params, w.cursor,
        w.rank, w.sorted);
    FFB6D_LAUNCH_OK("grid_build_kernel");
    return FFB6D_OK;
}

// Search a built grid.  `support` must be the array the grid was built from.
int knn_grid_query(const float *support, const float *query, int64_t B, int64_t S, int64_t Q, int K,
                   void *idx_out, int idx_is_i64, const void *grid_mem, size_t grid_bytes,
                   void *scratch, size_t scratch_bytes, cudaStream_t st, int64_t query_width)
{
    read_env();
    GridStore w = carve_grid(const_cast<void *>(grid_mem), B, S);
    QueryScratch qs = carve_query(scratch, B, Q);
    if (!grid_mem || grid_bytes < w.bytes || !scratch || scratch_bytes < qs.bytes) {
        set_error("knn grid query: storage too small (grid %zu/%zu, scratch %zu/%zu)", grid_bytes, w.bytes,
                  scratch_bytes, qs.bytes);
        return FFB6D_ERR_WORKSPACE;
    }
    if (idx_is_i64) return launch_search_k<long long>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
    return launch_search_k<int>(support, query, B, S, Q, K, idx_out, w, qs, query_width, st);
}

int knn_grid_launch(const float *support, const float *query, int64_t B, int64_t S, int64_t Q, int K,
                    void *idx_out, int idx_is_i64, void *workspace, size_t workspace_bytes,
                    cudaStream_t st)
{
    const size_t gb = knn_grid_store_bytes(B, S), qb = knn_grid_query_bytes(B, Q);
    if (!workspace || workspace_bytes < gb + qb) {
        set_error("knn grid: workspace too small (%zu < %zu)", workspace_bytes, gb + qb);
        return FFB6D_ERR_WORKSPACE;
    }
    int rc = knn_grid_build(support, B, S, K, workspace, gb, st);
    if (rc) return rc;
    return knn_grid_query(support, query, B, S, Q, K, idx_out, idx_is_i64, workspace, gb,
                          (char *)workspace + gb, qb, st);
}

}  // namespace ffb6d
