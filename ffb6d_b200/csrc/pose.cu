// pose.cu -- keypoint voting (mean shift) and least-squares pose fitting on the device (sm_90a).
//
// The step right after the network (SURVEY.md §8 f-4): every point of an object votes for the
// object's keypoints and centre, the votes are clustered with a Gaussian mean shift
// (MeanShiftTorch.fit, ffb6d/utils/meanshift_pytorch.py:28-57) and the cluster centres are aligned
// with the mesh keypoints by a least-squares rigid fit (best_fit_transform,
// ffb6d/utils/pvn3d_eval_utils_kpls.py:28-59).  The reference materialises the N x N distance and
// weight matrices in HBM every iteration (3 x 600 MB at N = 12288) and synchronises with the host
// once per iteration for the stop test; one call per keypoint, 9 calls per object.
//
// Here all G vote sets of an object (ffb6d_mean_shift_fit), or every vote set of a stage of a whole test batch
// (ffb6d_vote_poses, DESIGN.md §4.25), are ONE persistent cooperative kernel over a set table: the modes live in L2
// (16 B per point, ping-pong), a CTA owns 128 points of one set at a time and streams the whole
// set through shared memory, the N x N matrix never exists, and the stop test is a device-side
// max + grid barrier.  The arithmetic is exp-bound (one MUFU.EX2 + ~11 FP32 per pair), not
// HBM-bound.  Results are floating point: sums run in a different order than torch's, so parity is
// by tolerance (tests/test_gpu_pose.py), never bitwise.
#include <algorithm>
#include <climits>

#include "common.cuh"

namespace ffb6d {

constexpr int MS_THREADS = 256;
constexpr int MS_IT = 128;         // points of one work item (two per thread, four j-slices)
constexpr int MS_JT = 2048;        // points of one staged tile (32 KB)
constexpr int MS_MAX_G = 64;       // vote sets per ffb6d_mean_shift_fit call

// Per-set state, in global memory, zeroed before the launch except `n`.
struct MsSet {
    int n;                          // points of the set
    int iters;                      // rounds run; written once the set stops, 0 while it runs
    unsigned shift[3];              // max |new - old| of a round (float bits), rotating slots
    unsigned pad;
    unsigned long long best;        // (count << 32) | ~index of the densest mode
};
static_assert(sizeof(MsSet) == 32, "ffb6d_mean_shift_workspace_bytes counts 32 bytes per set");

// The sets of one launch: set j is the n points at base[j] of the packed buffers (NULL: j * N); its centre is row
// id[j] of the centres (NULL: j) and its labels row id[j] / lab_div of the labels [.., N], at the points' original
// indices (src).
struct MsTab {
    MsSet *state;
    const int *base;
    const int *id;
    int N;
    int lab_div;
};

struct MsShared {
    float4 tile[MS_JT];
    float part[4][MS_IT][4];
    int first[MS_THREADS + 1];      // first work item of every set of the chunk
    int base[MS_THREADS], n[MS_THREADS];
    float red[MS_THREADS / 32];
    unsigned long long red64[MS_THREADS / 32];
    int scan[MS_THREADS / 32 + 1];
};

__device__ __forceinline__ void grid_sync(unsigned *counter, unsigned &target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        __threadfence();
        atomicAdd(counter, 1u);
        unsigned v;
        do {
            asm volatile("ld.acquire.gpu.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
        } while ((int)(v - target) < 0);
        __threadfence();
    }
    __syncthreads();
}

__device__ __forceinline__ float4 ldcg4(const float4 *p) { return __ldcg(p); }
__device__ __forceinline__ int ld_relaxed(const int *p)
{
    int v;
    asm volatile("ld.relaxed.gpu.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_relaxed(const unsigned *p)
{
    unsigned v;
    asm volatile("ld.relaxed.gpu.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(int *p, int v) { asm volatile("st.relaxed.gpu.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// 2^x on the SFU without exp2f's denormal-range fix-up (3 extra instructions per call): weights below 2^-126 flush
// to zero, and a weight of 1e-38 against the point's own weight of 1 is below fp32 resolution anyway
__device__ __forceinline__ float ex2_ftz(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// exclusive prefix sum of v over the CTA (MS_THREADS threads); the total goes to `total`
__device__ __forceinline__ int block_excl_scan(int v, int *s_scan, int &total)
{
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();                                  // an earlier scan's readers are done with s_scan
    if (lane == 31) s_scan[wid + 1] = x;
    __syncthreads();
    if (t == 0) {
        s_scan[0] = 0;
        for (int w = 0; w < MS_THREADS / 32; ++w) s_scan[w + 1] += s_scan[w];
    }
    __syncthreads();
    total = s_scan[MS_THREADS / 32];
    return s_scan[wid] + x - v;
}

// MODE 0: one mean-shift update of the item's points; MODE 1: neighbours within the bandwidth
template <int MODE>
__device__ __forceinline__ void ms_item(const float4 *__restrict__ cur, float4 *__restrict__ nxt, int n, int tile,
                                        float neg_scale, float bw, float4 *s_tile, float (*s_part)[MS_IT][4],
                                        float &cta_max, unsigned long long &cta_best)
{
    const int t = threadIdx.x, il = t & 63, slice = t >> 6;
    const int i0 = tile * MS_IT + il, i1 = i0 + 64;
    const float4 p0 = i0 < n ? ldcg4(cur + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 p1 = i1 < n ? ldcg4(cur + i1) : make_float4(0.f, 0.f, 0.f, 0.f);
    float a0x = 0.f, a0y = 0.f, a0z = 0.f, a0w = 0.f, a1x = 0.f, a1y = 0.f, a1z = 0.f, a1w = 0.f;
    for (int j0 = 0; j0 < n; j0 += MS_JT) {
        const int jn = min(MS_JT, n - j0);
        __syncthreads();
        for (int j = t; j < jn; j += MS_THREADS) s_tile[j] = ldcg4(cur + j0 + j);
        __syncthreads();
#pragma unroll 4
        for (int j = slice; j < jn; j += 4) {
            const float4 c = s_tile[j];            // the warp reads one address: a broadcast
            float dx = p0.x - c.x, dy = p0.y - c.y, dz = p0.z - c.z;
            const float d0 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            dx = p1.x - c.x, dy = p1.y - c.y, dz = p1.z - c.z;
            const float d1 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            if (MODE == 0) {
                const float w0 = ex2_ftz(d0 * neg_scale), w1 = ex2_ftz(d1 * neg_scale);
                a0x = fmaf(w0, c.x, a0x), a0y = fmaf(w0, c.y, a0y), a0z = fmaf(w0, c.z, a0z), a0w += w0;
                a1x = fmaf(w1, c.x, a1x), a1y = fmaf(w1, c.y, a1y), a1z = fmaf(w1, c.z, a1z), a1w += w1;
            } else {
                a0w += (sqrtf(d0) < bw) ? 1.f : 0.f;   // counts stay exact in fp32 (n < 2^24)
                a1w += (sqrtf(d1) < bw) ? 1.f : 0.f;
            }
        }
    }
    s_part[slice][il][0] = a0x, s_part[slice][il][1] = a0y, s_part[slice][il][2] = a0z, s_part[slice][il][3] = a0w;
    s_part[slice][il + 64][0] = a1x, s_part[slice][il + 64][1] = a1y, s_part[slice][il + 64][2] = a1z, s_part[slice][il + 64][3] = a1w;
    __syncthreads();
    if (t < MS_IT) {
        const int i = tile * MS_IT + t;
        if (i < n) {
            float sx = 0.f, sy = 0.f, sz = 0.f, sw = 0.f;
#pragma unroll
            for (int s = 0; s < 4; ++s) sx += s_part[s][t][0], sy += s_part[s][t][1], sz += s_part[s][t][2], sw += s_part[s][t][3];
            if (MODE == 0) {
                const float4 p = ldcg4(cur + i);
                const float nx = sx / sw, ny = sy / sw, nz = sz / sw;      // sw >= 1: the point's own weight
                const float ex = nx - p.x, ey = ny - p.y, ez = nz - p.z;
                nxt[i] = make_float4(nx, ny, nz, 0.f);
                cta_max = fmaxf(cta_max, sqrtf(fmaf(ez, ez, fmaf(ey, ey, ex * ex))));
            } else {
                const unsigned long long key = ((unsigned long long)(unsigned)sw << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
                cta_best = max(cta_best, key);
            }
        }
    }
}

// The work list of a phase, the same in every CTA and built from global state, so shared memory does not grow with
// the set count: the sets are taken in chunks of MS_THREADS, set j contributes items(j, n_j) work items numbered
// after those of all earlier sets, and this CTA runs run(j, base_j, n_j, k) for the items g = k-th of set j with
// g % gridDim.x == blockIdx.x.  Returns the number of items of the phase.
template <class Items, class Run>
__device__ __forceinline__ int ms_for_items(const MsTab &tab, int S, MsShared &sh, Items items, Run run)
{
    const int t = threadIdx.x;
    int acc = 0;
    for (int j0 = 0; j0 < S; j0 += MS_THREADS) {
        const int j = j0 + t;
        int n = 0, k = 0;
        if (j < S) {
            n = ld_relaxed(&tab.state[j].n);
            k = items(j, n);
        }
        int tot;
        const int first = block_excl_scan(k, sh.scan, tot);
        sh.first[t] = first;
        if (t == 0) sh.first[MS_THREADS] = tot;
        sh.n[t] = n;
        sh.base[t] = j < S ? (tab.base ? tab.base[j] : j * tab.N) : 0;
        __syncthreads();
        const int grid = (int)gridDim.x;
        for (int g = acc + ((int)blockIdx.x - acc % grid + grid) % grid; g < acc + tot; g += grid) {
            const int loc = g - acc;
            int lo = 0, hi = MS_THREADS - 1;             // the last set whose first item is <= loc
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (sh.first[mid] <= loc) lo = mid;
                else hi = mid - 1;
            }
            run(j0 + lo, sh.base[lo], sh.n[lo], loc - sh.first[lo]);
        }
        acc += tot;
    }
    return acc;
}

// Mean shift of every set of `tab` to convergence, then the densest mode, the centre and the inlier labels: phases
// B-D of a persistent cooperative kernel whose packed points (buf0) and `n`s are in place (after a grid barrier).
// Sets run their rounds independently, and an item's arithmetic depends only on its set's points, so a set's
// centre, labels and rounds do not depend on the other sets of the launch or on the grid.
__device__ void ms_run(const MsTab &tab, int S, float bandwidth, float stop_thresh, int max_iter, unsigned *barrier,
                       unsigned &target, MsShared &sh, float4 *__restrict__ buf0, float4 *__restrict__ buf1,
                       const int *__restrict__ src, float *__restrict__ centres, unsigned char *__restrict__ labels,
                       int *__restrict__ iters_out, float *__restrict__ modes, int *__restrict__ lab_count)
{
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const int grid = (int)gridDim.x, me = (int)blockIdx.x;

    // ---- phase B: mean-shift rounds.  A set runs round `it` when it ran round it - 1 and that round's shift was
    // not below stop_thresh (the reference's `torch.max(Cdis) < stop_thresh or it > max_iter`,
    // meanshift_pytorch.py:46); its owner CTA (j % grid) records the rounds when it stops.  Every CTA reads the same
    // flags and shifts, so every CTA builds the same list; a stale `iters` read (0 where the owner has just written
    // it - 1) takes the shift test to the same answer. ----
    const float neg_scale = -0.5f * 1.4426950408889634f / (bandwidth * bandwidth);   // exp(-d^2 / 2bw^2) as exp2
    for (int it = 1;; ++it) {
        auto live = [&](int j, int n) -> int {
            MsSet &st = tab.state[j];
            if (n == 0 || ld_relaxed(&st.iters) != 0) return 0;
            const bool own = j % grid == me;
            if (it > 1) {
                const float s = __uint_as_float(ld_relaxed(&st.shift[(it - 1) % 3]));
                if (s < stop_thresh || it - 1 > max_iter) {
                    if (own) st_relaxed(&st.iters, it - 1);
                    return 0;
                }
            }
            if (own) st.shift[(it + 1) % 3] = 0u;      // the slot of the NEXT round
            return (n + MS_IT - 1) / MS_IT;
        };
        auto update = [&](int j, int base, int n, int tile) {
            const int par = (it - 1) & 1;              // a running set has run it - 1 rounds
            float cta_max = 0.f;
            unsigned long long unused = 0;
            ms_item<0>((par ? buf1 : buf0) + base, (par ? buf0 : buf1) + base, n, tile, neg_scale, bandwidth, sh.tile,
                       sh.part, cta_max, unused);
#pragma unroll
            for (int o = 16; o; o >>= 1) cta_max = fmaxf(cta_max, __shfl_xor_sync(0xffffffffu, cta_max, o));
            if (lane == 0) sh.red[wid] = cta_max;
            __syncthreads();
            if (t == 0) {
                float m = 0.f;
                for (int w = 0; w < MS_THREADS / 32; ++w) m = fmaxf(m, sh.red[w]);
                atomicMax(&tab.state[j].shift[it % 3], __float_as_uint(m));   // non-negative floats order as unsigned
            }
        };
        const int total = ms_for_items(tab, S, sh, live, update);
        if (total == 0) break;
        grid_sync(barrier, target);
    }
    grid_sync(barrier, target);                        // the owners' final `iters`

    // ---- phase C: the mode with the most modes within one bandwidth (first index on ties) ----
    auto items_of = [&](int, int n) -> int { return (n + MS_IT - 1) / MS_IT; };
    ms_for_items(tab, S, sh, items_of, [&](int j, int base, int n, int tile) {
        const float4 *cur = ((ld_relaxed(&tab.state[j].iters) & 1) ? buf1 : buf0) + base;
        float unused = 0.f;
        unsigned long long best = 0;
        ms_item<1>(cur, nullptr, n, tile, 0.f, bandwidth, sh.tile, sh.part, unused, best);
#pragma unroll
        for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (lane == 0) sh.red64[wid] = best;
        __syncthreads();
        if (t == 0) {
            unsigned long long m = 0;
            for (int w = 0; w < MS_THREADS / 32; ++w) m = max(m, sh.red64[w]);
            atomicMax(&tab.state[j].best, m);
        }
    });
    grid_sync(barrier, target);

    // ---- phase D: centre, inlier labels (original point order), rounds; a set without points gets centre 0 ----
    auto items_d = [&](int j, int n) -> int {
        if (n == 0 && j % grid == me) {
            const int id = tab.id ? tab.id[j] : j;
            centres[3 * (size_t)id] = 0.f, centres[3 * (size_t)id + 1] = 0.f, centres[3 * (size_t)id + 2] = 0.f;
            if (iters_out) iters_out[id] = 0;
        }
        return (n + MS_IT - 1) / MS_IT;
    };
    ms_for_items(tab, S, sh, items_d, [&](int j, int base, int n, int tile) {
        const int iters = ld_relaxed(&tab.state[j].iters);
        const float4 *cur = ((iters & 1) ? buf1 : buf0) + base;
        const unsigned long long best = ld_relaxed(&tab.state[j].best);
        const int mi = (int)(0xFFFFFFFFu - (unsigned)(best & 0xFFFFFFFFull));
        const float4 c = ldcg4(cur + mi);
        const int id = tab.id ? tab.id[j] : j;
        if (tile == 0 && t == 0) {
            centres[3 * (size_t)id] = c.x, centres[3 * (size_t)id + 1] = c.y, centres[3 * (size_t)id + 2] = c.z;
            if (iters_out) iters_out[id] = iters;
        }
        const int i = tile * MS_IT + t;
        int lab = 0;
        if (t < MS_IT && i < n) {
            const float4 p = ldcg4(cur + i);
            const float dx = c.x - p.x, dy = c.y - p.y, dz = c.z - p.z;
            lab = sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx))) < bandwidth;
            const size_t o = (size_t)(id / tab.lab_div) * tab.N + src[base + i];
            if (labels) labels[o] = (unsigned char)lab;
            if (modes) modes[o * 3] = p.x, modes[o * 3 + 1] = p.y, modes[o * 3 + 2] = p.z;
        }
        if (lab_count) {
            const int cnt = __syncthreads_count(lab);
            if (t == 0 && cnt) atomicAdd(&lab_count[id], cnt);
        }
    });
}

// ---- ffb6d_mean_shift_fit: G <= 64 dense sets, set g at g * N of the packed buffers ----
__global__ void __launch_bounds__(MS_THREADS, 2)
mean_shift_kernel(const float *__restrict__ votes, const unsigned char *__restrict__ valid, long long valid_stride, int G,
                  int N, float bandwidth, float stop_thresh, int max_iter, unsigned *__restrict__ barrier,
                  MsSet *__restrict__ state, float4 *__restrict__ buf0, float4 *__restrict__ buf1, int *__restrict__ src,
                  float *__restrict__ centres, unsigned char *__restrict__ labels, int *__restrict__ iters_out,
                  float *__restrict__ modes)
{
    __shared__ MsShared sh;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    unsigned target = 0;

    // ---- phase A: ordered compaction of the valid votes of every set (the reference's votes[mask]) ----
    for (int g = blockIdx.x; g < G; g += gridDim.x) {
        const unsigned char *v = valid ? valid + (size_t)g * valid_stride : nullptr;
        const float *src_pts = votes + (size_t)g * N * 3;
        float4 *dst = buf0 + (size_t)g * N;
        int base = 0;
        for (int i0 = 0; i0 < N; i0 += MS_THREADS) {
            const int i = i0 + t;
            const bool ok = i < N && (!v || v[i] != 0);
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) sh.scan[wid + 1] = __popc(m);
            __syncthreads();
            if (t == 0) {
                sh.scan[0] = 0;
                for (int w = 0; w < MS_THREADS / 32; ++w) sh.scan[w + 1] += sh.scan[w];
            }
            __syncthreads();
            if (ok) {
                const int k = base + sh.scan[wid] + __popc(m & ((1u << lane) - 1u));
                dst[k] = make_float4(src_pts[3 * (size_t)i], src_pts[3 * (size_t)i + 1], src_pts[3 * (size_t)i + 2], 0.f);
                src[(size_t)g * N + k] = i;
            }
            if (i < N) {
                labels[(size_t)g * N + i] = 0;
                if (modes) modes[((size_t)g * N + i) * 3] = 0.f, modes[((size_t)g * N + i) * 3 + 1] = 0.f, modes[((size_t)g * N + i) * 3 + 2] = 0.f;
            }
            base += sh.scan[MS_THREADS / 32];
            __syncthreads();
        }
        if (t == 0) state[g].n = base;
    }
    grid_sync(barrier, target);
    const MsTab tab{state, nullptr, nullptr, N, 1};
    ms_run(tab, G, bandwidth, stop_thresh, max_iter, barrier, target, sh, buf0, buf1, src, centres, labels, iters_out,
           modes, nullptr);
}

// ---- ffb6d_vote_poses: one stage's vote sets (b, c, k), their table built by vote_table_kernel ----
// Set (b, c, k) holds the points i of frame b with cls[b,i] == c (and keep[b,i] when keep is given), in ascending
// order, as pcld[b,i] - of[b,k,i]: the reference's `pcld - of` and `votes[mask]`, bit for bit.
__global__ void __launch_bounds__(MS_THREADS, 2)
vote_ms_kernel(const float *__restrict__ pcld, const float *__restrict__ of, const int *__restrict__ cls,
               const unsigned char *__restrict__ keep, int N, int C, int K, const int *__restrict__ n_sets,
               const int *__restrict__ set_base, const int *__restrict__ set_id, MsSet *__restrict__ state,
               float bandwidth, float stop_thresh, int max_iter, unsigned *__restrict__ barrier,
               float4 *__restrict__ buf0, float4 *__restrict__ buf1, int *__restrict__ src, float *__restrict__ centres,
               unsigned char *__restrict__ labels, int *__restrict__ lab_count)
{
    __shared__ MsShared sh;
    const int t = threadIdx.x, lane = t & 31;
    unsigned target = 0;
    const int S = *n_sets;

    // ---- phase A: ordered compaction of every set's votes ----
    for (int j = blockIdx.x; j < S; j += gridDim.x) {
        const int id = set_id[j], k = id % K, c = (id / K) % C, b = id / K / C;
        const int *cl = cls + (size_t)b * N;
        const unsigned char *kp = keep ? keep + (size_t)b * N : nullptr;
        const float *p = pcld + (size_t)b * N * 3, *o = of + ((size_t)b * K + k) * N * 3;
        float4 *dst = buf0 + set_base[j];
        int *ix = src + set_base[j];
        int base = 0;
        for (int i0 = 0; i0 < N; i0 += MS_THREADS) {
            const int i = i0 + t;
            const bool ok = i < N && cl[i] == c && (!kp || kp[i] != 0);
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            int tot;
            const int r = __shfl_sync(0xffffffffu, block_excl_scan(lane == 0 ? __popc(m) : 0, sh.scan, tot), 0);
            if (ok) {
                const int q = base + r + __popc(m & ((1u << lane) - 1u));
                const size_t e = 3 * (size_t)i;
                dst[q] = make_float4(p[e] - o[e], p[e + 1] - o[e + 1], p[e + 2] - o[e + 2], 0.f);
                ix[q] = i;
            }
            base += tot;
        }
    }
    grid_sync(barrier, target);
    const MsTab tab{state, set_base, set_id, N, C * K};
    ms_run(tab, S, bandwidth, stop_thresh, max_iter, barrier, target, sh, buf0, buf1, src, centres, labels, nullptr,
           nullptr, lab_count);
}

// ---- least-squares rigid fit (Kabsch) of M point pairs, one thread per problem, fp64 like numpy ----
__global__ void best_fit_kernel(const float *__restrict__ A, const float *__restrict__ Bp, int G, int M, double *__restrict__ T)
{
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const float *a = A + (size_t)g * M * 3, *b = Bp + (size_t)g * M * 3;
    double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0};
    for (int m = 0; m < M; ++m)
        for (int d = 0; d < 3; ++d) ca[d] += (double)a[3 * m + d], cb[d] += (double)b[3 * m + d];
    for (int d = 0; d < 3; ++d) ca[d] /= (double)M, cb[d] /= (double)M;
    double H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};          // H = AA^T BB  (pvn3d_eval_utils_kpls.py:47)
    for (int m = 0; m < M; ++m)
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) H[r][c] += ((double)a[3 * m + r] - ca[r]) * ((double)b[3 * m + c] - cb[c]);
    // one-sided Jacobi: rotate column pairs of H (and of V) until orthogonal: H V = U S
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double al = 0, be = 0, ga = 0;
                for (int r = 0; r < 3; ++r) al += H[r][p] * H[r][p], be += H[r][q] * H[r][q], ga += H[r][p] * H[r][q];
                // a pair is done when its columns are orthogonal to working precision, or when one of them is
                // negligible next to the other (norm ratio <= 1e-15, below the rank cut-off `tiny` further down, so
                // its direction is never used: rotating it only spins on rounding noise).  sqrt(al) * sqrt(be),
                // not sqrt(al * be): the product underflows to 0 for spreads of float32 subnormals.
                const double nrm = sqrt(al) * sqrt(be);
                if (fabs(ga) <= 1e-17 * nrm || fmin(al, be) <= 1e-30 * fmax(al, be)) continue;
                off = fmax(off, fabs(ga) / nrm);
                const double zeta = (be - al) / (2.0 * ga);
                const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
                for (int r = 0; r < 3; ++r) {
                    const double hp = H[r][p], hq = H[r][q];
                    H[r][p] = cs * hp - sn * hq, H[r][q] = sn * hp + cs * hq;
                    const double vp = V[r][p], vq = V[r][q];
                    V[r][p] = cs * vp - sn * vq, V[r][q] = sn * vp + cs * vq;
                }
            }
        if (off < 1e-15) break;
    }
    double sg[3];
    int ord[3] = {0, 1, 2};
    for (int k = 0; k < 3; ++k) sg[k] = sqrt(H[0][k] * H[0][k] + H[1][k] * H[1][k] + H[2][k] * H[2][k]);
    for (int x = 0; x < 2; ++x)                      // singular values in descending order
        for (int y = 0; y < 2 - x; ++y)
            if (sg[ord[y]] < sg[ord[y + 1]]) { const int tmp = ord[y]; ord[y] = ord[y + 1], ord[y + 1] = tmp; }
    double U[3][3], W[3][3];
    for (int k = 0; k < 3; ++k)
        for (int r = 0; r < 3; ++r) W[r][k] = V[r][ord[k]];
    // U = H V / S where a singular value is above `tiny`; the rest of the basis is completed so that U stays
    // orthonormal: rank 3 none, rank 2 (coplanar) U2 = U0 x U1, rank 1 (collinear, or M = 2) U1 = the coordinate
    // axis least aligned with U0 made orthogonal to it, then U2 = U0 x U1, rank 0 (all points identical) the
    // identity.  Below rank 3 the fit is not unique: any such completion gives a proper rotation (after the
    // reflection flip) that reaches the least-squares minimum, as every choice of numpy's SVD does.
    const double tiny = 1e-12 * fmax(sg[ord[0]], 1e-300);
    for (int k = 0; k < 2; ++k)
        for (int r = 0; r < 3; ++r) U[r][k] = sg[ord[k]] > tiny ? H[r][ord[k]] / sg[ord[k]] : (r == k ? 1.0 : 0.0);
    if (sg[ord[0]] > tiny && sg[ord[1]] <= tiny) {
        int k = 0;
        for (int r = 1; r < 3; ++r)
            if (fabs(U[r][0]) < fabs(U[k][0])) k = r;
        for (int r = 0; r < 3; ++r) U[r][1] = (r == k ? 1.0 : 0.0) - U[k][0] * U[r][0];      // Gram-Schmidt of e_k
        const double nu = sqrt(U[0][1] * U[0][1] + U[1][1] * U[1][1] + U[2][1] * U[2][1]);    // >= sqrt(2/3)
        for (int r = 0; r < 3; ++r) U[r][1] /= nu;
    }
    if (sg[ord[2]] > tiny)
        for (int r = 0; r < 3; ++r) U[r][2] = H[r][ord[2]] / sg[ord[2]];
    else {                                           // rank <= 2: complete the basis
        U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
        U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
        U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
    }
    double R[3][3];
    for (int pass = 0; pass < 2; ++pass) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) R[r][c] = W[r][0] * U[c][0] + W[r][1] * U[c][1] + W[r][2] * U[c][2];   // R = V U^T
        const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) +
                           R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
        if (det >= 0) break;
        for (int r = 0; r < 3; ++r) W[r][2] = -W[r][2];     // the reflection case (:52-54)
    }
    double *out = T + (size_t)g * 12;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) out[4 * r + c] = R[r][c];
        out[4 * r + 3] = cb[r] - (R[r][0] * ca[0] + R[r][1] * ca[1] + R[r][2] * ca[2]);
    }
}

// ---- ffb6d_vote_poses: the per-frame and per-class steps around the three mean-shift stages ----
constexpr int VOTE_THREADS = 512;

// One CTA per frame: the class of every point (-1 for an id outside [0, C): the frame is then bad and gets no
// sets), the points and the first point of every class, the present classes (the reference's pred_cls_ids).
__global__ void __launch_bounds__(VOTE_THREADS)
vote_classes_kernel(const int64_t *__restrict__ mask, int N, int C, int *__restrict__ cls, unsigned char *__restrict__ keep,
                    int *__restrict__ counts, int *__restrict__ first, unsigned char *__restrict__ present,
                    int *__restrict__ bad)
{
    extern __shared__ int s_cls[];                    // counts [C], first points [C]
    __shared__ int s_bad;
    const int b = blockIdx.x, t = threadIdx.x;
    for (int c = t; c < C; c += VOTE_THREADS) s_cls[c] = 0, s_cls[C + c] = INT_MAX;
    if (t == 0) s_bad = 0;
    __syncthreads();
    for (int i = t; i < N; i += VOTE_THREADS) {
        const int64_t m = mask[(size_t)b * N + i];
        const int c = (m >= 0 && m < C) ? (int)m : -1;
        if (c < 0) s_bad = 1;
        cls[(size_t)b * N + i] = c;
        keep[(size_t)b * N + i] = 0;
        if (c > 0) atomicAdd(&s_cls[c], 1), atomicMin(&s_cls[C + c], i);
    }
    __syncthreads();
    for (int c = t; c < C; c += VOTE_THREADS) {
        const int n = s_bad ? 0 : s_cls[c];
        counts[(size_t)b * C + c] = c > 0 ? n : 0;
        first[(size_t)b * C + c] = s_cls[C + c];
        present[(size_t)b * C + c] = c > 0 && n > 0;
    }
    if (t == 0) bad[b] = s_bad;
}

// One CTA per frame: the centre-clustering refinement (pvn3d_eval_utils_kpls.py:85-109).  An object point takes the
// class of the nearest fitted centre of its frame's present classes (the lowest class id on distance ties; a NaN
// distance wins, as torch.min propagates it, and then nothing changes) when that distance, |pred_ctr - ctr| in the
// reference's difference form, is below thr[class].  Counts and first points of the refined classes.
__global__ void __launch_bounds__(VOTE_THREADS)
vote_refine_kernel(const float *__restrict__ pcld, const float *__restrict__ ctr_of, const int *__restrict__ cls0,
                   const unsigned char *__restrict__ present, const float *__restrict__ ctrs, const float *__restrict__ thr,
                   const int *__restrict__ bad, int N, int C, int *__restrict__ cls1, int *__restrict__ counts,
                   int *__restrict__ first)
{
    extern __shared__ int s_ref[];                    // counts [C], first points [C], present ids [C], centres [C][3]
    __shared__ int s_np;
    int *s_cnt = s_ref, *s_first = s_ref + C, *s_ids = s_ref + 2 * C;
    float *s_ctr = (float *)(s_ref + 3 * C);
    const int b = blockIdx.x, t = threadIdx.x;
    for (int c = t; c < C; c += VOTE_THREADS) s_cnt[c] = 0, s_first[c] = INT_MAX;
    if (t == 0) {
        int np = 0;
        for (int c = 1; c < C; ++c)
            if (present[(size_t)b * C + c]) {
                s_ids[np] = c;
                for (int d = 0; d < 3; ++d) s_ctr[3 * np + d] = ctrs[((size_t)b * C + c) * 3 + d];
                ++np;
            }
        s_np = np;
    }
    __syncthreads();
    const int np = s_np;
    for (int i = t; i < N; i += VOTE_THREADS) {
        const size_t e = (size_t)b * N + i;
        int c = cls0[e];
        if (c > 0) {
            const float px = pcld[3 * e] - ctr_of[3 * e], py = pcld[3 * e + 1] - ctr_of[3 * e + 1],
                        pz = pcld[3 * e + 2] - ctr_of[3 * e + 2];
            float best = INFINITY;
            int near = -1;
            for (int q = 0; q < np; ++q) {
                const float dx = px - s_ctr[3 * q], dy = py - s_ctr[3 * q + 1], dz = pz - s_ctr[3 * q + 2];
                const float d = sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
                if (d != d) {
                    near = -1;
                    break;
                }
                if (d < best) best = d, near = s_ids[q];
            }
            if (near > 0 && best < thr[near]) c = near;
        }
        cls1[e] = c;
        if (c > 0) atomicAdd(&s_cnt[c], 1), atomicMin(&s_first[c], i);
    }
    __syncthreads();
    for (int c = t; c < C; c += VOTE_THREADS) {
        counts[(size_t)b * C + c] = (bad[b] || c == 0) ? 0 : s_cnt[c];
        first[(size_t)b * C + c] = s_first[c];
    }
}

// One CTA: the set table of a stage, sets (b, c, k) in ascending order, one per k for every (b, c) with points.
// With lab_count (the keypoint stage under the centre-label filter) a class keeps the points its centre fit
// labelled, or its first point when none was (the reference's `ctr_labels[0] = 1`, :126-127).
__global__ void __launch_bounds__(MS_THREADS)
vote_table_kernel(const int *__restrict__ counts, const int *__restrict__ lab_count, const int *__restrict__ first,
                  unsigned char *__restrict__ keep, int BC, int C, int K, int N, MsSet *__restrict__ state,
                  int *__restrict__ set_base, int *__restrict__ set_id, int *__restrict__ n_sets)
{
    __shared__ int s_scan[MS_THREADS / 32 + 1];
    const int t = threadIdx.x;
    int sets = 0, slots = 0;
    for (int p0 = 0; p0 < BC; p0 += MS_THREADS) {
        const int p = p0 + t;
        int n = p < BC ? counts[p] : 0;
        if (lab_count && n > 0) {
            n = lab_count[p];
            if (n == 0) {
                keep[(size_t)(p / C) * N + first[p]] = 1;
                n = 1;
            }
        }
        int n_set, n_slot;
        const int j = sets + block_excl_scan(n > 0 ? K : 0, s_scan, n_set);
        const int o = slots + block_excl_scan(n * K, s_scan, n_slot);
        if (n > 0)
            for (int k = 0; k < K; ++k) {
                set_base[j + k] = o + k * n;
                set_id[j + k] = p * K + k;
                state[j + k] = MsSet{n, 0, {0u, 0u, 0u}, 0u, 0ull};
            }
        sets += n_set, slots += n_slot;
    }
    if (t == 0) *n_sets = sets;
}

// (b, c, r): the mesh row r of class c as the fit's source, and the voted row (keypoint r, or the centre last) as
// its target, written to kps; zero for a class without points (the row is fixed up by vote_finish_kernel).
__global__ void vote_gather_kernel(const float *__restrict__ mesh_kps, const float *__restrict__ kp_ctr,
                                   const float *__restrict__ ctr, const int *__restrict__ counts, int BC, int C, int K,
                                   int R, float *__restrict__ A, float *__restrict__ kps)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)BC * R) return;
    const int p = (int)(e / R), r = (int)(e % R), c = p % C;
    const bool has = counts[p] > 0;
    for (int d = 0; d < 3; ++d) {
        A[3 * e + d] = mesh_kps[((size_t)c * R + r) * 3 + d];
        kps[3 * e + d] = !has ? 0.f : r < K ? kp_ctr[((size_t)p * K + r) * 3 + d] : ctr[(size_t)p * 3 + d];
    }
}

// (b, c): the rows that get no fit.  A bad frame: NaN; an absent class: zeros; a present class that refinement left
// without points: the identity and zero keypoints; a present class without a mesh: NaN.
__global__ void vote_finish_kernel(const unsigned char *__restrict__ present, const int *__restrict__ counts,
                                   const unsigned char *__restrict__ has_mesh, const int *__restrict__ bad, int BC,
                                   int C, int R, int *__restrict__ count, float *__restrict__ kps,
                                   double *__restrict__ poses)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= BC) return;
    const int c = p % C;
    count[p] = counts[p];
    const bool nan = bad[p / C] || (present[p] && !has_mesh[c]);
    if (!nan && present[p] && counts[p] > 0) return;
    const double v = nan ? (double)NAN : 0.0;
    for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 4; ++q) poses[(size_t)p * 12 + 4 * r + q] = (!nan && present[p] && r == q) ? 1.0 : v;
    for (int q = 0; q < 3 * R; ++q) kps[(size_t)p * 3 * R + q] = (float)v;
}

}  // namespace ffb6d

using namespace ffb6d;

static size_t ms_header_bytes(int64_t G) { return align_up(256 + (size_t)G * sizeof(MsSet), 256); }

extern "C" size_t ffb6d_mean_shift_workspace_bytes(int64_t G, int64_t N)
{
    if (G <= 0 || N <= 0) return 0;
    return ms_header_bytes(G) + 2 * align_up((size_t)G * N * sizeof(float4), 256) + align_up((size_t)G * N * sizeof(int), 256);
}

extern "C" int ffb6d_mean_shift_fit(const float *votes, const unsigned char *valid, int64_t valid_stride, int64_t G, int64_t N,
                                    float bandwidth, int max_iter, float *centres, unsigned char *labels, int *iters,
                                    float *modes, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(G >= 0 && G <= MS_MAX_G && N >= 0 && N < (1ll << 24), "mean_shift_fit: G must be <= %d and N < 2^24", MS_MAX_G);
    FFB6D_CHECK_ARG(bandwidth > 0.f && max_iter >= 0, "mean_shift_fit: bandwidth must be positive, max_iter >= 0");
    if (G == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(centres && iters, "mean_shift_fit: null output");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        FFB6D_CUDA(cudaMemsetAsync(centres, 0, (size_t)G * 3 * sizeof(float), st));
        FFB6D_CUDA(cudaMemsetAsync(iters, 0, (size_t)G * sizeof(int), st));
        return FFB6D_OK;
    }
    FFB6D_CHECK_ARG(votes && labels && workspace, "mean_shift_fit: null pointer");
    FFB6D_CHECK_ARG(valid_stride == 0 || valid_stride >= N, "mean_shift_fit: valid_stride must be 0 (shared mask) or >= N");
    FFB6D_CHECK_ARG(workspace_bytes >= ffb6d_mean_shift_workspace_bytes(G, N), "mean_shift_fit: workspace too small");
    char *ws = (char *)workspace;
    unsigned *barrier = (unsigned *)ws;
    MsSet *state = (MsSet *)(ws + 256);
    const size_t hb = ms_header_bytes(G), cb = align_up((size_t)G * N * sizeof(float4), 256);
    float4 *buf0 = (float4 *)(ws + hb), *buf1 = (float4 *)(ws + hb + cb);
    int *src = (int *)(ws + hb + 2 * cb);
    FFB6D_CUDA(cudaMemsetAsync(ws, 0, hb, st));
    // all CTAs must be co-resident for the grid barrier: a cooperative launch sized from the occupancy
    static std::atomic<int> per_sm[kMaxDevices];
    const int dev = current_device() & (kMaxDevices - 1);
    int occ = per_sm[dev].load(std::memory_order_relaxed);
    if (occ == 0) {
        FFB6D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mean_shift_kernel, MS_THREADS, 0));
        FFB6D_CHECK_ARG(occ >= 1, "mean_shift_fit: kernel does not fit an SM");
        per_sm[dev].store(occ, std::memory_order_relaxed);
    }
    const int64_t items = G * ceil_div(N, MS_IT);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)num_sms() * std::min(occ, 2), items));
    int Gi = (int)G, Ni = (int)N;
    long long vs = valid_stride;
    float stop = (float)((double)bandwidth * 1e-3);        // MeanShiftTorch.stop_thresh (:31)
    void *args[] = {&votes, &valid, &vs, &Gi, &Ni, &bandwidth, &stop, &max_iter, &barrier, &state, &buf0, &buf1, &src,
                    &centres, &labels, &iters, &modes};
    FFB6D_CUDA(cudaLaunchCooperativeKernel((const void *)mean_shift_kernel, dim3((unsigned)grid), dim3(MS_THREADS), args, 0, st));
    count_launch();
    return FFB6D_OK;
}

extern "C" int ffb6d_best_fit_transform(const float *A, const float *B, int64_t G, int64_t M, double *T, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(G >= 0 && M >= 1 && M <= 4096, "best_fit_transform: need 1 <= M <= 4096 point pairs");
    if (G == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(A && B && T, "best_fit_transform: null pointer");
    best_fit_kernel<<<(unsigned)ceil_div(G, 64), 64, 0, (cudaStream_t)stream>>>(A, B, (int)G, (int)M, T);
    FFB6D_LAUNCH_OK("best_fit_kernel");
    return FFB6D_OK;
}

// a cooperative launch of `kern` over every SM (at most two CTAs each): all CTAs must be co-resident for the grid
// barrier.  The occupancy is queried once per device.
static int coop_grid(const void *kern, std::atomic<int> *per_sm, int &grid)
{
    const int dev = current_device() & (kMaxDevices - 1);
    int occ = per_sm[dev].load(std::memory_order_relaxed);
    if (occ == 0) {
        FFB6D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, MS_THREADS, 0));
        FFB6D_CHECK_ARG(occ >= 1, "mean shift: kernel does not fit an SM");
        per_sm[dev].store(occ, std::memory_order_relaxed);
    }
    grid = num_sms() * std::min(occ, 2);
    return FFB6D_OK;
}

// The workspace of ffb6d_vote_poses: one region per array, each 256-byte aligned, in this order.
struct VoteLayout {
    size_t off[27], total;
};
enum VoteRegion {
    V_ZERO,                       // 3 grid barriers + lab_count [B*C], zeroed by the call
    V_STATE_R, V_STATE_C, V_STATE_K, V_BASE_R, V_BASE_C, V_BASE_K, V_ID_R, V_ID_C, V_ID_K, V_NSETS,
    V_BUF0, V_BUF1, V_SRC, V_CLS0, V_CLS1, V_KEEP, V_CNT0, V_CNT1, V_FIRST0, V_FIRST1, V_BAD, V_CTR_R, V_CTR_C,
    V_KP, V_MESH, V_END
};
static_assert(V_END <= 27, "VoteLayout holds every region");

static VoteLayout vote_layout(int64_t B, int64_t N, int64_t C, int64_t K)
{
    const size_t BC = (size_t)(B * C), S = BC * (size_t)K, slots = (size_t)(K * B * N), BN = (size_t)(B * N);
    const size_t sz[V_END] = {
        256 + BC * 4,
        BC * sizeof(MsSet), BC * sizeof(MsSet), S * sizeof(MsSet), BC * 4, BC * 4, S * 4, BC * 4, BC * 4, S * 4, 3 * 4,
        slots * 16, slots * 16, slots * 4, BN * 4, BN * 4, BN, BC * 4, BC * 4, BC * 4, BC * 4, (size_t)B * 4,
        BC * 12, BC * 12, S * 12, BC * (size_t)(K + 1) * 12};
    VoteLayout L;
    size_t o = 0;
    for (int r = 0; r < V_END; ++r) L.off[r] = o, o += align_up(sz[r], 256);
    L.total = o;
    return L;
}

static bool vote_sizes_ok(int64_t B, int64_t N, int64_t C, int64_t K)
{
    return B >= 0 && N >= 1 && N <= FFB6D_VOTE_MAX_POINTS && C >= 2 && C <= FFB6D_VOTE_MAX_CLASSES && K >= 1 &&
           K <= FFB6D_VOTE_MAX_KPS && B * C * K <= FFB6D_VOTE_MAX_SETS && K * B * N <= FFB6D_VOTE_MAX_SLOTS;
}

extern "C" size_t ffb6d_vote_poses_workspace_bytes(int64_t B, int64_t N, int64_t n_cls, int64_t n_kps)
{
    if (B <= 0 || !vote_sizes_ok(B, N, n_cls, n_kps)) return 0;
    return vote_layout(B, N, n_cls, n_kps).total;
}

extern "C" int ffb6d_vote_poses(const float *pcld, const int64_t *mask, const float *ctr_of, const float *kp_of,
                                const float *mesh_kps, const unsigned char *has_mesh, const float *refine_thr, int64_t B,
                                int64_t N, int64_t n_cls, int64_t n_kps, int use_ctr, int ctr_filter, float bandwidth,
                                int max_iter, unsigned char *present, int *count, float *kps, double *poses,
                                void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && N >= 1 && N <= FFB6D_VOTE_MAX_POINTS, "vote_poses: need B >= 0 and 1 <= N <= %d",
                    FFB6D_VOTE_MAX_POINTS);
    FFB6D_CHECK_ARG(n_cls >= 2 && n_cls <= FFB6D_VOTE_MAX_CLASSES, "vote_poses: need 2 <= n_cls <= %d",
                    FFB6D_VOTE_MAX_CLASSES);
    FFB6D_CHECK_ARG(n_kps >= 1 && n_kps <= FFB6D_VOTE_MAX_KPS, "vote_poses: need 1 <= n_kps <= %d", FFB6D_VOTE_MAX_KPS);
    FFB6D_CHECK_ARG(B * n_cls * n_kps <= FFB6D_VOTE_MAX_SETS, "vote_poses: B * n_cls * n_kps sets exceed %d",
                    FFB6D_VOTE_MAX_SETS);
    FFB6D_CHECK_ARG(n_kps * B * N <= FFB6D_VOTE_MAX_SLOTS, "vote_poses: n_kps * B * N packed points exceed %d",
                    FFB6D_VOTE_MAX_SLOTS);
    FFB6D_CHECK_ARG((use_ctr == 0 || use_ctr == 1) && (ctr_filter == 0 || ctr_filter == 1),
                    "vote_poses: use_ctr and ctr_filter must be 0 or 1");
    FFB6D_CHECK_ARG(bandwidth > 0.f && bandwidth < INFINITY && max_iter >= 0,
                    "vote_poses: bandwidth must be positive and finite, max_iter >= 0");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(pcld && mask && ctr_of && kp_of && mesh_kps && has_mesh && present && count && kps && poses,
                    "vote_poses: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)pcld | (uintptr_t)ctr_of | (uintptr_t)kp_of | (uintptr_t)mesh_kps |
                     (uintptr_t)refine_thr | (uintptr_t)count | (uintptr_t)kps) % 4 == 0 &&
                        ((uintptr_t)mask | (uintptr_t)poses) % 8 == 0,
                    "vote_poses: pointers must be aligned to their element size");
    FFB6D_CHECK_ARG((uintptr_t)workspace % 256 == 0, "vote_poses: workspace must be 256-byte aligned");
    const VoteLayout L = vote_layout(B, N, n_cls, n_kps);
    if (!workspace || workspace_bytes < L.total) {
        set_error("vote_poses: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
        return FFB6D_ERR_WORKSPACE;
    }
    static std::atomic<int> per_sm[kMaxDevices];
    int grid;
    if (int rc = coop_grid((const void *)vote_ms_kernel, per_sm, grid)) return rc;

    char *ws = (char *)workspace;
    auto at = [&](int r) { return (void *)(ws + L.off[r]); };
    const cudaStream_t st = (cudaStream_t)stream;
    const int Bi = (int)B, Ni = (int)N, C = (int)n_cls, K = (int)n_kps, R = K + use_ctr, BC = Bi * C;
    unsigned *barrier = (unsigned *)at(V_ZERO);
    int *lab_count = (int *)(ws + L.off[V_ZERO] + 256);
    int *n_sets = (int *)at(V_NSETS), *cls0 = (int *)at(V_CLS0), *cls1 = (int *)at(V_CLS1);
    int *cnt0 = (int *)at(V_CNT0), *cnt1 = (int *)at(V_CNT1), *first0 = (int *)at(V_FIRST0), *first1 = (int *)at(V_FIRST1);
    int *bad = (int *)at(V_BAD);
    unsigned char *keep = (unsigned char *)at(V_KEEP);
    float4 *buf0 = (float4 *)at(V_BUF0), *buf1 = (float4 *)at(V_BUF1);
    int *src = (int *)at(V_SRC);
    float *ctr_r = (float *)at(V_CTR_R), *ctr_c = (float *)at(V_CTR_C), *kp_w = (float *)at(V_KP), *A = (float *)at(V_MESH);
    float stop = (float)((double)bandwidth * 1e-3);        // MeanShiftTorch.stop_thresh (meanshift_pytorch.py:31)

    FFB6D_CUDA(cudaMemsetAsync(ws + L.off[V_ZERO], 0, 256 + (size_t)BC * 4, st));
    vote_classes_kernel<<<Bi, VOTE_THREADS, 2 * C * sizeof(int), st>>>(mask, Ni, C, cls0, keep, cnt0, first0, present, bad);
    FFB6D_LAUNCH_OK("vote_classes_kernel");

    // one mean-shift stage: the table of its sets, then one cooperative launch over all of them
    auto stage = [&](int s, MsSet *state, int *base, int *id, const int *counts, const int *labc, const int *first,
                     const float *of, int k, const int *cls, const unsigned char *keep_in, float *centres,
                     unsigned char *labels, int *lab_out) -> int {
        vote_table_kernel<<<1, MS_THREADS, 0, st>>>(counts, labc, first, keep, BC, C, k, Ni, state, base, id, n_sets + s);
        FFB6D_LAUNCH_OK("vote_table_kernel");
        const int *ns = n_sets + s;
        unsigned *bar = barrier + s;
        void *args[] = {&pcld, &of, &cls, &keep_in, (void *)&Ni, (void *)&C, &k, &ns, &base, &id, &state, &bandwidth,
                        &stop, &max_iter, &bar, &buf0, &buf1, &src, &centres, &labels, &lab_out};
        FFB6D_CUDA(cudaLaunchCooperativeKernel((const void *)vote_ms_kernel, dim3((unsigned)grid), dim3(MS_THREADS), args, 0, st));
        count_launch();
        return FFB6D_OK;
    };
    const int *cls = cls0, *cnt = cnt0, *first = first0;
    if (refine_thr) {
        if (int rc = stage(0, (MsSet *)at(V_STATE_R), (int *)at(V_BASE_R), (int *)at(V_ID_R), cnt0, nullptr, nullptr,
                           ctr_of, 1, cls0, nullptr, ctr_r, nullptr, nullptr))
            return rc;
        vote_refine_kernel<<<Bi, VOTE_THREADS, 6 * C * sizeof(int), st>>>(
            pcld, ctr_of, cls0, present, ctr_r, refine_thr, bad, Ni, C, cls1, cnt1, first1);
        FFB6D_LAUNCH_OK("vote_refine_kernel");
        cls = cls1, cnt = cnt1, first = first1;
    }
    if (int rc = stage(1, (MsSet *)at(V_STATE_C), (int *)at(V_BASE_C), (int *)at(V_ID_C), cnt, nullptr, nullptr, ctr_of,
                       1, cls, nullptr, ctr_c, keep, lab_count))
        return rc;
    if (int rc = stage(2, (MsSet *)at(V_STATE_K), (int *)at(V_BASE_K), (int *)at(V_ID_K), cnt,
                       ctr_filter ? lab_count : nullptr, first, kp_of, K, cls, ctr_filter ? keep : nullptr, kp_w,
                       nullptr, nullptr))
        return rc;

    vote_gather_kernel<<<(unsigned)ceil_div((int64_t)BC * R, 256), 256, 0, st>>>(mesh_kps, kp_w, ctr_c, cnt, BC, C, K, R,
                                                                                 A, kps);
    FFB6D_LAUNCH_OK("vote_gather_kernel");
    best_fit_kernel<<<(unsigned)ceil_div(BC, 64), 64, 0, st>>>(A, kps, BC, R, poses);
    FFB6D_LAUNCH_OK("best_fit_kernel");
    vote_finish_kernel<<<(unsigned)ceil_div(BC, 256), 256, 0, st>>>(present, cnt, has_mesh, bad, BC, C, R, count, kps,
                                                                      poses);
    FFB6D_LAUNCH_OK("vote_finish_kernel");
    return FFB6D_OK;
}
