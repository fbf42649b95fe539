// segment_sum.cu -- deterministic backward of the K = 1 pixel -> point gather (sm_90a).
//
// The restructured fusion stage computes z = W1 * rgb + Z[idx] with Z = W2 * p2r on the N' points
// (fusion_mlp.cu, SURVEY.md §8f-3).  Its backward needs the transpose of the gather:
//     dZ[b, c, s] = sum over pixels p with idx[b, p] = s of dz[b, c, p]
// Pixel p belongs to segment idx[b, p].  Two steps:
//   plan  (ffb6d_segment_plan): a CSR per frame -- offsets[NA+1] and the pixels of each segment in ascending
//         order -- built stably from idx: warps count their 1024-pixel tile per segment (__match_any_sync groups,
//         integer atomics), one CTA per frame scans the (segment, tile) counts, and every warp places its tile's
//         pixels at (segment, tile) base + rank within the warp's group, walking its tile in order.
//   sum   (ffb6d_segment_sum): lane = channel, a warp sums a segment's pixels in plan order into an fp64
//         accumulator and rounds once to fp32.  A segment longer than SS_SPLIT pixels (the hole pixels of a
//         frame all map to one point) is split into one contiguous slice per warp of the CTA, and the slices
//         are added in warp order.  Every output element is written exactly once, by one thread, in an order
//         fixed by the plan: the result is bit-identical from run to run and from graph replay to replay.
// The sum is HBM bound: dz is read once (4 C P bytes per frame); the pixel list is a broadcast load.
#include "common.cuh"

#include <algorithm>

namespace ffb6d {

constexpr int SP_TILE = 1024;       // pixels per tile of the plan (one warp each)
constexpr int SP_WARPS = 8;         // tiles per CTA of the count / place kernels
constexpr int SS_WARPS = 32;        // warps per CTA of the sum; also the segments per CTA
constexpr int SS_SPLIT = 256;       // longer segments are split across the CTA's warps

// int32 words of one frame's plan: offsets [NA+1], pixels [P], tile counts [NA][T]; padded to 16 bytes
static inline int64_t plan_frame_ints(int64_t P, int64_t NA)
{
    const int64_t T = ceil_div(P, SP_TILE);
    return (NA + 1 + P + NA * T + 3) / 4 * 4;
}

template <typename I>
__device__ __forceinline__ int seg_key(const I *row, int p, int P, int NA)
{
    if (p >= P) return -1;
    const I v = __ldg(row + p);
    return (v >= 0 && v < (I)NA) ? (int)v : -1;     // out-of-range indices belong to no segment
}

template <typename I>
__global__ void __launch_bounds__(32 * SP_WARPS)
segment_count_kernel(const I *__restrict__ idx, int P, int NA, int T, long long frame_ints, int *__restrict__ plan)
{
    const int lane = threadIdx.x & 31, t = blockIdx.x * SP_WARPS + (threadIdx.x >> 5), b = blockIdx.y;
    if (t >= T) return;
    const I *row = idx + (size_t)b * P;
    int *tc = plan + (size_t)b * frame_ints + NA + 1 + P;
    const int p1 = min(P, (t + 1) * SP_TILE);
    for (int p0 = t * SP_TILE; p0 < p1; p0 += 32) {
        const int key = seg_key(row, p0 + lane, P, NA);
        const unsigned m = __match_any_sync(0xffffffffu, key);
        if (key >= 0 && lane == __ffs(m) - 1) atomicAdd(tc + (size_t)key * T + t, __popc(m));
    }
}

// exclusive scan of the frame's (segment, tile) counts in place; offsets[s] = the scan at (s, 0)
__global__ void __launch_bounds__(1024)
segment_scan_kernel(int P, int NA, int T, long long frame_ints, int *__restrict__ plan)
{
    __shared__ int wsum[32];
    int *off = plan + (size_t)blockIdx.x * frame_ints;
    int *tc = off + NA + 1 + P;
    const int rows = (NA + 1023) / 1024;                // whole segments per thread
    const int r0 = min(NA, (int)threadIdx.x * rows), r1 = min(NA, r0 + rows);
    const long long a = (long long)r0 * T, e = (long long)r1 * T;
    int s = 0;
    for (long long i = a; i < e; ++i) s += tc[i];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = s;                                          // inclusive warp scan
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int w = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        wsum[lane] = w;                                 // inclusive over warps
    }
    __syncthreads();
    int base = x - s + (wid > 0 ? wsum[wid - 1] : 0);
    for (int r = r0; r < r1; ++r) {
        off[r] = base;
        int *row = tc + (size_t)r * T;
        for (int t = 0; t < T; ++t) {
            const int v = row[t];
            row[t] = base;
            base += v;
        }
    }
    if (threadIdx.x == 1023) off[NA] = wsum[31];
}

template <typename I>
__global__ void __launch_bounds__(32 * SP_WARPS)
segment_place_kernel(const I *__restrict__ idx, int P, int NA, int T, long long frame_ints, int *__restrict__ plan)
{
    const int lane = threadIdx.x & 31, t = blockIdx.x * SP_WARPS + (threadIdx.x >> 5), b = blockIdx.y;
    if (t >= T) return;
    const I *row = idx + (size_t)b * P;
    int *pix = plan + (size_t)b * frame_ints + NA + 1;
    int *tc = pix + P;
    const int p1 = min(P, (t + 1) * SP_TILE);
    for (int p0 = t * SP_TILE; p0 < p1; p0 += 32) {
        const int key = seg_key(row, p0 + lane, P, NA);
        const unsigned m = __match_any_sync(0xffffffffu, key);
        const int leader = __ffs(m) - 1;
        int base = 0;
        if (key >= 0 && lane == leader) {               // this warp alone owns cursor (key, t)
            base = tc[(size_t)key * T + t];
            tc[(size_t)key * T + t] = base + __popc(m);
        }
        base = __shfl_sync(0xffffffffu, base, leader);
        if (key >= 0) pix[base + __popc(m & ((1u << lane) - 1u))] = p0 + lane;
        __syncwarp();                                   // the next leader of `key` reads the cursor written here
    }
}

// sum of g[pix[j]] for j in [a, e), in ascending j, in fp64
__device__ __forceinline__ double seg_range_sum(const float *__restrict__ g, const int *__restrict__ pix, int a, int e)
{
    double acc = 0.0;
    int j = a;
    for (; j + 8 <= e; j += 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldg(g + __ldg(pix + j + u));
#pragma unroll
        for (int u = 0; u < 8; ++u) acc += (double)v[u];
    }
    for (; j < e; ++j) acc += (double)__ldg(g + __ldg(pix + j));
    return acc;
}

// grid (ceil(NA / SS_WARPS), ceil(C / 32), B): a CTA owns SS_WARPS segments x 32 channels of one frame
__global__ void __launch_bounds__(32 * SS_WARPS)
segment_sum_kernel(const float *__restrict__ grad, const int *__restrict__ plan, long long frame_ints, int C, int P, int NA,
                   float *__restrict__ out)
{
    __shared__ double red[SS_WARPS][33];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, b = blockIdx.z;
    const int c = blockIdx.y * 32 + lane;
    const bool live = c < C;
    const int *off = plan + (size_t)b * frame_ints;
    const int *pix = off + NA + 1;
    const float *g = grad + ((size_t)b * C + (live ? c : C - 1)) * P;
    float *o = out + ((size_t)b * C + c) * NA;
    const int s0 = blockIdx.x * SS_WARPS, s1 = min(NA, s0 + SS_WARPS);
    const int s = s0 + wid;
    if (s < s1) {                                       // a warp per segment of at most SS_SPLIT pixels
        const int a = __ldg(off + s), e = __ldg(off + s + 1);
        if (e - a <= SS_SPLIT) {
            const double acc = seg_range_sum(g, pix, a, e);
            if (live) o[s] = (float)acc;
        }
    }
    for (int k = s0; k < s1; ++k) {                     // longer ones: one contiguous slice per warp
        const int a = __ldg(off + k), e = __ldg(off + k + 1);
        if (e - a <= SS_SPLIT) continue;
        const int chunk = (e - a + SS_WARPS - 1) / SS_WARPS;
        const int wa = min(e, a + wid * chunk), we = min(e, wa + chunk);
        red[wid][lane] = seg_range_sum(g, pix, wa, we);
        __syncthreads();
        if (wid == 0) {
            double acc = 0.0;
            for (int w = 0; w < SS_WARPS; ++w) acc += red[w][lane];
            if (live) o[k] = (float)acc;
        }
        __syncthreads();
    }
}

template <typename I>
static int plan_launch(const I *idx, int64_t B, int64_t P, int64_t NA, int *plan, cudaStream_t st)
{
    const int T = (int)ceil_div(P, SP_TILE);
    const long long F = plan_frame_ints(P, NA);
    FFB6D_CUDA(cudaMemsetAsync(plan, 0, (size_t)B * F * sizeof(int), st));
    const dim3 grid((unsigned)ceil_div(T, SP_WARPS), (unsigned)B);
    segment_count_kernel<I><<<grid, 32 * SP_WARPS, 0, st>>>(idx, (int)P, (int)NA, T, F, plan);
    FFB6D_LAUNCH_OK("segment_count_kernel");
    segment_scan_kernel<<<(unsigned)B, 1024, 0, st>>>((int)P, (int)NA, T, F, plan);
    FFB6D_LAUNCH_OK("segment_scan_kernel");
    segment_place_kernel<I><<<grid, 32 * SP_WARPS, 0, st>>>(idx, (int)P, (int)NA, T, F, plan);
    FFB6D_LAUNCH_OK("segment_place_kernel");
    return FFB6D_OK;
}

static bool plan_sizes_ok(int64_t B, int64_t P, int64_t NA)
{
    return B >= 1 && P >= 1 && NA >= 1 && B < 65536 && P < (1ll << 31) && NA < (1ll << 31) &&
           plan_frame_ints(P, NA) < (1ll << 31);
}

// ===================================================================== CSR plan in O(P + NA) (deterministic backward)
// The plan above keeps a (segment, 1024-pixel tile) counter table and scans it with one CTA per frame: cheap for the
// p2r maps (few segments), quadratic for the gathers of a training step whose index has as many segments as entries
// (`choose`: 307 200 segments, 12 288 entries).  ffb6d_segment_csr builds the same CSR -- offsets[NA+1], then every
// segment's entries in ascending position -- in work and memory linear in P + NA:
//   count   integer atomics per segment (warp-aggregated with __match_any_sync);
//   scan    a device-wide exclusive scan of the counts (tile sums, a scan of the tile sums, the tiles again);
//   place   every entry at an atomic cursor of its segment: the right set, in arbitrary order;
//   sort    each segment by position: <= CSR_SMALL entries by one thread (insertion sort), the others queue for
//           csr_sort_long_kernel (a CTA per segment: a bitonic sort in shared memory up to CSR_SMEM entries, and
//           for longer ones an ordered compaction of the whole index row, which writes the positions in order).
// The CSR of an index is unique, so the result does not depend on the order the atomics landed in.
// Frame layout (int32 words): offsets [NA+1] | entries [P] | counts / cursors [NA] | long count [1] |
// long segments [P / (CSR_SMALL+1) + 1] | tile sums [ceil(NA / CSR_SCAN)], padded to 16 bytes.
constexpr int CSR_SMALL = 32;       // segments up to this length are sorted by one thread
constexpr int CSR_SMEM = 8192;      // longer ones up to this length by a CTA in shared memory
constexpr int CSR_SCAN = 4096;      // counts per CTA of the scan (1024 threads x 4)
constexpr int CSR_LONG_CTAS = 64;   // CTAs per frame of the long-segment sort

struct CsrLayout {
    long long off, ent, cnt, nlong, longs, tiles, frame;
};

static inline CsrLayout csr_layout(int64_t P, int64_t NA)
{
    CsrLayout L;
    L.off = 0;
    L.ent = NA + 1;
    L.cnt = L.ent + P;
    L.nlong = L.cnt + NA;
    L.longs = L.nlong + 1;
    L.tiles = L.longs + P / (CSR_SMALL + 1) + 1;
    L.frame = (L.tiles + ceil_div(NA, CSR_SCAN) + 3) / 4 * 4;
    return L;
}

static bool csr_sizes_ok(int64_t B, int64_t P, int64_t NA)
{
    return B >= 1 && P >= 1 && NA >= 1 && B < 65536 && P < (1ll << 31) && NA < (1ll << 31) &&
           csr_layout(P, NA).frame < (1ll << 31);
}

template <typename I>
__global__ void __launch_bounds__(256)
csr_count_kernel(const I *__restrict__ idx, int P, int NA, CsrLayout L, int *__restrict__ plan)
{
    const int p = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    const int key = seg_key(idx + (size_t)b * P, p, P, NA);
    const unsigned m = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && (threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(plan + (size_t)b * L.frame + L.cnt + key, __popc(m));
}

// exclusive scan of 4 values per thread over a 1024-thread CTA; returns the thread's base, *total = the CTA's sum
__device__ __forceinline__ int cta_scan4(const int (&v)[4], int *wsum, int *total)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int s = v[0] + v[1] + v[2] + v[3];
    int x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int w = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        wsum[lane] = w;
    }
    __syncthreads();
    *total = wsum[31];
    return x - s + (wid > 0 ? wsum[wid - 1] : 0);
}

// grid (tiles, B): the sum of every CSR_SCAN counts
__global__ void __launch_bounds__(1024)
csr_tile_sum_kernel(int NA, CsrLayout L, int *__restrict__ plan)
{
    __shared__ int wsum[32];
    int *fr = plan + (size_t)blockIdx.y * L.frame;
    const int s0 = blockIdx.x * CSR_SCAN + 4 * threadIdx.x;
    int v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = (s0 + u < NA) ? fr[L.cnt + s0 + u] : 0;
    int total;
    cta_scan4(v, wsum, &total);
    if (threadIdx.x == 0) fr[L.tiles + blockIdx.x] = total;
}

// one CTA per frame: exclusive scan of the tile sums in place; offsets[NA] = the frame's entry count
__global__ void __launch_bounds__(1024)
csr_tile_scan_kernel(int NA, CsrLayout L, int *__restrict__ plan)
{
    __shared__ int wsum[32];
    int *fr = plan + (size_t)blockIdx.x * L.frame;
    int *ts = fr + L.tiles;
    const int nt = (NA + CSR_SCAN - 1) / CSR_SCAN;
    const int per = (nt + 4095) / 4096;                 // tile sums per (thread, slot)
    int v[4];
    for (int u = 0; u < 4; ++u) {
        const int a = min(nt, (4 * (int)threadIdx.x + u) * per), e = min(nt, a + per);
        int s = 0;
        for (int i = a; i < e; ++i) s += ts[i];
        v[u] = s;
    }
    int total;
    int base = cta_scan4(v, wsum, &total);
    for (int u = 0; u < 4; ++u) {
        const int a = min(nt, (4 * (int)threadIdx.x + u) * per), e = min(nt, a + per);
        for (int i = a; i < e; ++i) {
            const int c = ts[i];
            ts[i] = base;
            base += c;
        }
    }
    if (threadIdx.x == 0) fr[L.off + NA] = total;
}

// grid (tiles, B): offsets[s] = tile base + exclusive scan within the tile; the cursor of s starts there
__global__ void __launch_bounds__(1024)
csr_offsets_kernel(int NA, CsrLayout L, int *__restrict__ plan)
{
    __shared__ int wsum[32];
    int *fr = plan + (size_t)blockIdx.y * L.frame;
    const int s0 = blockIdx.x * CSR_SCAN + 4 * threadIdx.x;
    int v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = (s0 + u < NA) ? fr[L.cnt + s0 + u] : 0;
    int total;
    int base = cta_scan4(v, wsum, &total) + fr[L.tiles + blockIdx.x];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        if (s0 + u < NA) {
            fr[L.off + s0 + u] = base;
            fr[L.cnt + s0 + u] = base;
        }
        base += v[u];
    }
}

template <typename I>
__global__ void __launch_bounds__(256)
csr_place_kernel(const I *__restrict__ idx, int P, int NA, CsrLayout L, int *__restrict__ plan)
{
    const int lane = threadIdx.x & 31, p = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    int *fr = plan + (size_t)b * L.frame;
    const int key = seg_key(idx + (size_t)b * P, p, P, NA);
    const unsigned m = __match_any_sync(0xffffffffu, key);
    const int leader = __ffs(m) - 1;
    int base = 0;
    if (key >= 0 && lane == leader) base = atomicAdd(fr + L.cnt + key, __popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (key >= 0) fr[L.ent + base + __popc(m & ((1u << lane) - 1u))] = p;
}

// grid (ceil(NA / 256), B): a thread per segment sorts a short one, queues a long one
__global__ void __launch_bounds__(256)
csr_sort_short_kernel(int NA, CsrLayout L, int *__restrict__ plan)
{
    const int s = blockIdx.x * 256 + threadIdx.x;
    if (s >= NA) return;
    int *fr = plan + (size_t)blockIdx.y * L.frame;
    const int a = fr[L.off + s], e = fr[L.off + s + 1];
    if (e - a <= 1) return;
    if (e - a > CSR_SMALL) {
        fr[L.longs + atomicAdd(fr + L.nlong, 1)] = s;
        return;
    }
    int *v = fr + L.ent;
    for (int i = a + 1; i < e; ++i) {
        const int x = v[i];
        int j = i - 1;
        for (; j >= a && v[j] > x; --j) v[j + 1] = v[j];
        v[j + 1] = x;
    }
}

// grid (CSR_LONG_CTAS, B): the CTAs of a frame take its queued segments in turn
template <typename I>
__global__ void __launch_bounds__(1024)
csr_sort_long_kernel(const I *__restrict__ idx, int P, int NA, CsrLayout L, int *__restrict__ plan)
{
    __shared__ int key[CSR_SMEM];
    __shared__ int wsum[32];
    int *fr = plan + (size_t)blockIdx.y * L.frame;
    const int nlong = fr[L.nlong];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int i = blockIdx.x; i < nlong; i += gridDim.x) {
        const int s = fr[L.longs + i];
        const int a = fr[L.off + s], e = fr[L.off + s + 1], len = e - a;
        int *v = fr + L.ent + a;
        if (len <= CSR_SMEM) {                          // bitonic sort of the padded power of two
            int n = 1;
            while (n < len) n <<= 1;
            for (int t = tid; t < n; t += 1024) key[t] = t < len ? v[t] : 0x7fffffff;
            __syncthreads();
            for (int k = 2; k <= n; k <<= 1)
                for (int j = k >> 1; j > 0; j >>= 1) {
                    for (int t = tid; t < n; t += 1024) {
                        const int u = t ^ j;
                        if (u > t) {
                            const int x = key[t], y = key[u];
                            if ((x > y) == ((t & k) == 0)) {
                                key[t] = y;
                                key[u] = x;
                            }
                        }
                    }
                    __syncthreads();
                }
            for (int t = tid; t < len; t += 1024) v[t] = key[t];
        } else {                                        // ordered compaction of the row: positions come out sorted
            const I *row = idx + (size_t)blockIdx.y * P;
            int base = 0;
            for (int p0 = 0; p0 < P; p0 += 1024) {
                const bool hit = seg_key(row, p0 + tid, P, NA) == s;
                const unsigned bal = __ballot_sync(0xffffffffu, hit);
                if (lane == 0) wsum[wid] = __popc(bal);
                __syncthreads();
                int before = 0, total = 0;
                for (int w = 0; w < 32; ++w) {
                    const int c = wsum[w];
                    before += (w < wid) ? c : 0;
                    total += c;
                }
                if (hit) v[base + before + __popc(bal & ((1u << lane) - 1u))] = p0 + tid;
                base += total;
                __syncthreads();
            }
        }
        __syncthreads();
    }
}

template <typename I>
static int csr_launch(const I *idx, int64_t B, int64_t P, int64_t NA, int *plan, cudaStream_t st)
{
    const CsrLayout L = csr_layout(P, NA);
    FFB6D_CUDA(cudaMemsetAsync(plan, 0, (size_t)B * L.frame * sizeof(int), st));
    const dim3 gp((unsigned)ceil_div(P, 256), (unsigned)B), gt((unsigned)ceil_div(NA, CSR_SCAN), (unsigned)B);
    csr_count_kernel<I><<<gp, 256, 0, st>>>(idx, (int)P, (int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_count_kernel");
    csr_tile_sum_kernel<<<gt, 1024, 0, st>>>((int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_tile_sum_kernel");
    csr_tile_scan_kernel<<<(unsigned)B, 1024, 0, st>>>((int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_tile_scan_kernel");
    csr_offsets_kernel<<<gt, 1024, 0, st>>>((int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_offsets_kernel");
    csr_place_kernel<I><<<gp, 256, 0, st>>>(idx, (int)P, (int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_place_kernel");
    csr_sort_short_kernel<<<dim3((unsigned)ceil_div(NA, 256), (unsigned)B), 256, 0, st>>>((int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_sort_short_kernel");
    const unsigned nl = (unsigned)std::min<int64_t>(CSR_LONG_CTAS, P / (CSR_SMALL + 1) + 1);
    csr_sort_long_kernel<I><<<dim3(nl, (unsigned)B), 1024, 0, st>>>(idx, (int)P, (int)NA, L, plan);
    FFB6D_LAUNCH_OK("csr_sort_long_kernel");
    return FFB6D_OK;
}

static int csr_build(const void *idx, int idx_is_i64, int64_t B, int64_t P, int64_t NA, void *plan, cudaStream_t st)
{
    if (idx_is_i64) return csr_launch((const long long *)idx, B, P, NA, (int *)plan, st);
    return csr_launch((const int *)idx, B, P, NA, (int *)plan, st);
}

// ===================================================================== masked segment sum
// out[b, c, s] = sum over the entries x of segment s of g[b, c, x / K], counted only when amap[b, c, x / K] == x % K
// (amap null: every entry, K = 1).  g and amap share the strides (gb, gc, gq); out has (ob, oc, os).  Lane = channel,
// fp64 in plan order, one rounding; long segments are split across the CTA's warps as in segment_sum_kernel.
__device__ __forceinline__ double masked_range_sum(const float *__restrict__ g, const unsigned char *__restrict__ m,
                                                   long long gq, int K, const int *__restrict__ ent, int a, int e)
{
    double acc = 0.0;
    int j = a;
    for (; j + 4 <= e; j += 4) {
        float v[4];
        bool on[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int x = __ldg(ent + j + u), q = x / K;
            const long long o = (long long)q * gq;
            on[u] = !m || __ldg(m + o) == x - q * K;
            v[u] = on[u] ? __ldg(g + o) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (on[u]) acc += (double)v[u];
    }
    for (; j < e; ++j) {
        const int x = __ldg(ent + j), q = x / K;
        const long long o = (long long)q * gq;
        if (!m || __ldg(m + o) == x - q * K) acc += (double)__ldg(g + o);
    }
    return acc;
}

// grid (ceil(NA / SS_WARPS), ceil(C / 32), B)
__global__ void __launch_bounds__(32 * SS_WARPS)
segment_sum_masked_kernel(const float *__restrict__ grad, const unsigned char *__restrict__ amap, long long gb, long long gc,
                          long long gq, int K, const int *__restrict__ plan, CsrLayout L, int C, int NA,
                          float *__restrict__ out, long long ob, long long oc, long long os)
{
    __shared__ double red[SS_WARPS][33];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, b = blockIdx.z;
    const int c = blockIdx.y * 32 + lane;
    const bool live = c < C;
    const int *off = plan + (size_t)b * L.frame + L.off;
    const int *ent = plan + (size_t)b * L.frame + L.ent;
    const long long go = (long long)b * gb + (long long)(live ? c : C - 1) * gc;
    const float *g = grad + go;
    const unsigned char *m = amap ? amap + go : nullptr;
    float *o = out + (size_t)b * ob + (size_t)c * oc;
    const int s0 = blockIdx.x * SS_WARPS, s1 = min(NA, s0 + SS_WARPS);
    const int s = s0 + wid;
    if (s < s1) {
        const int a = __ldg(off + s), e = __ldg(off + s + 1);
        if (e - a <= SS_SPLIT) {
            const double acc = masked_range_sum(g, m, gq, K, ent, a, e);
            if (live) o[(size_t)s * os] = (float)acc;
        }
    }
    for (int k = s0; k < s1; ++k) {
        const int a = __ldg(off + k), e = __ldg(off + k + 1);
        if (e - a <= SS_SPLIT) continue;
        const int chunk = (e - a + SS_WARPS - 1) / SS_WARPS;
        const int wa = min(e, a + wid * chunk), we = min(e, wa + chunk);
        red[wid][lane] = masked_range_sum(g, m, gq, K, ent, wa, we);
        __syncthreads();
        if (wid == 0) {
            double acc = 0.0;
            for (int w = 0; w < SS_WARPS; ++w) acc += red[w][lane];
            if (live) o[(size_t)k * os] = (float)acc;
        }
        __syncthreads();
    }
}

// arg-max k of every (b, c, q) of a gather + max, by the rule of gather_max_bwd_kernel (gather.cu): a NaN wins,
// otherwise the first strict maximum; out-of-range indices read the clamped row.  amap in the order of grad_out.
template <typename IdxT>
__global__ void __launch_bounds__(256)
gather_argmax_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx, unsigned char *__restrict__ amap, int C,
                     int S, int Q, int K, int layout, long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    int b, c, q;
    size_t fs_c, fs_s;
    if (layout == FFB6D_LAYOUT_NCS) {
        q = (int)(t % Q);
        c = (int)((t / Q) % C);
        b = (int)(t / ((long long)Q * C));
        fs_c = (size_t)S;
        fs_s = 1;
    } else {
        c = (int)(t % C);
        q = (int)((t / C) % Q);
        b = (int)(t / ((long long)Q * C));
        fs_c = 1;
        fs_s = (size_t)C;
    }
    const IdxT *ip = idx + ((size_t)b * Q + q) * K;
    const float *f = feat + (size_t)b * C * S + (size_t)c * fs_c;
    const unsigned Su = (unsigned)S;
    int best = 0;
    float m = __ldg(f + (size_t)min((unsigned)(int)__ldg(ip), Su - 1) * fs_s);
    for (int k = 1; k < K; ++k) {
        const float v = __ldg(f + (size_t)min((unsigned)(int)__ldg(ip + k), Su - 1) * fs_s);
        if ((v > m || v != v) && !(m != m)) {
            m = v;
            best = k;
        }
    }
    amap[t] = (unsigned char)best;
}

static int masked_sum_launch(const float *grad, const unsigned char *amap, long long gb, long long gc, long long gq, int K,
                             const int *plan, const CsrLayout &L, int64_t B, int64_t C, int64_t NA, float *out, long long ob,
                             long long oc, long long os, cudaStream_t st)
{
    const dim3 grid((unsigned)ceil_div(NA, SS_WARPS), (unsigned)ceil_div(C, 32), (unsigned)B);
    segment_sum_masked_kernel<<<grid, 32 * SS_WARPS, 0, st>>>(grad, amap, gb, gc, gq, K, plan, L, (int)C, (int)NA, out, ob,
                                                              oc, os);
    FFB6D_LAUNCH_OK("segment_sum_masked_kernel");
    return FFB6D_OK;
}

static inline size_t csr_bytes(int64_t B, int64_t P, int64_t NA)
{
    if (!csr_sizes_ok(B, P, NA)) return 0;
    return (size_t)B * (size_t)csr_layout(P, NA).frame * sizeof(int);
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" {

size_t ffb6d_segment_plan_bytes(int64_t B, int64_t P, int64_t NA)
{
    if (!plan_sizes_ok(B, P, NA)) return 0;
    return (size_t)B * (size_t)plan_frame_ints(P, NA) * sizeof(int);
}

int ffb6d_segment_plan(const void *idx, int idx_is_i64, int64_t B, int64_t P, int64_t NA, void *plan, size_t plan_bytes,
                       ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(plan_sizes_ok(B, P, NA), "segment_plan: bad size");
    FFB6D_CHECK_ARG(idx_is_i64 == 0 || idx_is_i64 == 1, "segment_plan: idx_is_i64=%d", idx_is_i64);
    FFB6D_CHECK_ARG(idx && plan, "segment_plan: null pointer");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(idx) & (idx_is_i64 ? 7 : 3)) == 0, "segment_plan: idx misaligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(plan) & 15) == 0, "segment_plan: plan must be 16-byte aligned");
    FFB6D_CHECK_ARG(plan_bytes >= ffb6d_segment_plan_bytes(B, P, NA), "segment_plan: plan too small");
    cudaStream_t st = (cudaStream_t)stream;
    if (idx_is_i64) return plan_launch((const long long *)idx, B, P, NA, (int *)plan, st);
    return plan_launch((const int *)idx, B, P, NA, (int *)plan, st);
}

int ffb6d_segment_sum(const float *grad, const void *plan, size_t plan_bytes, int64_t B, int64_t C, int64_t P, int64_t NA,
                      float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(plan_sizes_ok(B, P, NA) && C >= 1 && ceil_div(C, 32) <= 65535, "segment_sum: bad size");
    FFB6D_CHECK_ARG(grad && plan && out, "segment_sum: null pointer");
    FFB6D_CHECK_ARG(((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(out)) & 3) == 0,
                    "segment_sum: grad and out must be 4-byte aligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(plan) & 15) == 0, "segment_sum: plan must be 16-byte aligned");
    FFB6D_CHECK_ARG(plan_bytes >= ffb6d_segment_plan_bytes(B, P, NA), "segment_sum: plan too small");
    const dim3 grid((unsigned)ceil_div(NA, SS_WARPS), (unsigned)ceil_div(C, 32), (unsigned)B);
    segment_sum_kernel<<<grid, 32 * SS_WARPS, 0, (cudaStream_t)stream>>>(grad, (const int *)plan, plan_frame_ints(P, NA),
                                                                       (int)C, (int)P, (int)NA, out);
    FFB6D_LAUNCH_OK("segment_sum_kernel");
    return FFB6D_OK;
}

size_t ffb6d_segment_csr_bytes(int64_t B, int64_t P, int64_t NA)
{
    return csr_bytes(B, P, NA);
}

int ffb6d_segment_csr(const void *idx, int idx_is_i64, int64_t B, int64_t P, int64_t NA, void *plan, size_t plan_bytes,
                      ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(csr_sizes_ok(B, P, NA), "segment_csr: bad size");
    FFB6D_CHECK_ARG(idx_is_i64 == 0 || idx_is_i64 == 1, "segment_csr: idx_is_i64=%d", idx_is_i64);
    FFB6D_CHECK_ARG(idx && plan, "segment_csr: null pointer");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(idx) & (idx_is_i64 ? 7 : 3)) == 0, "segment_csr: idx misaligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(plan) & 15) == 0, "segment_csr: plan must be 16-byte aligned");
    FFB6D_CHECK_ARG(plan_bytes >= csr_bytes(B, P, NA), "segment_csr: plan too small");
    return csr_build(idx, idx_is_i64, B, P, NA, plan, (cudaStream_t)stream);
}

int ffb6d_segment_sum_csr(const float *grad, const void *plan, size_t plan_bytes, int64_t B, int64_t C, int64_t P, int64_t NA,
                          float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(csr_sizes_ok(B, P, NA) && C >= 1 && ceil_div(C, 32) <= 65535, "segment_sum_csr: bad size");
    FFB6D_CHECK_ARG(grad && plan && out, "segment_sum_csr: null pointer");
    FFB6D_CHECK_ARG(((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(out)) & 3) == 0,
                    "segment_sum_csr: grad and out must be 4-byte aligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(plan) & 15) == 0, "segment_sum_csr: plan must be 16-byte aligned");
    FFB6D_CHECK_ARG(plan_bytes >= csr_bytes(B, P, NA), "segment_sum_csr: plan too small");
    const dim3 grid((unsigned)ceil_div(NA, SS_WARPS), (unsigned)ceil_div(C, 32), (unsigned)B);
    segment_sum_kernel<<<grid, 32 * SS_WARPS, 0, (cudaStream_t)stream>>>(grad, (const int *)plan, csr_layout(P, NA).frame,
                                                                       (int)C, (int)P, (int)NA, out);
    FFB6D_LAUNCH_OK("segment_sum_kernel");
    return FFB6D_OK;
}

size_t ffb6d_gather_max_bwd_det_workspace_bytes(int64_t B, int64_t C, int64_t S, int64_t Q, int K)
{
    if (B < 1 || C < 1 || S < 1 || Q < 1 || K < 1 || K > FFB6D_MAX_K || C > 65535ll * 32 || Q * K >= (1ll << 31))
        return 0;
    const size_t plan = csr_bytes(B, Q * K, S);
    if (plan == 0) return 0;
    return plan + (K > 1 ? align_up((size_t)B * C * Q, 16) : 0);
}

int ffb6d_gather_max_bwd_det(const float *feat, const void *idx, int idx_is_i64, const float *grad_out, int64_t B, int64_t C,
                             int64_t S, int64_t Q, int K, int layout, void *workspace, size_t workspace_bytes,
                             float *grad_feat, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && C >= 0 && S >= 0 && Q >= 0, "gather_max_bwd_det: negative size");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "gather_max_bwd_det: K=%d outside [1,%d]", K, FFB6D_MAX_K);
    FFB6D_CHECK_ARG(layout == FFB6D_LAYOUT_NCS || layout == FFB6D_LAYOUT_NSC, "gather_max_bwd_det: unknown layout %d", layout);
    FFB6D_CHECK_ARG(idx_is_i64 == 0 || idx_is_i64 == 1, "gather_max_bwd_det: idx_is_i64=%d", idx_is_i64);
    cudaStream_t st = (cudaStream_t)stream;
    if (B == 0 || C == 0 || Q == 0) {                   // nothing gathered: a zero gradient
        if (B * C * S > 0) {
            FFB6D_CHECK_ARG(grad_feat, "gather_max_bwd_det: null pointer");
            FFB6D_CUDA(cudaMemsetAsync(grad_feat, 0, (size_t)B * C * S * sizeof(float), st));
        }
        return FFB6D_OK;
    }
    const size_t need = ffb6d_gather_max_bwd_det_workspace_bytes(B, C, S, Q, K);
    FFB6D_CHECK_ARG(need > 0, "gather_max_bwd_det: bad size");
    FFB6D_CHECK_ARG(feat && idx && grad_out && grad_feat && workspace, "gather_max_bwd_det: null pointer");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(idx) & (idx_is_i64 ? 7 : 3)) == 0, "gather_max_bwd_det: idx misaligned");
    FFB6D_CHECK_ARG(((reinterpret_cast<uintptr_t>(feat) | reinterpret_cast<uintptr_t>(grad_out) |
                      reinterpret_cast<uintptr_t>(grad_feat)) & 3) == 0,
                    "gather_max_bwd_det: feat, grad_out and grad_feat must be 4-byte aligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "gather_max_bwd_det: workspace must be 16-byte aligned");
    FFB6D_CHECK_ARG(workspace_bytes >= need, "gather_max_bwd_det: workspace too small");
    const int64_t P = Q * K;
    int rc = csr_build(idx, idx_is_i64, B, P, S, workspace, st);
    if (rc != FFB6D_OK) return rc;
    unsigned char *amap = nullptr;
    if (K > 1) {
        amap = (unsigned char *)workspace + csr_bytes(B, P, S);
        const long long total = (long long)B * C * Q;
        const unsigned blocks = (unsigned)ceil_div(total, 256);
        if (idx_is_i64)
            gather_argmax_kernel<long long><<<blocks, 256, 0, st>>>(feat, (const long long *)idx, amap, (int)C, (int)S, (int)Q,
                                                                   K, layout, total);
        else
            gather_argmax_kernel<int><<<blocks, 256, 0, st>>>(feat, (const int *)idx, amap, (int)C, (int)S, (int)Q, K, layout,
                                                             total);
        FFB6D_LAUNCH_OK("gather_argmax_kernel");
    }
    const bool ncs = layout == FFB6D_LAYOUT_NCS;
    return masked_sum_launch(grad_out, amap, C * Q, ncs ? Q : 1, ncs ? 1 : C, K, (const int *)workspace, csr_layout(P, S), B, C,
                             S, grad_feat, C * S, ncs ? S : 1, ncs ? 1 : C, st);
}

size_t ffb6d_gather_neighbour_bwd_det_workspace_bytes(int64_t B, int64_t S, int64_t N, int K)
{
    if (K < 1 || N < 1 || (int64_t)N * K >= (1ll << 31)) return 0;
    return csr_bytes(B, N * K, S);
}

int ffb6d_gather_neighbour_bwd_det(const float *grad_out, const void *idx, int idx_is_i64, int64_t B, int64_t S, int64_t D,
                                   int64_t N, int K, void *workspace, size_t workspace_bytes, float *grad_pc,
                                   ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && S >= 0 && D >= 0 && N >= 0 && K >= 0, "gather_neighbour_bwd_det: negative size");
    FFB6D_CHECK_ARG(idx_is_i64 == 0 || idx_is_i64 == 1, "gather_neighbour_bwd_det: idx_is_i64=%d", idx_is_i64);
    cudaStream_t st = (cudaStream_t)stream;
    if (B == 0 || D == 0 || N == 0 || K == 0) {
        if (B * S * D > 0) {
            FFB6D_CHECK_ARG(grad_pc, "gather_neighbour_bwd_det: null pointer");
            FFB6D_CUDA(cudaMemsetAsync(grad_pc, 0, (size_t)B * S * D * sizeof(float), st));
        }
        return FFB6D_OK;
    }
    const size_t need = ffb6d_gather_neighbour_bwd_det_workspace_bytes(B, S, N, K);
    FFB6D_CHECK_ARG(need > 0 && ceil_div(D, 32) <= 65535, "gather_neighbour_bwd_det: bad size");
    FFB6D_CHECK_ARG(grad_out && idx && grad_pc && workspace, "gather_neighbour_bwd_det: null pointer");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(idx) & (idx_is_i64 ? 7 : 3)) == 0, "gather_neighbour_bwd_det: idx misaligned");
    FFB6D_CHECK_ARG(((reinterpret_cast<uintptr_t>(grad_out) | reinterpret_cast<uintptr_t>(grad_pc)) & 3) == 0,
                    "gather_neighbour_bwd_det: grad_out and grad_pc must be 4-byte aligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0,
                    "gather_neighbour_bwd_det: workspace must be 16-byte aligned");
    FFB6D_CHECK_ARG(workspace_bytes >= need, "gather_neighbour_bwd_det: workspace too small");
    const int64_t P = N * K;
    const int rc = csr_build(idx, idx_is_i64, B, P, S, workspace, st);
    if (rc != FFB6D_OK) return rc;
    // grad_out [B, N*K, D] read as channel d of entry (n, k): the transposed gradient, without a transpose
    return masked_sum_launch(grad_out, nullptr, P * D, 1, D, 1, (const int *)workspace, csr_layout(P, S), B, D, S, grad_pc,
                             S * D, 1, D, st);
}

}  // extern "C"
