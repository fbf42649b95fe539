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

}  // extern "C"
