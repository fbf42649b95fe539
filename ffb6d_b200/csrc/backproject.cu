// backproject.cu -- depth map -> the point sets the fusion schedule searches (sm_90a).
//
// The reference back-projects the depth image on the CPU (dpt_2_pcld, datasets/ycb/ycb_dataset.py:
// 165-176), keeps the organised cloud [H,W,3], samples N pixels from it (`choose`, :218-237) and
// slices stride-2/4/8 sub-grids out of it (:253-267).  Only those four point sets are ever searched
// (sr = 1 never is), so this kernel produces them directly from the depth map: the 3.7 MB organised
// cloud per frame is neither shipped to the GPU nor materialised on it; the host sends the depth
// map (1.2 MB) and `choose` (48 KB).
//
// Arithmetic is the reference's, which numpy evaluates in float64 (integer pixel grid minus a
// float64 intrinsic): x = ((col - cx) * d) / fx, y = ((row - cy) * d) / fy, z = d, each multiplied by
// the validity mask (d > 1e-8 ? 1 : 0 -- holes become signed zeros), then rounded once to float32
// where the reference casts (`cld.astype(np.float32)`, NN/knn.pyx:95-96).
#include "common.cuh"

namespace ffb6d {

__device__ __forceinline__ void backproject_px(const float *__restrict__ depth, int W, int row, int col,
                                               double fx, double fy, double cx, double cy, float *o)
{
    const float d = __ldg(depth + (size_t)row * W + col);
    const double msk = (d > 1e-8f) ? 1.0 : 0.0;
    const double dd = (double)d;
    o[0] = __double2float_rn(__dmul_rn(__ddiv_rn(__dmul_rn((double)col - cx, dd), fx), msk));
    o[1] = __double2float_rn(__dmul_rn(__ddiv_rn(__dmul_rn((double)row - cy, dd), fy), msk));
    o[2] = __double2float_rn(__dmul_rn(dd, msk));
}

// flat work list per frame: [0,N) sampled points, then the stride-2, -4, -8 sub-grids
__global__ void __launch_bounds__(256)
backproject_kernel(const float *__restrict__ depth, int H, int W, const double *__restrict__ intr,
                   int intr_per_frame, const int *__restrict__ choose, int N, float *__restrict__ cld,
                   float *__restrict__ p2, float *__restrict__ p4, float *__restrict__ p8)
{
    const int b = blockIdx.y;
    const int n2 = (H / 2) * (W / 2), n4 = (H / 4) * (W / 4), n8 = (H / 8) * (W / 8);
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N + n2 + n4 + n8) return;
    const double *k = intr + (intr_per_frame ? (size_t)b * 4 : 0);
    const double fx = k[0], fy = k[1], cx = k[2], cy = k[3];
    const float *dp = depth + (size_t)b * H * W;
    int row, col;
    float *o;
    if (t < N) {
        const int px = __ldg(choose + (size_t)b * N + t);
        row = px / W;
        col = px % W;
        o = cld + ((size_t)b * N + t) * 3;
    } else {
        int u = t - N, s, nw;
        float *base;
        if (u < n2) { s = 2; nw = W / 2; base = p2 + (size_t)b * n2 * 3; }
        else if ((u -= n2) < n4) { s = 4; nw = W / 4; base = p4 + (size_t)b * n4 * 3; }
        else { u -= n4; s = 8; nw = W / 8; base = p8 + (size_t)b * n8 * 3; }
        row = (u / nw) * s;
        col = (u % nw) * s;
        o = base + (size_t)u * 3;
    }
    float v[3];
    backproject_px(dp, W, row, col, fx, fy, cx, cy, v);
    o[0] = v[0];
    o[1] = v[1];
    o[2] = v[2];
}

// ------------------------------------------------------------------ valid-pixel compaction + seeded sampling
// The reference picks the network's N input points on the CPU (datasets/ycb/ycb_dataset.py:218-235):
// `choose = msk_dp.flatten().nonzero()`, then, with more than N valid pixels, a uniformly random subset of N of
// them (`np.random.shuffle` of a 0/1 mask), otherwise all of them repeated cyclically (`np.pad(..., 'wrap')`),
// and finally a random permutation of the N picks (`np.random.shuffle(sf_idx)`).  Here:
//   compact_valid_kernel : ordered stream compaction of the valid pixels of a frame (one CTA per frame)
//   sample_pixels_kernel : pick i = the image of i under a keyed pseudo-random PERMUTATION of [0, n_valid)
//                          (a 4-round Feistel network on the next even power of two, cycle-walked back into
//                          range): the first N images of a permutation are a random subset in random order, no
//                          sort and no selection needed; with n_valid < N a permutation of [0, N) taken modulo
//                          n_valid reproduces 'wrap' + shuffle.
// Same distribution and determinism per seed as the reference's recipe; numpy's Mersenne-Twister stream itself is
// not reproduced (the picks are equally valid, not identical).
constexpr int COMPACT_THREADS = 1024;

__global__ void __launch_bounds__(COMPACT_THREADS)
compact_valid_kernel(const float *__restrict__ depth, int HW, float min_depth, int *__restrict__ list, int *__restrict__ count)
{
    __shared__ int warp_tot[COMPACT_THREADS / 32];
    __shared__ int base_s;
    const int b = blockIdx.x;
    const float *d = depth + (size_t)b * HW;
    int *out = list + (size_t)b * HW;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    for (int p0 = 0; p0 < HW; p0 += 4 * COMPACT_THREADS) {
        const int p = p0 + 4 * threadIdx.x;
        bool v[4];
        int c = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            v[u] = (p + u < HW) && (__ldg(d + min(p + u, HW - 1)) > min_depth);
            c += v[u] ? 1 : 0;
        }
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            int w = warp_tot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            warp_tot[lane] = w;
        }
        __syncthreads();
        int pos = base_s + (wid ? warp_tot[wid - 1] : 0) + incl - c;
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (v[u]) out[pos++] = p + u;
        __syncthreads();
        if (threadIdx.x == 0) base_s += warp_tot[COMPACT_THREADS / 32 - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) count[b] = base_s;
}

__device__ __forceinline__ unsigned mix32(unsigned x)
{
    x ^= x >> 16; x *= 0x85ebca6bu; x ^= x >> 13; x *= 0xc2b2ae35u; x ^= x >> 16;   // murmur3 finaliser
    return x;
}

// keyed bijection of [0, 2^(2*half)): four Feistel rounds
__device__ __forceinline__ unsigned feistel(unsigned x, int half, unsigned key)
{
    const unsigned mask = (1u << half) - 1u;
    unsigned l = x >> half, r = x & mask;
#pragma unroll
    for (int round = 0; round < 4; ++round) {
        const unsigned f = mix32(r * 0x9e3779b1u + key + (unsigned)round * 0x7f4a7c15u) & mask;
        const unsigned t = l ^ f;
        l = r;
        r = t;
    }
    return (l << half) | r;
}

__device__ __forceinline__ unsigned permute_below(unsigned i, unsigned n, unsigned key)
{
    int half = 1;
    while ((1u << (2 * half)) < n) ++half;
    unsigned x = i;
    do {
        x = feistel(x, half, key);
    } while (x >= n);   // cycle walking: stays a bijection of [0, n); expected < 4 steps
    return x;
}

__global__ void __launch_bounds__(256)
sample_pixels_kernel(const int *__restrict__ list, const int *__restrict__ count, int HW, int N, unsigned long long seed,
                     int *__restrict__ choose)
{
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int n = count[b];
    const unsigned key = mix32((unsigned)seed ^ mix32((unsigned)(seed >> 32) + 0x632be5abu * (unsigned)(b + 1)));
    int px = 0;
    if (n >= N) {
        px = list[(size_t)b * HW + permute_below((unsigned)i, (unsigned)n, key)];
    } else if (n > 0) {
        px = list[(size_t)b * HW + permute_below((unsigned)i, (unsigned)N, key) % (unsigned)n];   // 'wrap', shuffled
    }
    choose[(size_t)b * N + i] = px;
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_backproject(const float *depth, int64_t B, int64_t H, int64_t W,
                                 const double *intrinsics, int intrinsics_per_frame,
                                 const int *choose, int64_t N, float *cld, float *pyr2, float *pyr4,
                                 float *pyr8, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && H >= 8 && W >= 8 && N >= 0 && H * W < (1ll << 31) && B < 65536,
                    "backproject: bad size (B=%lld H=%lld W=%lld N=%lld)", (long long)B, (long long)H,
                    (long long)W, (long long)N);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(depth && intrinsics && cld && pyr2 && pyr4 && pyr8 && (N == 0 || choose),
                    "backproject: null pointer");
    const int64_t work = N + (H / 2) * (W / 2) + (H / 4) * (W / 4) + (H / 8) * (W / 8);
    dim3 grid((unsigned)ceil_div(work, 256), (unsigned)B);
    backproject_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(depth, (int)H, (int)W, intrinsics,
                                                              intrinsics_per_frame, choose, (int)N, cld,
                                                              pyr2, pyr4, pyr8);
    FFB6D_LAUNCH_OK("backproject_kernel");
    return FFB6D_OK;
}

extern "C" size_t ffb6d_sample_pixels_workspace_bytes(int64_t B, int64_t H, int64_t W)
{
    if (B <= 0 || H <= 0 || W <= 0) return 0;
    return align_up((size_t)B * (size_t)H * (size_t)W * sizeof(int), 256) + align_up((size_t)B * sizeof(int), 256);
}

extern "C" int ffb6d_sample_pixels(const float *depth, int64_t B, int64_t H, int64_t W, float min_depth, int64_t N,
                                   uint64_t seed, int *choose, int *valid_count, void *workspace, size_t workspace_bytes,
                                   ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && H >= 1 && W >= 1 && N >= 0 && H * W < (1ll << 30) && N < (1ll << 30) && B < 65536,
                    "sample_pixels: bad size");
    if (B == 0 || N == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(depth && choose && workspace, "sample_pixels: null pointer");
    FFB6D_CHECK_ARG(workspace_bytes >= ffb6d_sample_pixels_workspace_bytes(B, H, W), "sample_pixels: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int HW = (int)(H * W);
    int *list = (int *)workspace;
    int *count = (int *)((char *)workspace + align_up((size_t)B * HW * sizeof(int), 256));
    compact_valid_kernel<<<(unsigned)B, COMPACT_THREADS, 0, st>>>(depth, HW, min_depth, list, count);
    FFB6D_LAUNCH_OK("compact_valid_kernel");
    sample_pixels_kernel<<<dim3((unsigned)ceil_div(N, 256), (unsigned)B), 256, 0, st>>>(list, count, HW, (int)N, seed, choose);
    FFB6D_LAUNCH_OK("sample_pixels_kernel");
    if (valid_count) FFB6D_CUDA(cudaMemcpyAsync(valid_count, count, (size_t)B * sizeof(int), cudaMemcpyDeviceToDevice, st));
    return FFB6D_OK;
}
