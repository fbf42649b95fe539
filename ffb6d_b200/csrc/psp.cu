// psp.cu -- pyramid pooling of PSPNet's PSPModule (models/cnn/pspnet.py:19-28) on sm_90a: AdaptiveAvgPool2d at the
// sizes 1, 2, 3 and 6 (the 50 bins of every channel) in one read of the feature map (DESIGN.md 4.17).
//
// torch's bins (aten/src/ATen/native/AdaptiveAveragePooling.cpp): bin i of s along an axis of length n covers
// [floor(i n / s), ceil((i + 1) n / s)); neighbouring bins overlap when s does not divide n, and repeat when n < s.
// One CTA per (frame, channel) plane.  Pass 1: every warp takes whole rows, and each lane adds its columns into
// the 12 column ranges of the four sizes (1 + 2 + 3 + 6); the warp's sums of a row go to shared memory in fp64.
// Pass 2: one thread per bin adds the row sums of its row range in fp64 and divides by the bin's area once.
// The output is scale-major: four blocks [B, C, s, s] (s = 1, 2, 3, 6) one after the other, each equal to
// adaptive_avg_pool2d(x, s).
#include "common.cuh"

namespace ffb6d {

constexpr int POOL_THREADS = 256;
constexpr int POOL_RANGES = 12;        // column (and row) ranges of the four sizes
constexpr int POOL_BINS = 50;
constexpr int POOL_MAX_H = 1024;       // fp64 row sums in shared memory: 96 KB

__device__ __forceinline__ void pool_range(int r, int n, int &lo, int &hi, int &s, int &i)
{
    // range r of 12: sizes 1 (r = 0), 2 (1-2), 3 (3-5), 6 (6-11)
    s = (r == 0) ? 1 : (r < 3) ? 2 : (r < 6) ? 3 : 6;
    i = r - ((s == 1) ? 0 : (s == 2) ? 1 : (s == 3) ? 3 : 6);
    lo = (int)(((long long)i * n) / s);
    hi = (int)(((long long)(i + 1) * n + s - 1) / s);
}

__global__ void __launch_bounds__(POOL_THREADS)
psp_pool_kernel(const float *__restrict__ x, int B, int C, int H, int W, float *__restrict__ out)
{
    extern __shared__ double rowsum[];   // [H][12]
    __shared__ int clo[POOL_RANGES], chi[POOL_RANGES];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const long long plane = blockIdx.x;  // b * C + c
    const float *xp = x + (size_t)plane * H * W;
    if (tid < POOL_RANGES) {
        int s, i;
        pool_range(tid, W, clo[tid], chi[tid], s, i);
    }
    __syncthreads();
    int lo[POOL_RANGES], hi[POOL_RANGES];
#pragma unroll
    for (int r = 0; r < POOL_RANGES; ++r) {
        lo[r] = clo[r];
        hi[r] = chi[r];
    }
    for (int y = wid; y < H; y += POOL_THREADS / 32) {
        const float *row = xp + (size_t)y * W;
        float acc[POOL_RANGES];
#pragma unroll
        for (int r = 0; r < POOL_RANGES; ++r) acc[r] = 0.f;
        for (int c = lane; c < W; c += 32) {   // a lane adds W / 32 values per range (3 at W = 80) in fp32
            const float v = __ldg(row + c);
#pragma unroll
            for (int r = 0; r < POOL_RANGES; ++r)
                if (c >= lo[r] && c < hi[r]) acc[r] += v;
        }
#pragma unroll
        for (int r = 0; r < POOL_RANGES; ++r) {
            double d = (double)acc[r];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (lane == 0) rowsum[y * POOL_RANGES + r] = d;
        }
    }
    __syncthreads();
    if (tid < POOL_BINS) {
        // bin tid: size s, row range i, column range j; its block of the output starts at bin offset off
        const int s = (tid == 0) ? 1 : (tid < 5) ? 2 : (tid < 14) ? 3 : 6;
        const int off = (s == 1) ? 0 : (s == 2) ? 1 : (s == 3) ? 5 : 14;
        const int first = (s == 1) ? 0 : (s == 2) ? 1 : (s == 3) ? 3 : 6;   // the size's first range of the 12
        const int i = (tid - off) / s, j = (tid - off) % s;
        const int y0 = (int)(((long long)i * H) / s), y1 = (int)(((long long)(i + 1) * H + s - 1) / s);
        const int r = first + j;
        double acc = 0.0;
        for (int y = y0; y < y1; ++y) acc += rowsum[y * POOL_RANGES + r];
        const double area = (double)(y1 - y0) * (double)(chi[r] - clo[r]);
        out[(size_t)B * C * off + (size_t)plane * s * s + i * s + j] = (float)(acc / area);
    }
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_psp_pool(const float *x, int64_t B, int64_t C, int64_t H, int64_t W, float *out,
                              ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && C >= 1 && H >= 1 && W >= 1, "psp_pool: bad size");
    FFB6D_CHECK_ARG(H <= POOL_MAX_H && W < (1ll << 24) && B * C < (1ll << 31) && B * C * 50 < (1ll << 40) &&
                        H * W < (1ll << 31),
                    "psp_pool: size too large (H <= %d)", POOL_MAX_H);
    FFB6D_CHECK_ARG(x && out, "psp_pool: null pointer");
    const size_t smem = (size_t)H * POOL_RANGES * sizeof(double);
    if (smem > 48 * 1024) FFB6D_OPTIN_SMEM(psp_pool_kernel, POOL_MAX_H * POOL_RANGES * sizeof(double));
    psp_pool_kernel<<<(unsigned)(B * C), POOL_THREADS, smem, (cudaStream_t)stream>>>(x, (int)B, (int)C, (int)H, (int)W,
                                                                                       out);
    FFB6D_LAUNCH_OK("psp_pool_kernel");
    return FFB6D_OK;
}
