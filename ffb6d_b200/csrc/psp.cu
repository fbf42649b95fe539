// psp.cu -- pyramid pooling of PSPNet's PSPModule (models/cnn/pspnet.py:19-28) on sm_90a: AdaptiveAvgPool2d at the
// sizes 1, 2, 3 and 6 (the 50 bins of every channel) in one read of the feature map (DESIGN.md 4.17).
//
// torch's bins (pool_range, psp.cuh): bin i of s along an axis of length n covers [floor(i n / s), ceil((i + 1) n / s));
// neighbouring bins overlap when s does not divide n, and repeat when n < s.
// One CTA per (frame, channel) plane.  Pass 1: every warp takes whole rows, and each lane adds its columns into
// the 12 column ranges of the four sizes (1 + 2 + 3 + 6); the warp's sums of a row go to shared memory in fp64.
// Pass 2: one thread per bin adds the row sums of its row range in fp64 and divides by the bin's area once.
// The output is scale-major: four blocks [B, C, s, s] (s = 1, 2, 3, 6) one after the other, each equal to
// adaptive_avg_pool2d(x, s).
//
// The adjoints of the PSP head's training path (DESIGN.md 4.18) live here too: the restructured bottleneck's backward
// (ReLU mask and the transposed bilinear taps of the four prior tables), the pooling's adjoint, the log-softmax
// backward of `final` and the align_corners=True bilinear upsampling backward of PSPUpsample.  None uses atomics: every
// output element is written by one thread, its sum taken in a fixed order, so the results are bit-identical from run
// to run and from graph replay to replay.
#include "common.cuh"
#include "psp.cuh"

#include <algorithm>

namespace ffb6d {

constexpr int POOL_THREADS = 256;
constexpr int POOL_RANGES = 12;        // column (and row) ranges of the four sizes
constexpr int POOL_BINS = 50;
constexpr int POOL_MAX_H = 1024;       // fp64 row sums in shared memory: 96 KB

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
        int k, s, off, i, j, y0, y1, s_, i_;
        psp_bin(tid, k, s, off, i, j);
        pool_range(psp_first_range(k) + i, H, y0, y1, s_, i_);   // the row range, from the same bounds as the columns
        const int r = psp_first_range(k) + j;
        double acc = 0.0;
        for (int y = y0; y < y1; ++y) acc += rowsum[y * POOL_RANGES + r];
        const double area = (double)(y1 - y0) * (double)(chi[r] - clo[r]);
        out[(size_t)B * C * off + (size_t)plane * s * s + i * s + j] = (float)(acc / area);
    }
}

// ===================================================================== backward of the PSP head (DESIGN.md 4.18)
constexpr int PSPB_THREADS = 256;
constexpr int PSPB_STRIDE = POOL_RANGES + 1;   // a row's 12 column-weighted sums and its plain sum (the bias)
constexpr int PSPB_MAX_SMEM = 227 * 1024;

__host__ __device__ __forceinline__ size_t pspb_smem_bytes(long long H, long long W)
{
    return (size_t)H * PSPB_STRIDE * sizeof(double) + (size_t)4 * (H + W) * sizeof(PspTap);
}

// The forward (fusion_mlp.cu) is out = relu(z), z = W_f x + b + sum_s up_s(T_s), up_s reading taps (psp_tap) of the
// channels-last table.  One CTA per (frame, output channel) plane, psp_pool_kernel run in reverse.  Pass 1: every warp
// takes whole rows; a lane masks its columns' gradient (torch's threshold_backward on the result: 0 where out <= 0,
// the gradient elsewhere, NaN out included), writes grad_z, and adds lambda_x * grad_z into the 12 column taps of the
// four sizes in fp64 (every tap, weight 0 included, as upsample_bilinear2d's backward does).  The warp's sums of a
// row go to shared memory.  Pass 2: one thread per bin adds lambda_y times the row sums of the rows that tap it, in
// ascending row order, in fp64; one more thread adds the rows' plain sums (the plane's share of the bias gradient).
__global__ void __launch_bounds__(PSPB_THREADS)
psp_bottleneck_bwd_kernel(const float *__restrict__ gout, const float *__restrict__ out, int B, int Co, int H, int W,
                          float *__restrict__ gz, float *__restrict__ gtable, float *__restrict__ gsum)
{
    extern __shared__ double rowsum[];   // [H][13], then the taps: columns [4][W], rows [4][H]
    PspTap *ctap = reinterpret_cast<PspTap *>(rowsum + (size_t)H * PSPB_STRIDE), *rtap = ctap + 4 * W;
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
    const long long plane = blockIdx.x;  // b * Co + co
    const int b = (int)(plane / Co), co = (int)(plane % Co);
    const size_t base = (size_t)plane * H * W;
    for (int t = tid; t < 4 * (H + W); t += PSPB_THREADS) {
        if (t < 4 * W)
            ctap[t] = psp_tap(t % W, W, psp_size_k(t / W));
        else
            rtap[t - 4 * W] = psp_tap((t - 4 * W) % H, H, psp_size_k((t - 4 * W) / H));
    }
    __syncthreads();
    for (int y = wid; y < H; y += PSPB_THREADS / 32) {
        double acc[PSPB_STRIDE];
#pragma unroll
        for (int r = 0; r < PSPB_STRIDE; ++r) acc[r] = 0.0;
        for (int c = lane; c < W; c += 32) {
            const size_t e = base + (size_t)y * W + c;
            const float o = __ldg(out + e), g = __ldg(gout + e);
            const float v = (o <= 0.f) ? 0.f : g;
            gz[e] = v;
            const double d = (double)v;
            acc[POOL_RANGES] += d;
            PspTap t[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) t[k] = ctap[k * W + c];
#pragma unroll
            for (int r = 0; r < POOL_RANGES; ++r) {
                const int k = psp_range_size_k(r), j = r - psp_first_range(k);
                if (t[k].i0 == j) acc[r] += (double)t[k].l0 * d;
                if (t[k].i1 == j) acc[r] += (double)t[k].l1 * d;
            }
        }
#pragma unroll
        for (int r = 0; r < PSPB_STRIDE; ++r) {
            double d = acc[r];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (lane == 0) rowsum[y * PSPB_STRIDE + r] = d;
        }
    }
    __syncthreads();
    if (tid < POOL_BINS) {
        int k, s, off, i, j;
        psp_bin(tid, k, s, off, i, j);
        const int r = psp_first_range(k) + j;
        double acc = 0.0;
        for (int y = 0; y < H; ++y) {
            const PspTap t = rtap[k * H + y];
            const double v = rowsum[y * PSPB_STRIDE + r];
            if (t.i0 == i) acc += (double)t.l0 * v;
            if (t.i1 == i) acc += (double)t.l1 * v;
        }
        // row (B * off + b * s * s + i * s + j) of the [B * 50, Co] table, as the forward reads it
        gtable[((size_t)B * off + (size_t)b * s * s + i * s + j) * Co + co] = (float)acc;
    } else if (tid == POOL_BINS) {
        double acc = 0.0;
        for (int y = 0; y < H; ++y) acc += rowsum[y * PSPB_STRIDE + POOL_RANGES];
        gsum[plane] = (float)acc;
    }
}

// Adjoint of psp_pool_kernel: grad_x[h, w] += sum over the 50 bins that contain (h, w) of grad_pooled[bin] / area(bin).
// One CTA per (frame, channel) plane: the plane's 50 bin values (divided by the area in fp64) and a 12-bit membership
// mask of every row and column go to shared memory; each thread then adds, for its pixels, the bins of the four sizes
// in block order (size, row bin, column bin) in fp64 and rounds once into the caller's grad_x.
constexpr int POOLB_MAX_W = 16384;

__global__ void __launch_bounds__(POOL_THREADS)
psp_pool_bwd_kernel(const float *__restrict__ gp, int B, int C, int H, int W, float *__restrict__ gx)
{
    extern __shared__ unsigned short mask[];   // rows [H], then columns [W]
    __shared__ double val[POOL_BINS];
    __shared__ int rlo[POOL_RANGES], rhi[POOL_RANGES], clo[POOL_RANGES], chi[POOL_RANGES];
    const int tid = threadIdx.x;
    const long long plane = blockIdx.x;  // b * C + c
    if (tid < POOL_RANGES) {
        int s, i;
        pool_range(tid, H, rlo[tid], rhi[tid], s, i);
        pool_range(tid, W, clo[tid], chi[tid], s, i);
    }
    __syncthreads();
    if (tid < POOL_BINS) {
        int k, s, off, i, j;
        psp_bin(tid, k, s, off, i, j);
        const int f = psp_first_range(k);
        const double area = (double)(rhi[f + i] - rlo[f + i]) * (double)(chi[f + j] - clo[f + j]);
        val[tid] = (double)__ldg(gp + (size_t)B * C * off + (size_t)plane * s * s + i * s + j) / area;
    }
    unsigned short *rmask = mask, *cmask = mask + H;
    for (int t = tid; t < H + W; t += POOL_THREADS) {
        const int v = (t < H) ? t : t - H;
        const int *lo = (t < H) ? rlo : clo, *hi = (t < H) ? rhi : chi;
        unsigned m = 0;
#pragma unroll
        for (int r = 0; r < POOL_RANGES; ++r)
            if (v >= lo[r] && v < hi[r]) m |= 1u << r;
        mask[t] = (unsigned short)m;
    }
    __syncthreads();
    float *g = gx + (size_t)plane * H * W;
    const int HW = H * W;
    for (int e = tid; e < HW; e += POOL_THREADS) {
        const int y = e / W, x = e - y * W;
        const unsigned rm = rmask[y], cm = cmask[x];
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int s = psp_size_k(k), f = psp_first_range(k), off = psp_bin_offset(k);
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                if (i >= s || !((rm >> (f + i)) & 1u)) continue;
#pragma unroll
                for (int j = 0; j < 6; ++j)
                    if (j < s && ((cm >> (f + j)) & 1u)) acc += val[off + i * s + j];
            }
        }
        g[e] = (float)((double)g[e] + acc);
    }
}

// Backward of log_softmax over the channels of out [B, C, P] (torch's _log_softmax_backward_data):
// grad_in = grad_out - exp(out) * sum_c grad_out.  One thread per pixel, coalesced across the pixels; the channel sum
// in fp64 in channel order, the rest in fp32 as torch.
constexpr int LSMB_THREADS = 256;

__global__ void __launch_bounds__(LSMB_THREADS)
log_softmax_bwd_kernel(const float *__restrict__ gout, const float *__restrict__ out, int C, long long P,
                       float *__restrict__ gin)
{
    const long long p = (long long)blockIdx.x * LSMB_THREADS + threadIdx.x;
    if (p >= P) return;
    const size_t base = (size_t)blockIdx.y * C * P + p;
    double sum = 0.0;
    for (int c = 0; c < C; ++c) sum += (double)__ldg(gout + base + (size_t)c * P);
    const float sf = (float)sum;
    for (int c = 0; c < C; ++c) {
        const size_t e = base + (size_t)c * P;
        gin[e] = __fsub_rn(__ldg(gout + e), __fmul_rn(expf(__ldg(out + e)), sf));
    }
}

// Backward of upsample_bilinear2d with align_corners=True (PSPUpsample's x2), in gather form.  Each tap is torch's
// float arithmetic (upsample_bilinear2d_backward_out_frame): scale = (float)(in - 1) / (out - 1) (0 when out == 1),
// src = scale * dst, i0 = (int)src, i1 = i0 + (i0 < in - 1), lambda1 = src - i0, lambda0 = 1 - lambda1.  Output
// coordinate dst taps input coordinate v iff i0(dst) is v - 1 or v; i0 is non-decreasing in dst, so those dst form
// one range, found from an estimate and then walked to its exact ends on the recomputed i0.  One thread per input
// element adds, for the output rows and then columns of its ranges in ascending order, each matching product
// (lambda_y * lambda_x) * grad in fp64 -- weight-0 taps included -- and rounds once.
constexpr int UPB_THREADS = 256;

__global__ void __launch_bounds__(UPB_THREADS)
upsample_bilinear_ac_bwd_kernel(const float *__restrict__ gout, long long planes, int Hi, int Wi, int Ho, int Wo,
                                float *__restrict__ gin)
{
    const AcAxis ay{(Ho > 1) ? (float)(Hi - 1) / (float)(Ho - 1) : 0.f, Hi, Ho};
    const AcAxis ax{(Wo > 1) ? (float)(Wi - 1) / (float)(Wo - 1) : 0.f, Wi, Wo};
    const long long n = planes * Hi * Wi;
    for (long long e = (long long)blockIdx.x * UPB_THREADS + threadIdx.x; e < n;
         e += (long long)gridDim.x * UPB_THREADS) {
        const int x = (int)(e % Wi);
        const long long q = e / Wi;
        const int y = (int)(q % Hi);
        const long long plane = q / Hi;
        const float *g = gout + (size_t)plane * Ho * Wo;
        const int y0 = ay.first_ge(y - 1), y1 = ay.first_ge(y + 1);
        const int x0 = ax.first_ge(x - 1), x1 = ax.first_ge(x + 1);
        double acc = 0.0;
        for (int ho = y0; ho < y1; ++ho) {
            bool hy0, hy1;
            float ly0, ly1;
            ay.tap(ho, y, hy0, ly0, hy1, ly1);
            const float *row = g + (size_t)ho * Wo;
            for (int wo = x0; wo < x1; ++wo) {
                bool hx0, hx1;
                float lx0, lx1;
                ax.tap(wo, x, hx0, lx0, hx1, lx1);
                const float v = __ldg(row + wo);
                // torch's order of the four taps: (h0, w0), (h0, w1), (h1, w0), (h1, w1)
                if (hy0 && hx0) acc += (double)__fmul_rn(__fmul_rn(ly0, lx0), v);
                if (hy0 && hx1) acc += (double)__fmul_rn(__fmul_rn(ly0, lx1), v);
                if (hy1 && hx0) acc += (double)__fmul_rn(__fmul_rn(ly1, lx0), v);
                if (hy1 && hx1) acc += (double)__fmul_rn(__fmul_rn(ly1, lx1), v);
            }
        }
        gin[e] = (float)acc;
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

static inline bool misaligned4(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 3) != 0; }

extern "C" int ffb6d_psp_bottleneck_bwd(const float *grad_out, const float *out, int64_t B, int64_t Co, int64_t H,
                                        int64_t W, float *grad_z, float *grad_table, float *grad_sum,
                                        ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && Co >= 1 && H >= 1 && W >= 1, "psp_bottleneck_bwd: bad size");
    FFB6D_CHECK_ARG(H <= 1024 && W <= 1024 && pspb_smem_bytes(H, W) <= (size_t)PSPB_MAX_SMEM && B * Co < (1ll << 31) &&
                        B * 50 * Co < (1ll << 40),
                    "psp_bottleneck_bwd: size too large (H, W <= 1024 and %d KB of shared memory)",
                    PSPB_MAX_SMEM / 1024);
    FFB6D_CHECK_ARG(grad_out && out && grad_z && grad_table && grad_sum, "psp_bottleneck_bwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned4(grad_out) && !misaligned4(out) && !misaligned4(grad_z) && !misaligned4(grad_table) &&
                        !misaligned4(grad_sum),
                    "psp_bottleneck_bwd: pointers must be 4-byte aligned");
    const size_t smem = pspb_smem_bytes(H, W);
    if (smem > 48 * 1024) FFB6D_OPTIN_SMEM(psp_bottleneck_bwd_kernel, PSPB_MAX_SMEM);
    psp_bottleneck_bwd_kernel<<<(unsigned)(B * Co), PSPB_THREADS, smem, (cudaStream_t)stream>>>(
        grad_out, out, (int)B, (int)Co, (int)H, (int)W, grad_z, grad_table, grad_sum);
    FFB6D_LAUNCH_OK("psp_bottleneck_bwd_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_psp_pool_bwd(const float *grad_pooled, int64_t B, int64_t C, int64_t H, int64_t W, float *grad_x,
                                  ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && C >= 1 && H >= 1 && W >= 1, "psp_pool_bwd: bad size");
    FFB6D_CHECK_ARG(H <= POOL_MAX_H && W <= POOLB_MAX_W && B * C < (1ll << 31) && B * C * 50 < (1ll << 40) &&
                        H * W < (1ll << 31),
                    "psp_pool_bwd: size too large (H <= %d, W <= %d)", POOL_MAX_H, POOLB_MAX_W);
    FFB6D_CHECK_ARG(grad_pooled && grad_x, "psp_pool_bwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned4(grad_pooled) && !misaligned4(grad_x), "psp_pool_bwd: pointers must be 4-byte aligned");
    const size_t smem = (size_t)(H + W) * sizeof(unsigned short);
    psp_pool_bwd_kernel<<<(unsigned)(B * C), POOL_THREADS, smem, (cudaStream_t)stream>>>(grad_pooled, (int)B, (int)C,
                                                                                          (int)H, (int)W, grad_x);
    FFB6D_LAUNCH_OK("psp_pool_bwd_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_log_softmax_bwd(const float *grad_out, const float *out, int64_t B, int64_t C, int64_t P,
                                     float *grad_in, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && C >= 1 && P >= 1, "log_softmax_bwd: bad size");
    FFB6D_CHECK_ARG(B < 65536 && C < (1ll << 31) && P < (1ll << 38) && C * P < (1ll << 50),
                    "log_softmax_bwd: size too large");
    FFB6D_CHECK_ARG(grad_out && out && grad_in, "log_softmax_bwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned4(grad_out) && !misaligned4(out) && !misaligned4(grad_in),
                    "log_softmax_bwd: pointers must be 4-byte aligned");
    const dim3 grid((unsigned)((P + LSMB_THREADS - 1) / LSMB_THREADS), (unsigned)B);
    log_softmax_bwd_kernel<<<grid, LSMB_THREADS, 0, (cudaStream_t)stream>>>(grad_out, out, (int)C, P, grad_in);
    FFB6D_LAUNCH_OK("log_softmax_bwd_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_upsample_bilinear2d_bwd(const float *grad_out, int64_t B, int64_t C, int64_t Hi, int64_t Wi,
                                             int64_t Ho, int64_t Wo, float *grad_in, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && C >= 1 && Hi >= 1 && Wi >= 1 && Ho >= 1 && Wo >= 1, "upsample_bilinear2d_bwd: bad size");
    FFB6D_CHECK_ARG(Hi < (1ll << 24) && Wi < (1ll << 24) && Ho < (1ll << 24) && Wo < (1ll << 24) &&
                        B * C < (1ll << 40) && B * C * Hi * Wi < (1ll << 50) && B * C * Ho * Wo < (1ll << 50),
                    "upsample_bilinear2d_bwd: size too large");
    FFB6D_CHECK_ARG(grad_out && grad_in, "upsample_bilinear2d_bwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned4(grad_out) && !misaligned4(grad_in),
                    "upsample_bilinear2d_bwd: pointers must be 4-byte aligned");
    const long long n = B * C * Hi * Wi;
    const long long blocks = std::min<long long>((n + UPB_THREADS - 1) / UPB_THREADS, 1ll << 20);
    upsample_bilinear_ac_bwd_kernel<<<(unsigned)blocks, UPB_THREADS, 0, (cudaStream_t)stream>>>(
        grad_out, B * C, (int)Hi, (int)Wi, (int)Ho, (int)Wo, grad_in);
    FFB6D_LAUNCH_OK("upsample_bilinear_ac_bwd_kernel");
    return FFB6D_OK;
}
