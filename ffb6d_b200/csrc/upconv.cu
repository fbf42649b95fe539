// upconv.cu -- PSPUpsample (models/cnn/pspnet.py:36-48: x2 bilinear upsampling with align_corners=True, 3x3 conv,
// BatchNorm, PReLU) at the input's resolution (DESIGN.md 4.23).
//
// Upsampling and a shift of the grid act on every channel alike, so they commute with the conv's channel mixing.  With
// W_t = W[:, :, ky, kx] (t = 3 ky + kx) and S_t the shift to tap t on the upsampled grid (zero outside it):
//
//     conv3x3(up(x)) + b  =  b + sum_t S_t(up(W_t x))
//
// The stacked product T = [W_0; ..; W_8] x is one packed GEMM at the input's resolution (ffb6d_fusion_mlp_fwd_ex);
// the kernels here are its epilogue (the nine shifted, upsampled planes of T added per output element), that
// epilogue's adjoint, and the PReLU of the training path.  The taps are torch's (AcAxis, psp.cuh), all four read even
// at weight 0 as torch's upsampling reads them, so a non-finite input spreads to every output it reaches in torch.
// No kernel uses atomics: every output element is written by one thread, its sum taken in a fixed order.
#include "common.cuh"
#include "psp.cuh"

#include <algorithm>

namespace ffb6d {

constexpr int UPC_THREADS = 256;
constexpr long long UPC_MAX_BLOCKS = 1ll << 20;

// out[b, co0 + j, y, x] = act(affine(bias + sum_t sum_4 lambda * T[b, t Cc + j, src])) for the Cc channels of a chunk;
// T [B, 9 Cc, Hi, Wi].  Taps in the order t = 0..8, and within a tap as torch's bilinear forward adds them.
__global__ void __launch_bounds__(UPC_THREADS)
upconv_taps_fwd_kernel(const float *__restrict__ table, int B, int Co, int co0, int Cc, int Hi, int Wi,
                       const float *__restrict__ bias, const float *__restrict__ scale, const float *__restrict__ shift,
                       const float *__restrict__ alpha, float *__restrict__ out)
{
    const int Ho = 2 * Hi, Wo = 2 * Wi;
    const AcAxis ay = ac_axis(Hi, Ho), ax = ac_axis(Wi, Wo);
    const size_t HWi = (size_t)Hi * Wi;
    const long long n = (long long)B * Cc * Ho * Wo;
    const float a = alpha ? __ldg(alpha) : 0.f;
    for (long long e = (long long)blockIdx.x * UPC_THREADS + threadIdx.x; e < n;
         e += (long long)gridDim.x * UPC_THREADS) {
        const int x = (int)(e % Wo);
        long long q = e / Wo;
        const int y = (int)(q % Ho);
        q /= Ho;
        const int j = (int)(q % Cc), b = (int)(q / Cc), co = co0 + j;
        const float *tb = table + ((size_t)b * 9 * Cc + j) * HWi;
        float acc = 0.f;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int Y = y + ky - 1;
            if (Y < 0 || Y >= Ho) continue;
            int h0, h1;
            float hl0, hl1;
            ay.taps(Y, h0, h1, hl0, hl1);
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int X = x + kx - 1;
                if (X < 0 || X >= Wo) continue;
                int w0, w1;
                float wl0, wl1;
                ax.taps(X, w0, w1, wl0, wl1);
                const float *p = tb + (size_t)(3 * ky + kx) * Cc * HWi;
                const float *r0 = p + (size_t)h0 * Wi, *r1 = p + (size_t)h1 * Wi;
                acc += hl0 * (wl0 * __ldg(r0 + w0) + wl1 * __ldg(r0 + w1)) +
                       hl1 * (wl0 * __ldg(r1 + w0) + wl1 * __ldg(r1 + w1));
            }
        }
        float v = (bias ? __ldg(bias + co) : 0.f) + acc;
        if (scale) v = __fmaf_rn(v, __ldg(scale + co), __ldg(shift + co));
        if (alpha) v = (v > 0.f) ? v : a * v;
        out[(((size_t)b * Co + co) * Ho + y) * Wo + x] = v;
    }
}

// G[b, t Cc + j, vy, vx] = up^T(S_t^T grad_z[b, co0 + j]) at (vy, vx): the output positions whose tap-t shift lands on
// an upsampled position that taps (vy, vx), in ascending row then column order, each product
// (lambda_y * lambda_x) * grad added in fp64 (weight-0 taps included), rounded once.  The walk over the upsampled
// positions is that of upsample_bilinear_ac_bwd_kernel (psp.cu), on the grid shifted by (ky - 1, kx - 1).
__global__ void __launch_bounds__(UPC_THREADS)
upconv_taps_bwd_kernel(const float *__restrict__ gz, int B, int Co, int co0, int Cc, int Hi, int Wi,
                       float *__restrict__ gt)
{
    const int Ho = 2 * Hi, Wo = 2 * Wi;
    const AcAxis ay = ac_axis(Hi, Ho), ax = ac_axis(Wi, Wo);
    const long long n = (long long)B * 9 * Cc * Hi * Wi;
    for (long long e = (long long)blockIdx.x * UPC_THREADS + threadIdx.x; e < n;
         e += (long long)gridDim.x * UPC_THREADS) {
        const int vx = (int)(e % Wi);
        long long q = e / Wi;
        const int vy = (int)(q % Hi);
        q /= Hi;
        const int r = (int)(q % (9 * Cc)), b = (int)(q / (9 * Cc));
        const int t = r / Cc, j = r - t * Cc, ky = t / 3, kx = t - 3 * ky;
        const float *g = gz + ((size_t)b * Co + co0 + j) * Ho * Wo;
        const int Y0 = ay.first_ge(vy - 1), Y1 = ay.first_ge(vy + 1);
        const int X0 = ax.first_ge(vx - 1), X1 = ax.first_ge(vx + 1);
        double acc = 0.0;
        for (int Y = Y0; Y < Y1; ++Y) {
            const int y = Y - ky + 1;
            if (y < 0 || y >= Ho) continue;
            bool hy0, hy1;
            float ly0, ly1;
            ay.tap(Y, vy, hy0, ly0, hy1, ly1);
            const float *row = g + (size_t)y * Wo;
            for (int X = X0; X < X1; ++X) {
                const int x = X - kx + 1;
                if (x < 0 || x >= Wo) continue;
                bool hx0, hx1;
                float lx0, lx1;
                ax.tap(X, vx, hx0, lx0, hx1, lx1);
                const float v = __ldg(row + x);
                if (hy0 && hx0) acc += (double)__fmul_rn(__fmul_rn(ly0, lx0), v);
                if (hy0 && hx1) acc += (double)__fmul_rn(__fmul_rn(ly0, lx1), v);
                if (hy1 && hx0) acc += (double)__fmul_rn(__fmul_rn(ly1, lx0), v);
                if (hy1 && hx1) acc += (double)__fmul_rn(__fmul_rn(ly1, lx1), v);
            }
        }
        gt[e] = (float)acc;
    }
}

// nn.PReLU() with one alpha, read on the device: y = x > 0 ? x : alpha x (NaN stays NaN).  x may be y.
__global__ void __launch_bounds__(UPC_THREADS)
prelu_fwd_kernel(const float *x, long long n, const float *__restrict__ alpha, float *y)
{
    const float a = __ldg(alpha);
    for (long long i = (long long)blockIdx.x * UPC_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * UPC_THREADS) {
        const float v = x[i];
        y[i] = (v > 0.f) ? v : a * v;
    }
}

// Backward of PReLU(BatchNorm(z)) down to the BatchNorm's output, one CTA per (frame, channel) row: the BatchNorm
// output is recomputed from z and the forward's stats as bn_apply_kernel (train.cu) computes it, u = (z - mean) *
// (gamma invstd) + beta; grad_u = u > 0 ? g : alpha g, and the row's share of grad_alpha, sum of (u > 0 ? 0 : u g), in
// fp64: each thread adds its columns in order, then a fixed shuffle tree and the warps in order.
__global__ void __launch_bounds__(UPC_THREADS)
bn_prelu_bwd_kernel(const float *__restrict__ z, const float *__restrict__ g, const float4 *__restrict__ stats, int C,
                    long long P, const float *__restrict__ alpha, float *__restrict__ gu, double *__restrict__ part)
{
    __shared__ double red[UPC_THREADS / 32];
    const size_t row = blockIdx.x;
    const float4 st = stats[row % C];
    const float a = __ldg(alpha);
    const float *zr = z + row * P, *gr = g + row * P;
    float *ur = gu + row * P;
    double acc = 0.0;
    for (long long p = threadIdx.x; p < P; p += UPC_THREADS) {
        const float u = __fmaf_rn(__fsub_rn(__ldg(zr + p), st.x), st.z, st.w), gv = __ldg(gr + p);
        if (u > 0.f) {
            ur[p] = gv;
        } else {
            ur[p] = a * gv;
            acc += (double)__fmul_rn(u, gv);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < UPC_THREADS / 32; ++w) s += red[w];
        part[row] = s;
    }
}

static inline bool misaligned(const void *p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

static inline unsigned grid_for(long long n)
{
    return (unsigned)std::min<long long>((n + UPC_THREADS - 1) / UPC_THREADS, UPC_MAX_BLOCKS);
}

static int upconv_sizes_ok(const char *name, int64_t B, int64_t Co, int64_t co0, int64_t Cc, int64_t Hi, int64_t Wi)
{
    FFB6D_CHECK_ARG(B >= 1 && Co >= 1 && co0 >= 0 && Cc >= 1 && Hi >= 1 && Wi >= 1 && co0 < Co && Cc <= Co - co0,
                    "%s: bad size", name);
    FFB6D_CHECK_ARG(Hi < (1ll << 23) && Wi < (1ll << 23) && B * Co < (1ll << 31) && B * 9 * Cc < (1ll << 31) &&
                        B * Co * Hi * Wi < (1ll << 48) && B * 9 * Cc * Hi * Wi < (1ll << 50),
                    "%s: size too large", name);
    return FFB6D_OK;
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_upconv_taps_fwd(const float *table, int64_t B, int64_t Co, int64_t co0, int64_t Cc, int64_t Hi,
                                     int64_t Wi, const float *bias, const float *scale, const float *shift,
                                     const float *alpha, float *out, ffb6d_stream_t stream)
{
    const int rc = upconv_sizes_ok("upconv_taps_fwd", B, Co, co0, Cc, Hi, Wi);
    if (rc != FFB6D_OK) return rc;
    FFB6D_CHECK_ARG(table && out, "upconv_taps_fwd: null pointer");
    FFB6D_CHECK_ARG((scale == nullptr) == (shift == nullptr), "upconv_taps_fwd: scale and shift come together");
    FFB6D_CHECK_ARG(!misaligned(table, 4) && !misaligned(out, 4) && !misaligned(bias, 4) && !misaligned(scale, 4) &&
                        !misaligned(shift, 4) && !misaligned(alpha, 4),
                    "upconv_taps_fwd: pointers must be 4-byte aligned");
    const long long n = B * Cc * 4 * Hi * Wi;
    upconv_taps_fwd_kernel<<<grid_for(n), UPC_THREADS, 0, (cudaStream_t)stream>>>(
        table, (int)B, (int)Co, (int)co0, (int)Cc, (int)Hi, (int)Wi, bias, scale, shift, alpha, out);
    FFB6D_LAUNCH_OK("upconv_taps_fwd_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_upconv_taps_bwd(const float *grad_z, int64_t B, int64_t Co, int64_t co0, int64_t Cc, int64_t Hi,
                                     int64_t Wi, float *grad_table, ffb6d_stream_t stream)
{
    const int rc = upconv_sizes_ok("upconv_taps_bwd", B, Co, co0, Cc, Hi, Wi);
    if (rc != FFB6D_OK) return rc;
    FFB6D_CHECK_ARG(grad_z && grad_table, "upconv_taps_bwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned(grad_z, 4) && !misaligned(grad_table, 4),
                    "upconv_taps_bwd: pointers must be 4-byte aligned");
    const long long n = B * 9 * Cc * Hi * Wi;
    upconv_taps_bwd_kernel<<<grid_for(n), UPC_THREADS, 0, (cudaStream_t)stream>>>(
        grad_z, (int)B, (int)Co, (int)co0, (int)Cc, (int)Hi, (int)Wi, grad_table);
    FFB6D_LAUNCH_OK("upconv_taps_bwd_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_prelu_fwd(const float *x, int64_t n, const float *alpha, float *y, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(n >= 1, "prelu_fwd: bad size");
    FFB6D_CHECK_ARG(n < (1ll << 50), "prelu_fwd: size too large");
    FFB6D_CHECK_ARG(x && alpha && y, "prelu_fwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned(x, 4) && !misaligned(alpha, 4) && !misaligned(y, 4),
                    "prelu_fwd: pointers must be 4-byte aligned");
    prelu_fwd_kernel<<<grid_for(n), UPC_THREADS, 0, (cudaStream_t)stream>>>(x, n, alpha, y);
    FFB6D_LAUNCH_OK("prelu_fwd_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_bn_prelu_bwd(const float *z, const float *grad_y, const float *stats, int64_t B, int64_t C,
                                  int64_t P, const float *alpha, float *grad_u, double *grad_alpha_part,
                                  ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && C >= 1 && P >= 1, "bn_prelu_bwd: bad size");
    FFB6D_CHECK_ARG(B * C < (1ll << 31) && P < (1ll << 40) && B * C * P < (1ll << 50), "bn_prelu_bwd: size too large");
    FFB6D_CHECK_ARG(z && grad_y && stats && alpha && grad_u && grad_alpha_part, "bn_prelu_bwd: null pointer");
    FFB6D_CHECK_ARG(!misaligned(z, 4) && !misaligned(grad_y, 4) && !misaligned(alpha, 4) && !misaligned(grad_u, 4) &&
                        !misaligned(stats, 16) && !misaligned(grad_alpha_part, 8),
                    "bn_prelu_bwd: pointers must be aligned (stats 16 bytes, grad_alpha_part 8, the rest 4)");
    bn_prelu_bwd_kernel<<<(unsigned)(B * C), UPC_THREADS, 0, (cudaStream_t)stream>>>(
        z, grad_y, reinterpret_cast<const float4 *>(stats), (int)C, P, alpha, grad_u, grad_alpha_part);
    FFB6D_LAUNCH_OK("bn_prelu_bwd_kernel");
    return FFB6D_OK;
}
