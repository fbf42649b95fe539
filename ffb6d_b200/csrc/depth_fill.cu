// depth_fill.cu -- the YCB dataset's depth completion on the device (sm_90a).
//
// datasets/ycb/ycb_dataset.py:204 completes every raw depth frame with
// bs_utils.fill_missing(dpt_um, cam_scale, 1) (utils/basic_utils.py:467-487): ip_basic's
// fill_in_multiscale (utils/ip_basic/ip_basic/depth_map_utils_ycb.py:290-443) with max_depth 3.0,
// no extrapolation and the bilateral blur.  The stages, on x = fl32(raw) / cam_scale:
//   bands_kernel        invert (3 - x where x > 0.01), near / med / far bands dilated by cross
//                       7x7 / 5x5 / 3x3 and combined far -> med -> near                       (s2)
//   morph5_kernel x2    5x5 close: dilate, then erode                                         (s3)
//   median5_kernel      5x5 median where s3 > 0.01                                            (s4)
//   top_row_kernel      first row > 0.01 of each column (the top mask)
//   fill9_kernel        empty pixels below the top mask take the 9x9 dilation                 (s5 = s6)
//   top_row_kernel      top mask of s5
//   fill5_kernel x6     pixels < 0.01 below the top mask take the 5x5 dilation                (s7)
//   median5_kernel      5x5 median on s7 > 0.01 & top mask; also the frame's min / max
//   bilateral_kernel    bilateral (d 5, sigma_color 0.5, sigma_space 2.0) on the same mask, invert
//                       back, * cam_scale (raw units) and / cam_scale (metres)
// Every stage but the bilateral is bit-identical to numpy + OpenCV: thresholds are float32 constants
// like numpy's casts, every fp32 operation is a separately rounded _rn intrinsic, dilation / erosion
// ignore out-of-image pixels (OpenCV's default morphology border), the median replicates the edge.
// The bilateral uses exact float64 weights where OpenCV interpolates a float32 table (DESIGN.md §4.10).
// Every kernel is a stencil over global memory (L1 serves the reuse); the two column scans and the
// frame min / max are what separate the launches.
#include <cfloat>

#include "common.cuh"

namespace ffb6d {
namespace {

constexpr float kT = 0.01f;        // np.float32(0.01): every > 0.01 / < 0.01 of fill_in_multiscale
constexpr float kMaxDepth = 3.0f;
constexpr int TX = 32, TY = 8;

struct Plane {
    int H, W;
    __device__ __forceinline__ size_t frame(int b) const { return (size_t)b * H * W; }
};

// s1 and band membership of one pixel: the band products of the reference are s1 * mask, which only
// ever reach the result through `> 0.01`, so a pixel outside the band contributes 0
__device__ __forceinline__ void band_px(const uint16_t *__restrict__ raw, size_t i, float cs, float &s1, int &band)
{
    const float x = __fdiv_rn((float)__ldg(raw + i), cs);
    s1 = x > kT ? __fsub_rn(kMaxDepth, x) : x;
    band = x > 2.0f ? 3 : x > 1.0f ? 2 : x > kT ? 1 : 0;     // far 3x3, med 5x5, near 7x7 (radius = 4 - band)
}

__global__ void __launch_bounds__(TX * TY)
bands_kernel(const uint16_t *__restrict__ raw, Plane p, float cs, float *__restrict__ s2, unsigned *__restrict__ minmax)
{
    const int c = blockIdx.x * TX + threadIdx.x, r = blockIdx.y * TY + threadIdx.y, b = blockIdx.z;
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0) {
        minmax[2 * b] = 0xffffffffu;     // reset the frame's min / max for median5_kernel's second call
        minmax[2 * b + 1] = 0u;
    }
    if (r >= p.H || c >= p.W) return;
    const uint16_t *f = raw + p.frame(b);
    float d[4] = {0.f, 0.f, 0.f, 0.f};   // dilated band of index 1 (near) .. 3 (far)
    float centre = 0.f;
#pragma unroll
    for (int o = -3; o <= 3; ++o) {
#pragma unroll
        for (int axis = 0; axis < 2; ++axis) {
            if (axis == 1 && o == 0) continue;
            const int rr = axis == 0 ? r + o : r, cc = axis == 0 ? c : c + o;
            if (rr < 0 || rr >= p.H || cc < 0 || cc >= p.W) continue;
            float s1;
            int band;
            band_px(f, (size_t)rr * p.W + cc, cs, s1, band);
            if (o == 0) centre = s1;
            const int ad = o < 0 ? -o : o;
            if (band > 0 && ad <= 4 - band) d[band] = fmaxf(d[band], s1);
        }
    }
    float v = centre;
    if (d[3] > kT) v = d[3];
    if (d[2] > kT) v = d[2];
    if (d[1] > kT) v = d[1];
    s2[p.frame(b) + (size_t)r * p.W + c] = v;
}

// 5x5 full dilation (max) or erosion (min); out-of-image pixels take no part
template <bool kMax>
__global__ void __launch_bounds__(TX * TY) morph5_kernel(const float *__restrict__ src, Plane p, float *__restrict__ dst)
{
    const int c = blockIdx.x * TX + threadIdx.x, r = blockIdx.y * TY + threadIdx.y, b = blockIdx.z;
    if (r >= p.H || c >= p.W) return;
    const float *f = src + p.frame(b);
    float m = kMax ? -INFINITY : INFINITY;
    for (int rr = max(r - 2, 0); rr <= min(r + 2, p.H - 1); ++rr)
        for (int cc = max(c - 2, 0); cc <= min(c + 2, p.W - 1); ++cc) {
            const float v = __ldg(f + (size_t)rr * p.W + cc);
            m = kMax ? fmaxf(m, v) : fminf(m, v);
        }
    dst[p.frame(b) + (size_t)r * p.W + c] = m;
}

__device__ __forceinline__ float dilate_at(const float *__restrict__ f, Plane p, int r, int c, int rad)
{
    float m = -INFINITY;
    for (int rr = max(r - rad, 0); rr <= min(r + rad, p.H - 1); ++rr)
        for (int cc = max(c - rad, 0); cc <= min(c + rad, p.W - 1); ++cc) m = fmaxf(m, __ldg(f + (size_t)rr * p.W + cc));
    return m;
}

// 13th of the 25 edge-replicated values: a bitonic sort of 32 (7 of them +inf), fully unrolled into registers
__device__ __forceinline__ float median25_at(const float *__restrict__ f, Plane p, int r, int c)
{
    float v[32];
#pragma unroll
    for (int i = 0; i < 25; ++i) {
        const int rr = min(max(r + i / 5 - 2, 0), p.H - 1), cc = min(max(c + i % 5 - 2, 0), p.W - 1);
        v[i] = __ldg(f + (size_t)rr * p.W + cc);
    }
#pragma unroll
    for (int i = 25; i < 32; ++i) v[i] = INFINITY;
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1)
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1)
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int l = i ^ j;
                if (l > i) {
                    const float a = v[i], bb = v[l];
                    const bool asc = (i & k) == 0;
                    v[i] = asc ? fminf(a, bb) : fmaxf(a, bb);
                    v[l] = asc ? fmaxf(a, bb) : fminf(a, bb);
                }
            }
    return v[12];
}

// order-preserving float <-> unsigned (no NaN can occur: the inputs are finite depths)
__device__ __forceinline__ unsigned ordered(float x)
{
    const unsigned u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unordered(unsigned u)
{
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// dst = src > 0.01 [& below the top mask] ? median : src.  With `top`, also the frame's min / max of dst
__global__ void __launch_bounds__(TX * TY)
median5_kernel(const float *__restrict__ src, Plane p, const int *__restrict__ top, float *__restrict__ dst,
               unsigned *__restrict__ minmax)
{
    const int c = blockIdx.x * TX + threadIdx.x, r = blockIdx.y * TY + threadIdx.y, b = blockIdx.z;
    const bool in = r < p.H && c < p.W;
    float out = 0.f;
    if (in) {
        const float *f = src + p.frame(b);
        const float v = __ldg(f + (size_t)r * p.W + c);
        const bool sel = v > kT && (top == nullptr || r >= __ldg(top + (size_t)b * p.W + c));
        out = sel ? median25_at(f, p, r, c) : v;
        dst[p.frame(b) + (size_t)r * p.W + c] = out;
    }
    if (top == nullptr) return;
    unsigned lo = in ? ordered(out) : 0xffffffffu, hi = in ? ordered(out) : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if ((threadIdx.x & 31) == 0) {     // min / max commute: the result does not depend on the order
        atomicMin(minmax + 2 * b, lo);
        atomicMax(minmax + 2 * b + 1, hi);
    }
}

// first row with a value > 0.01 in each column; 0 for a column without one (np.argmax of all-False)
__global__ void __launch_bounds__(128) top_row_kernel(const float *__restrict__ src, Plane p, int *__restrict__ top)
{
    const int c = blockIdx.x * 128 + threadIdx.x, b = blockIdx.y;
    if (c >= p.W) return;
    const float *f = src + p.frame(b) + c;
    int row = 0;
    for (int r = 0; r < p.H; ++r)
        if (__ldg(f + (size_t)r * p.W) > kT) {
            row = r;
            break;
        }
    top[(size_t)b * p.W + c] = row;
}

// s5: pixels not > 0.01 at or below the top row take the 9x9 dilation
__global__ void __launch_bounds__(TX * TY)
fill9_kernel(const float *__restrict__ src, Plane p, const int *__restrict__ top, float *__restrict__ dst)
{
    const int c = blockIdx.x * TX + threadIdx.x, r = blockIdx.y * TY + threadIdx.y, b = blockIdx.z;
    if (r >= p.H || c >= p.W) return;
    const float *f = src + p.frame(b);
    float v = __ldg(f + (size_t)r * p.W + c);
    if (!(v > kT) && r >= __ldg(top + (size_t)b * p.W + c)) v = dilate_at(f, p, r, c, 4);
    dst[p.frame(b) + (size_t)r * p.W + c] = v;
}

// one of the six masked hole fills: pixels < 0.01 at or below the top row take the 5x5 dilation
__global__ void __launch_bounds__(TX * TY)
fill5_kernel(const float *__restrict__ src, Plane p, const int *__restrict__ top, float *__restrict__ dst)
{
    const int c = blockIdx.x * TX + threadIdx.x, r = blockIdx.y * TY + threadIdx.y, b = blockIdx.z;
    if (r >= p.H || c >= p.W) return;
    const float *f = src + p.frame(b);
    float v = __ldg(f + (size_t)r * p.W + c);
    if (v < kT && r >= __ldg(top + (size_t)b * p.W + c)) v = dilate_at(f, p, r, c, 2);
    dst[p.frame(b) + (size_t)r * p.W + c] = v;
}

// index folded into [0, n) by reflection without repeating the edge (OpenCV's BORDER_REFLECT_101)
__device__ __forceinline__ int reflect101(int i, int n)
{
    if (n == 1) return 0;
    const int period = 2 * (n - 1);
    i %= period;
    if (i < 0) i += period;
    return i >= n ? period - i : i;
}

// Bilateral blur on the pixels the second median selected (mask taken from s7 BEFORE that median, like
// the reference), then the inversion back and the unit conversions.  The filter reads the median's
// output `s7m`; when the frame's max - min < FLT_EPSILON it copies (cv::bilateralFilter does).
__global__ void __launch_bounds__(TX * TY)
bilateral_kernel(const float *__restrict__ s7, const float *__restrict__ s7m, Plane p, const int *__restrict__ top,
                 const unsigned *__restrict__ minmax, float cs, float *__restrict__ filled_raw, float *__restrict__ depth_m)
{
    const int c = blockIdx.x * TX + threadIdx.x, r = blockIdx.y * TY + threadIdx.y, b = blockIdx.z;
    if (r >= p.H || c >= p.W) return;
    const size_t i = p.frame(b) + (size_t)r * p.W + c;
    const float *f = s7m + p.frame(b);
    float v = __ldg(s7m + i);
    const bool sel = __ldg(s7 + i) > kT && r >= __ldg(top + (size_t)b * p.W + c);
    const double span = (double)unordered(minmax[2 * b + 1]) - (double)unordered(minmax[2 * b]);
    if (sel && !(fabs(span) < (double)FLT_EPSILON)) {
        const double v0 = (double)v;
        double num = 0.0, den = 0.0;
#pragma unroll
        for (int dy = -2; dy <= 2; ++dy) {
            const int rr = reflect101(r + dy, p.H);
#pragma unroll
            for (int dx = -2; dx <= 2; ++dx) {
                const int r2 = dy * dy + dx * dx;
                if (r2 > 4) continue;
                const double x = (double)__ldg(f + (size_t)rr * p.W + reflect101(c + dx, p.W));
                const double d = x - v0;
                // -0.5 / sigma^2: sigma_space 2.0 -> -0.125, sigma_color 0.5 -> -2.0
                const double w = exp((double)r2 * -0.125) * exp(d * d * -2.0);
                num += x * w;
                den += w;
            }
        }
        v = __double2float_rn(num / den);
    }
    if (v > kT) v = __fsub_rn(kMaxDepth, v);
    const float out = __fmul_rn(__fdiv_rn(v, 1.0f), cs);      // final_dpt / scale_2_80m * cam_scale
    if (filled_raw) filled_raw[i] = out;
    if (depth_m) depth_m[i] = __fdiv_rn(out, cs);              // dpt_um.astype(np.float32) / cam_scale
}

struct Workspace {
    float *a, *b;
    int *top;
    unsigned *minmax;
};

bool size_ok(int64_t B, int64_t H, int64_t W)
{
    return B >= 0 && H >= 1 && W >= 1 && B < 65536 && H < 65535ll * TY && H * W < (1ll << 31);
}

size_t plane_bytes(int64_t B, int64_t H, int64_t W) { return align_up((size_t)B * H * W * sizeof(float), 256); }

Workspace carve(void *ws, int64_t B, int64_t H, int64_t W)
{
    char *p = (char *)ws;
    Workspace w;
    w.a = (float *)p;
    p += plane_bytes(B, H, W);
    w.b = (float *)p;
    p += plane_bytes(B, H, W);
    w.top = (int *)p;
    p += align_up((size_t)B * W * sizeof(int), 256);
    w.minmax = (unsigned *)p;
    return w;
}

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" size_t ffb6d_fill_depth_workspace_bytes(int64_t B, int64_t H, int64_t W)
{
    if (B == 0 || !size_ok(B, H, W)) return 0;
    return 2 * plane_bytes(B, H, W) + align_up((size_t)B * W * sizeof(int), 256) + align_up((size_t)B * 2 * sizeof(unsigned), 256);
}

extern "C" int ffb6d_fill_depth(const uint16_t *depth_raw, int64_t B, int64_t H, int64_t W, float cam_scale,
                                float *filled_raw, float *depth_m, void *workspace, size_t workspace_bytes,
                                ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(size_ok(B, H, W), "fill_depth: bad size (B=%lld H=%lld W=%lld)", (long long)B, (long long)H, (long long)W);
    FFB6D_CHECK_ARG(cam_scale > 0.0f && cam_scale < INFINITY, "fill_depth: cam_scale must be positive and finite, got %g",
                    (double)cam_scale);
    FFB6D_CHECK_ARG(filled_raw || depth_m, "fill_depth: both outputs are null");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(depth_raw != nullptr, "fill_depth: null depth_raw");
    if (!workspace || workspace_bytes < ffb6d_fill_depth_workspace_bytes(B, H, W)) {
        set_error("fill_depth: workspace of %zu bytes, %zu needed", workspace_bytes, ffb6d_fill_depth_workspace_bytes(B, H, W));
        return FFB6D_ERR_WORKSPACE;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const Plane p{(int)H, (int)W};
    const Workspace w = carve(workspace, B, H, W);
    const dim3 blk(TX, TY), grid((unsigned)ceil_div(W, TX), (unsigned)ceil_div(H, TY), (unsigned)B);
    const dim3 cols((unsigned)ceil_div(W, 128), (unsigned)B);

    bands_kernel<<<grid, blk, 0, st>>>(depth_raw, p, cam_scale, w.a, w.minmax);                    // s2 -> a
    FFB6D_LAUNCH_OK("bands_kernel");
    morph5_kernel<true><<<grid, blk, 0, st>>>(w.a, p, w.b);
    FFB6D_LAUNCH_OK("morph5_kernel<dilate>");
    morph5_kernel<false><<<grid, blk, 0, st>>>(w.b, p, w.a);                                       // s3 -> a
    FFB6D_LAUNCH_OK("morph5_kernel<erode>");
    median5_kernel<<<grid, blk, 0, st>>>(w.a, p, nullptr, w.b, nullptr);                           // s4 -> b
    FFB6D_LAUNCH_OK("median5_kernel");
    top_row_kernel<<<cols, 128, 0, st>>>(w.b, p, w.top);
    FFB6D_LAUNCH_OK("top_row_kernel");
    fill9_kernel<<<grid, blk, 0, st>>>(w.b, p, w.top, w.a);                                        // s5 -> a
    FFB6D_LAUNCH_OK("fill9_kernel");
    top_row_kernel<<<cols, 128, 0, st>>>(w.a, p, w.top);
    FFB6D_LAUNCH_OK("top_row_kernel");
    for (int it = 0; it < 6; ++it) {                                                               // s7 -> a
        const bool even = (it & 1) == 0;
        fill5_kernel<<<grid, blk, 0, st>>>(even ? w.a : w.b, p, w.top, even ? w.b : w.a);
        FFB6D_LAUNCH_OK("fill5_kernel");
    }
    median5_kernel<<<grid, blk, 0, st>>>(w.a, p, w.top, w.b, w.minmax);                            // median -> b
    FFB6D_LAUNCH_OK("median5_kernel");
    bilateral_kernel<<<grid, blk, 0, st>>>(w.a, w.b, p, w.top, w.minmax, cam_scale, filled_raw, depth_m);
    FFB6D_LAUNCH_OK("bilateral_kernel");
    return FFB6D_OK;
}
