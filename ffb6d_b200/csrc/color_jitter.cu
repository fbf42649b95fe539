// color_jitter.cu -- the datasets' colour jitter on the GPU (sm_90a): torchvision's
// ColorJitter(0.2, 0.2, 0.2, 0.05) on a PIL RGB image (datasets/ycb/ycb_dataset.py:34, 190-193;
// datasets/linemod/linemod_dataset.py:35, 220-223), pinned to torchvision 0.26 and Pillow 12.2.
//
// Every frame has a float64 plan of FFB6D_JITTER_PLAN_LEN slots (ffb6d_b200/augment.py draw_color_jitter): the
// order of the four ops, then the brightness, contrast, saturation and hue factors.  The ops on uint8 RGB:
//   brightness  Image.blend(black, img, f)
//   contrast    Image.blend(mean, img, f), mean = int(sum L / (H*W) + 0.5) over the image the op receives
//   saturation  Image.blend(L, img, f), L replicated to three bands
//   hue         convert("HSV"), H += int32(hue * 255) mod 256, convert("RGB")
// with L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16 (convert("L")).  Image.blend takes the factor as a C float
// and computes a + f * (b - a) in float32, product and sum rounded separately; for 0 <= f <= 1 the result is
// truncated, otherwise clipped to [0, 255] and truncated.  The HSV conversions restate Pillow's rgb2hsv_row /
// hsv2rgb with their float32 / float64 mix.  The _rn intrinsics keep nvcc from contracting any of it into FMAs.
//
// Contrast is the only op that is not pointwise, so a frame's chain is a pointwise prefix, one frame-wide mean and a
// pointwise suffix.  jitter_sum_kernel applies the prefix and adds L of the result into the frame's int64 sum (exact,
// so independent of the order of the atomics); jitter_apply_kernel recomputes the prefix from the input, applies
// contrast with the frame's mean, then the suffix, and stores.  A thread owns 4 consecutive pixels (12 bytes, three
// 32-bit words when the frame's rows are 4-byte aligned).
#include <cfloat>
#include <cmath>

#include "common.cuh"

namespace ffb6d {

constexpr int JT = 256;      // threads per CTA
constexpr int JPX = 4;       // pixels per thread

// A frame's plan as the kernels use it: the order packed 2 bits per position, the blend factors as C floats.
struct Jitter {
    int order;               // op at position k: (order >> 2k) & 3; 0 brightness, 1 contrast, 2 saturation, 3 hue
    int contrast_pos;        // position of contrast in the order
    float f[3];              // brightness, contrast, saturation
    int shift;               // hue shift, mod 256
};

__device__ __forceinline__ Jitter load_jitter(const double *p)
{
    Jitter j;
    j.order = 0;
    j.contrast_pos = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int op = (int)__ldg(p + k);
        j.order |= op << (2 * k);
        if (op == 1) j.contrast_pos = k;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) j.f[k] = __double2float_rn(__ldg(p + 4 + k));
    j.shift = __double2int_rz(__dmul_rn(__ldg(p + 7), 255.0)) & 255;     // np.int32(hue * 255) as uint8
    return j;
}

__device__ __forceinline__ int luma(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16; }

// Image.blend(a, b, f) on one byte
__device__ __forceinline__ int blend(int a, int b, float f)
{
    const float t = __fadd_rn((float)a, __fmul_rn(f, (float)(b - a)));
    if (f >= 0.0f && f <= 1.0f) return __float2int_rz(t);
    return t <= 0.0f ? 0 : (t >= 255.0f ? 255 : __float2int_rz(t));
}

// Pillow's rgb2hsv_row: float32 ratios, the hue's sum and fmod in float64, each stored to float32
__device__ __forceinline__ void rgb2hsv(int r, int g, int b, int &H, int &S, int &V)
{
    const int mx = max(max(r, g), b), mn = min(min(r, g), b);
    V = mx;
    if (mx == mn) {
        H = S = 0;
        return;
    }
    const float cr = (float)(mx - mn);
    const float s = __fdiv_rn(cr, (float)mx);
    // only the two ratios a branch reads: rc = (mx - r) / cr and so on
    float h;
    if (r == mx)
        h = __fsub_rn(__fdiv_rn((float)(mx - b), cr), __fdiv_rn((float)(mx - g), cr));
    else if (g == mx)
        h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, (double)__fdiv_rn((float)(mx - r), cr)),
                                        (double)__fdiv_rn((float)(mx - b), cr)));
    else
        h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, (double)__fdiv_rn((float)(mx - g), cr)),
                                        (double)__fdiv_rn((float)(mx - r), cr)));
    // fmod(h / 6.0 + 1.0, 1.0): h is in [-1, 5], so the sum is in [5/6, 11/6] and the fmod is one exact subtraction
    double x = __dadd_rn(__ddiv_rn((double)h, 6.0), 1.0);
    x = x >= 1.0 ? __dsub_rn(x, 1.0) : x;
    h = __double2float_rn(x);
    H = min(255, max(0, __double2int_rz(__dmul_rn((double)h, 255.0))));
    S = min(255, max(0, __double2int_rz(__dmul_rn((double)s, 255.0))));
}

// The parts of Pillow's hsv2rgb that depend on one byte, per CTA in shared memory: for h the sextant
// i = floor(h * 6.0 / 255.0) mod 6 and the remainder f = (float)(h * 6.0 / 255.0 - i) in float64, for s
// fs = (float)(s / 255.0).  Filled by the kernel's 256 threads, one entry each.
struct HsvTables {
    float f[256], fs[256];
    uint8_t sextant[256];
};
static_assert(JT == 256, "one table entry per thread");

__device__ __forceinline__ void fill_tables(HsvTables &tab)
{
    const int t = threadIdx.x;
    const double hh = __ddiv_rn((double)t * 6.0, 255.0);
    const int i = (int)floor(hh);
    tab.f[t] = __double2float_rn(__dsub_rn(hh, (double)i));
    tab.sextant[t] = (uint8_t)(i % 6);
    tab.fs[t] = __double2float_rn(__ddiv_rn((double)t, 255.0));
}

// Pillow's hsv2rgb: p, q, t rounded half away from zero in float64; fs * f is a float32 product
__device__ __forceinline__ void hsv2rgb(int h, int s, int v, const HsvTables &tab, int &r, int &g, int &b)
{
    if (s == 0) {
        r = g = b = v;
        return;
    }
    const float f = tab.f[h], fs = tab.fs[s];
    const double dv = (double)v;
    const int p = min(255, max(0, (int)round(__dmul_rn(dv, __dsub_rn(1.0, (double)fs)))));
    const int q = min(255, max(0, (int)round(__dmul_rn(dv, __dsub_rn(1.0, (double)__fmul_rn(fs, f))))));
    const int t = min(255, max(0, (int)round(
        __dmul_rn(dv, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f)))))));
    switch (tab.sextant[h]) {
        case 0: r = v; g = t; b = p; break;
        case 1: r = q; g = v; b = p; break;
        case 2: r = p; g = v; b = t; break;
        case 3: r = p; g = q; b = v; break;
        case 4: r = t; g = p; b = v; break;
        default: r = v; g = p; b = q; break;
    }
}

// positions [0, hi) of the frame's chain on one pixel; contrast blends towards `mean`
__device__ __forceinline__ void chain(int c[3], const Jitter &j, const HsvTables &tab, int hi, int mean)
{
    for (int k = 0; k < hi; ++k) {
        const int op = (j.order >> (2 * k)) & 3;
        if (op == 3) {
            int H, S, V;
            rgb2hsv(c[0], c[1], c[2], H, S, V);
            hsv2rgb((H + j.shift) & 255, S, V, tab, c[0], c[1], c[2]);
        } else {
            const int a = op == 0 ? 0 : (op == 1 ? mean : luma(c[0], c[1], c[2]));
            const float f = op == 0 ? j.f[0] : (op == 1 ? j.f[1] : j.f[2]);     // selects, not a local array
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) c[ch] = blend(a, c[ch], f);
        }
    }
}

// the 4 pixels of thread t of frame `img` (HW pixels): n of them exist; three 32-bit words when aligned
__device__ __forceinline__ int load_px(const uint8_t *img, int HW, int px0, bool vec, uint32_t w[3])
{
    const int n = min(JPX, HW - px0);
    if (n <= 0) return 0;
    const uint8_t *s = img + (size_t)px0 * 3;
    if (vec && n == JPX) {
        const uint32_t *s4 = reinterpret_cast<const uint32_t *>(s);
        w[0] = s4[0]; w[1] = s4[1]; w[2] = s4[2];
    } else {
        w[0] = w[1] = w[2] = 0;
#pragma unroll
        for (int i = 0; i < 3 * JPX; ++i)        // unrolled, so that w stays in registers
            if (i < 3 * n) w[i >> 2] |= (uint32_t)s[i] << (8 * (i & 3));
    }
    return n;
}

__device__ __forceinline__ void store_px(uint8_t *img, int px0, int n, bool vec, const uint32_t w[3])
{
    uint8_t *d = img + (size_t)px0 * 3;
    if (vec && n == JPX) {
        uint32_t *d4 = reinterpret_cast<uint32_t *>(d);
        d4[0] = w[0]; d4[1] = w[1]; d4[2] = w[2];
    } else {
#pragma unroll
        for (int i = 0; i < 3 * JPX; ++i)
            if (i < 3 * n) d[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
    }
}

__device__ __forceinline__ int byte_of(const uint32_t w[3], int i) { return (w[i >> 2] >> (8 * (i & 3))) & 255; }

__global__ void __launch_bounds__(JT)
jitter_sum_kernel(const uint8_t *__restrict__ rgb, const double *__restrict__ plan,
                  const uint8_t *__restrict__ active, int HW, unsigned long long *__restrict__ sums)
{
    const int b = blockIdx.y;
    if (!__ldg(active + b)) return;
    __shared__ HsvTables tab;
    fill_tables(tab);
    const Jitter j = load_jitter(plan + (size_t)b * FFB6D_JITTER_PLAN_LEN);
    const uint8_t *img = rgb + (size_t)b * HW * 3;
    const int px0 = (blockIdx.x * JT + threadIdx.x) * JPX;
    uint32_t w[3];
    const int n = load_px(img, HW, px0, ((uintptr_t)img & 3) == 0, w);
    __syncthreads();
    unsigned sum = 0;
#pragma unroll
    for (int i = 0; i < JPX; ++i) {
        if (i < n) {
            int c[3] = {byte_of(w, 3 * i), byte_of(w, 3 * i + 1), byte_of(w, 3 * i + 2)};
            chain(c, j, tab, j.contrast_pos, 0);
            sum += luma(c[0], c[1], c[2]);
        }
    }
    __shared__ unsigned warp_sum[JT / 32];
    sum = __reduce_add_sync(0xffffffffu, sum);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x < 32) {
        unsigned s = threadIdx.x < JT / 32 ? warp_sum[threadIdx.x] : 0u;
        s = __reduce_add_sync(0xffffffffu, s);
        if (threadIdx.x == 0 && s) atomicAdd(sums + b, (unsigned long long)s);
    }
}

// rgb and out may be the same array: each thread reads its 12 bytes before it writes them
__global__ void __launch_bounds__(JT)
jitter_apply_kernel(const uint8_t *rgb, const double *__restrict__ plan, const uint8_t *__restrict__ active, int HW,
                    const unsigned long long *__restrict__ sums, uint8_t *out)
{
    const int b = blockIdx.y;
    const uint8_t *img = rgb + (size_t)b * HW * 3;
    uint8_t *dst = out + (size_t)b * HW * 3;
    const int px0 = (blockIdx.x * JT + threadIdx.x) * JPX;
    const bool vec = (((uintptr_t)img | (uintptr_t)dst) & 3) == 0;
    const bool on = __ldg(active + b) != 0;
    __shared__ HsvTables tab;
    if (on) fill_tables(tab);                 // before any thread leaves: on is the same for the whole CTA
    __syncthreads();
    uint32_t w[3];
    const int n = load_px(img, HW, px0, vec, w);
    if (n == 0) return;
    if (on) {
        const Jitter j = load_jitter(plan + (size_t)b * FFB6D_JITTER_PLAN_LEN);
        const int mean = __double2int_rz(__dadd_rn(__ddiv_rn((double)__ldg(sums + b), (double)HW), 0.5));
        uint32_t o[3] = {0u, 0u, 0u};
#pragma unroll
        for (int i = 0; i < JPX; ++i) {
            int c[3] = {byte_of(w, 3 * i), byte_of(w, 3 * i + 1), byte_of(w, 3 * i + 2)};
            if (i < n) chain(c, j, tab, 4, mean);
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) o[(3 * i + ch) >> 2] |= (uint32_t)c[ch] << (8 * ((3 * i + ch) & 3));
        }
        w[0] = o[0]; w[1] = o[1]; w[2] = o[2];
    }
    store_px(dst, px0, n, vec, w);
}

static const char *check_plan(const double *p)
{
    int seen = 0;
    for (int k = 0; k < 4; ++k) {
        const double v = p[k];
        if (!(v == 0.0 || v == 1.0 || v == 2.0 || v == 3.0)) return "order slot is not 0, 1, 2 or 3";
        seen |= 1 << (int)v;
    }
    if (seen != 15) return "order is not a permutation of 0..3";
    for (int k = 4; k < 7; ++k)
        if (!(std::isfinite(p[k]) && p[k] >= 0.0 && p[k] <= (double)FLT_MAX))
            return "brightness, contrast and saturation factors must be finite and >= 0";
    if (!(std::isfinite(p[7]) && std::fabs(p[7]) <= 0.5)) return "hue factor must lie in [-0.5, 0.5]";
    return nullptr;
}

static bool overlaps(const void *a, size_t na, const void *b, size_t nb)
{
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_color_jitter(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, const double *plan_host,
                                  const double *plan_dev, const uint8_t *active, uint8_t *out, int64_t *work,
                                  ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && B < 65536 && H >= 1 && W >= 1 && H < (1 << 20) && W < (1 << 20) &&
                        H * W * 3 < (1ll << 31),
                    "color_jitter: bad size (B=%lld H=%lld W=%lld)", (long long)B, (long long)H, (long long)W);
    FFB6D_CHECK_ARG(rgb && plan_host && plan_dev && active && out && work, "color_jitter: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)plan_host | (uintptr_t)plan_dev | (uintptr_t)work) % 8 == 0,
                    "color_jitter: misaligned pointer");
    const size_t img_bytes = (size_t)(B * H * W * 3), work_bytes = (size_t)B * sizeof(int64_t);
    FFB6D_CHECK_ARG(!overlaps(work, work_bytes, rgb, img_bytes) && !overlaps(work, work_bytes, out, img_bytes),
                    "color_jitter: work must not alias rgb or out");
    FFB6D_CHECK_ARG(out == rgb || !overlaps(out, img_bytes, rgb, img_bytes),
                    "color_jitter: out must be rgb itself or not overlap it");
    for (int64_t b = 0; b < B; ++b) {
        const char *bad = check_plan(plan_host + b * FFB6D_JITTER_PLAN_LEN);
        FFB6D_CHECK_ARG(!bad, "color_jitter: frame %lld: bad plan (%s)", (long long)b, bad);
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int HW = (int)(H * W);
    const dim3 grid((unsigned)ceil_div(HW, JT * JPX), (unsigned)B);
    FFB6D_CUDA(cudaMemsetAsync(work, 0, work_bytes, st));
    unsigned long long *sums = reinterpret_cast<unsigned long long *>(work);
    jitter_sum_kernel<<<grid, JT, 0, st>>>(rgb, plan_dev, active, HW, sums);
    FFB6D_LAUNCH_OK("jitter_sum_kernel");
    jitter_apply_kernel<<<grid, JT, 0, st>>>(rgb, plan_dev, active, HW, sums, out);
    FFB6D_LAUNCH_OK("jitter_apply_kernel");
    return FFB6D_OK;
}
