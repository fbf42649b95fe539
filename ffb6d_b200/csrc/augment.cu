// augment.cu -- the datasets' synthetic-frame augmentation on the GPU (sm_90a): rgb_add_noise and add_real_back
// (datasets/ycb/ycb_dataset.py:79-163, datasets/linemod/linemod_dataset.py:114-186).
//
// Images are uint8 [B,H,W,3]; every frame has its own float64 record (ffb6d_b200/augment.py, FFB6D_AUG_* in the
// header).  ffb6d_rgb_add_noise runs five launches, each over the whole batch, and a frame whose record disables a
// stage is copied through it unchanged:
//   hsv_kernel       COLOR_BGR2HSV (OpenCV's integer path), S and V scaled in float64 and truncated into uint16,
//                    clipped, COLOR_HSV2BGR (OpenCV 4.13's float path on x86-64: fused 1 - s*h; the product with
//                    255 truncated in its 32-pixel vector loop, rounded in the scalar tail of each row)
//   filter_kernel    filter2D, 8U with a float kernel rounded to float32: a running fma over the kernel's nonzero
//                    taps in row-major order, rounded half to even; once for the sharpen 3x3, once for motion blur
//   gauss_kernel     GaussianBlur 3x3 / 5x5: OpenCV's fixed-point separable path, integer taps of weight 1/256,
//                    (sum + 2^15) >> 16
//   noise_kernel     gaussian_noise and YCB's last normal(0, 7): clip(x + z*sigma, 0, 255) truncated, in float64
// All borders are BORDER_REFLECT_101.  With H, W >= 32 and kernels up to 30x30 one reflection maps every index the
// filters load into the frame (load_tile loads only the halo of in-range outputs).
//
// The normal draws come from Philox4x32-10 keyed by the seed, with counter (element pair, frame, stage, 0), and
// Box-Muller in float64: a draw depends on (seed, frame, stage, pixel, channel) only, never on the launch shape.
#include <cmath>

#include "common.cuh"

namespace ffb6d {

enum { R_VERSION = 0, R_DATASET = 1, R_PASS = 2, R_HSV = 3, R_SF = 4, R_VF = 5, R_SHARPEN = 6, R_SHARPEN_K = 7,
       R_MOTION_A = 16, R_GAUSS_K = 19, R_GAUSS_TAPS = 21, R_NOISE = 26, R_NOISE_SIGMA = 27, R_FINAL = 28,
       R_MOTION_K = 32 };
static_assert(R_MOTION_K + FFB6D_AUG_MAX_KSIZE * FFB6D_AUG_MAX_KSIZE <= FFB6D_AUG_REC_LEN, "record too short");

constexpr int TX = 32, TY = 8;                       // output tile of the 2-D filters
constexpr int MAXR = FFB6D_AUG_MAX_KSIZE - 1;        // largest halo (anchor a/2, a <= 30)

__device__ __forceinline__ int reflect101(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// ----------------------------------------------------------------------------------------------- Philox + normals
__device__ __forceinline__ uint4 philox10(uint4 c, uint2 k)
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

// standard normal number e (= pixel * 3 + channel) of (seed, frame, stage)
__device__ __forceinline__ double aug_normal(uint64_t seed, int frame, int stage, uint32_t e)
{
    const uint4 w = philox10(make_uint4(e >> 1, (uint32_t)frame, (uint32_t)stage, 0u),
                             make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const uint64_t a = ((uint64_t)w.x << 21) | (w.y >> 11), b = ((uint64_t)w.z << 21) | (w.w >> 11);
    const double u1 = (double)(a + 1) * 0x1p-53;    // (0, 1]
    const double u2 = (double)b * 0x1p-53;          // [0, 1)
    const double r = sqrt(-2.0 * log(u1));
    return (e & 1) ? r * sinpi(2.0 * u2) : r * cospi(2.0 * u2);
}

__global__ void noise_field_kernel(uint64_t seed, int stage, uint32_t n_el, double *__restrict__ out)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n_el) out[(size_t)blockIdx.y * n_el + e] = aug_normal(seed, blockIdx.y, stage, e);
}

// --------------------------------------------------------------------------------------------------------- HSV
__device__ __forceinline__ void hsv_pixel(const uint8_t *in, uint8_t *o, double sf, double vf, bool simd)
{
    // COLOR_BGR2HSV, 8U: the channel in slot 0 plays "blue", as the reference feeds it RGB data
    const int b = in[0], g = in[1], r = in[2];
    const int v = max(max(b, g), r), vmin = min(min(b, g), r), diff = v - vmin;
    const int sdiv = v ? __double2int_rn((double)(255 << 12) / v) : 0;
    const int hdiv = diff ? __double2int_rn((double)(180 << 12) / (6.0 * diff)) : 0;
    const int s = (diff * sdiv + (1 << 11)) >> 12;
    int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
    h = (h * hdiv + (1 << 11)) >> 12;
    h += h < 0 ? 180 : 0;
    // hsv_img.astype(uint16) * factor, truncated into uint16, then clipped to 255
    const int s2 = min(255, (int)__dmul_rn((double)s, sf));
    const int v2 = min(255, (int)__dmul_rn((double)v, vf));
    // COLOR_HSV2BGR, 8U
    const float fs = __fmul_rn((float)s2, 1.0f / 255.0f), fv = __fmul_rn((float)v2, 1.0f / 255.0f);
    float ob, og, orr;
    if (s2 == 0) {
        ob = og = orr = fv;
    } else {
        const float hh = __fmul_rn((float)h, 6.0f / 180.0f);
        const int sector = (int)floorf(hh);
        const float f = __fsub_rn(hh, (float)sector);
        float tab[4];
        tab[0] = fv;
        tab[1] = __fmul_rn(fv, __fsub_rn(1.0f, fs));
        tab[2] = __fmul_rn(fv, __fmaf_rn(-fs, f, 1.0f));
        tab[3] = __fmul_rn(fv, __fmaf_rn(-fs, __fsub_rn(1.0f, f), 1.0f));
        const int sd[6][3] = {{1, 3, 0}, {1, 0, 2}, {3, 0, 1}, {0, 2, 1}, {0, 1, 3}, {2, 1, 0}};
        const int sc = (unsigned)sector < 6u ? sector : 0;
        ob = tab[sd[sc][0]];
        og = tab[sd[sc][1]];
        orr = tab[sd[sc][2]];
    }
    // OpenCV's vector loop (32 pixels at a time) truncates the product; the scalar loop over a row's tail rounds it
    const float c[3] = {__fmul_rn(ob, 255.0f), __fmul_rn(og, 255.0f), __fmul_rn(orr, 255.0f)};
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
        o[ch] = (uint8_t)min(255, max(0, simd ? __float2int_rz(c[ch]) : __float2int_rn(c[ch])));
}

__global__ void hsv_kernel(const uint8_t *__restrict__ src, const double *__restrict__ plan, int HW, int W,
                           uint8_t *__restrict__ dst)
{
    const int b = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const double *rec = plan + (size_t)b * FFB6D_AUG_REC_LEN;
    const size_t off = ((size_t)b * HW + p) * 3;
    uint8_t in[3] = {src[off], src[off + 1], src[off + 2]}, o[3];
    if (__ldg(rec + R_HSV) != 0.0) {
        hsv_pixel(in, o, __ldg(rec + R_SF), __ldg(rec + R_VF), p % W < W - W % 32);
    } else {
        o[0] = in[0]; o[1] = in[1]; o[2] = in[2];
    }
    dst[off] = o[0]; dst[off + 1] = o[1]; dst[off + 2] = o[2];
}

// ------------------------------------------------------------------------------------------------ 2-D filters
// The tile of a frame with its reflected halo: rows y0-r .. y0+TY-1+(a-1-r), columns likewise, 3 channels, row
// stride tw.  Only the part that in-range outputs read is loaded: raw rows and columns then stay within
// [-r, n-1+(a-1-r)], which one reflection maps into [0, n) for n >= 32 and a <= 30.  The rest of a partial edge tile
// (halo of outputs past H or W) is left unset and never read.
__device__ __forceinline__ void load_tile(const uint8_t *img, int H, int W, int y0, int x0, int r, int a,
                                          uint8_t *tile, int tw, int th)
{
    const int tw_used = min(tw, W - x0 + a - 1), th_used = min(th, H - y0 + a - 1);
    for (int i = threadIdx.y * TX + threadIdx.x; i < tw_used * th_used; i += TX * TY) {
        const int ty = i / tw_used, tx = i % tw_used;
        const int yy = reflect101(y0 - r + ty, H), xx = reflect101(x0 - r + tx, W);
        const uint8_t *s = img + ((size_t)yy * W + xx) * 3;
        uint8_t *t = tile + (ty * tw + tx) * 3;
        t[0] = s[0];
        t[1] = s[1];
        t[2] = s[2];
    }
}

// which = 0: the sharpen 3x3 (record slots R_SHARPEN_K), 1: the motion-blur a x a (R_MOTION_K)
__global__ void __launch_bounds__(TX * TY)
filter_kernel(const uint8_t *__restrict__ src, const double *__restrict__ plan, int H, int W, int which,
              uint8_t *__restrict__ dst)
{
    __shared__ uint8_t tile[(TY + MAXR) * (TX + MAXR) * 3];
    __shared__ float coef[FFB6D_AUG_MAX_KSIZE * FFB6D_AUG_MAX_KSIZE];
    __shared__ short2 tap[FFB6D_AUG_MAX_KSIZE * FFB6D_AUG_MAX_KSIZE];
    __shared__ int n_tap;
    const int b = blockIdx.z, x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    const double *rec = plan + (size_t)b * FFB6D_AUG_REC_LEN;
    const uint8_t *img = src + (size_t)b * H * W * 3;
    const int a = which == 0 ? (__ldg(rec + R_SHARPEN) != 0.0 ? 3 : 0) : (int)__ldg(rec + R_MOTION_A);
    if (a == 0) {                                     // stage off for this frame: copy through
        if (x < W && y < H) {
            const size_t o = ((size_t)b * H * W + (size_t)y * W + x) * 3;
            dst[o] = src[o]; dst[o + 1] = src[o + 1]; dst[o + 2] = src[o + 2];
        }
        return;
    }
    const double *k = rec + (which == 0 ? R_SHARPEN_K : R_MOTION_K);
    // compact the nonzero taps in row-major order (warp 0, a ballot per 32 taps)
    if (threadIdx.y == 0) {
        int base = 0;
        for (int i0 = 0; i0 < a * a; i0 += 32) {
            const int i = i0 + threadIdx.x;
            const float c = i < a * a ? __double2float_rn(__ldg(k + i)) : 0.0f;
            const unsigned m = __ballot_sync(0xffffffffu, c != 0.0f);
            if (c != 0.0f) {
                const int j = base + __popc(m & ((1u << threadIdx.x) - 1u));
                coef[j] = c;
                tap[j] = make_short2((short)(i / a), (short)(i % a));
            }
            base += __popc(m);
        }
        if (threadIdx.x == 0) n_tap = base;
    }
    const int r = a / 2, tw = TX + a - 1, th = TY + a - 1;
    load_tile(img, H, W, y0, x0, r, a, tile, tw, th);
    __syncthreads();
    if (x >= W || y >= H) return;
    float acc[3] = {0.0f, 0.0f, 0.0f};
    for (int j = 0; j < n_tap; ++j) {
        const short2 t = tap[j];
        const float c = coef[j];
        const uint8_t *s = tile + ((threadIdx.y + t.x) * tw + threadIdx.x + t.y) * 3;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) acc[ch] = __fmaf_rn((float)s[ch], c, acc[ch]);
    }
    const size_t o = ((size_t)b * H * W + (size_t)y * W + x) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) dst[o + ch] = (uint8_t)min(255, max(0, __float2int_rn(acc[ch])));
}

__global__ void __launch_bounds__(TX * TY)
gauss_kernel(const uint8_t *__restrict__ src, const double *__restrict__ plan, int H, int W,
             uint8_t *__restrict__ dst)
{
    __shared__ uint8_t tile[(TY + 4) * (TX + 4) * 3];
    const int b = blockIdx.z, x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    const double *rec = plan + (size_t)b * FFB6D_AUG_REC_LEN;
    const int a = (int)__ldg(rec + R_GAUSS_K);
    if (a == 0) {
        if (x < W && y < H) {
            const size_t o = ((size_t)b * H * W + (size_t)y * W + x) * 3;
            dst[o] = src[o]; dst[o + 1] = src[o + 1]; dst[o + 2] = src[o + 2];
        }
        return;
    }
    int t[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) t[i] = i < a ? (int)__ldg(rec + R_GAUSS_TAPS + i) : 0;
    const int r = a / 2, tw = TX + a - 1, th = TY + a - 1;
    load_tile(src + (size_t)b * H * W * 3, H, W, y0, x0, r, a, tile, tw, th);
    __syncthreads();
    if (x >= W || y >= H) return;
    const size_t o = ((size_t)b * H * W + (size_t)y * W + x) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        int col = 0;                                  // exact: row sums fit 16 bits, the total 24
        for (int i = 0; i < a; ++i) {
            int row = 0;
            for (int j = 0; j < a; ++j) row += t[j] * tile[((threadIdx.y + i) * tw + threadIdx.x + j) * 3 + ch];
            col += t[i] * row;
        }
        dst[o + ch] = (uint8_t)min(255, (col + (1 << 15)) >> 16);
    }
}

// ------------------------------------------------------------------------------------------------------ noise
__device__ __forceinline__ uint8_t add_clip_trunc(double x, double n)
{
    const double v = __dadd_rn(x, n);
    return (uint8_t)(int)fmin(fmax(v, 0.0), 255.0);
}

// field (optional): [2,B,H,W,3] float64 normals to use instead of the generator's (stage 2*pass, 2*pass+1)
// seed_dev (optional): the seed read on the device instead of the value (ffb6d_rgb_add_noise_dseed)
__global__ void noise_kernel(const uint8_t *__restrict__ src, const double *__restrict__ plan, uint32_t n_el,
                             uint64_t seed, const uint64_t *__restrict__ seed_dev, const double *__restrict__ field,
                             int B, uint8_t *__restrict__ dst)
{
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (e >= n_el) return;
    if (seed_dev) seed = __ldg((const unsigned long long *)seed_dev);
    const double *rec = plan + (size_t)b * FFB6D_AUG_REC_LEN;
    const size_t o = (size_t)b * n_el + e;
    uint8_t v = src[o];
    const int pass = (int)__ldg(rec + R_PASS);
    if (__ldg(rec + R_NOISE) != 0.0) {
        const double z = field ? field[o] : aug_normal(seed, b, 2 * pass, e);
        v = add_clip_trunc((double)v, __dmul_rn(z, __ldg(rec + R_NOISE_SIGMA)));
    }
    if (__ldg(rec + R_FINAL) != 0.0) {
        const double z = field ? field[(size_t)B * n_el + o] : aug_normal(seed, b, 2 * pass + 1, e);
        v = add_clip_trunc((double)v, __dadd_rn(0.0, __dmul_rn(7.0, z)));    // loc + scale * gauss
    }
    dst[o] = v;
}

// -------------------------------------------------------------------------------------------- add_real_back
// mode[b]: bit 0 the frame goes through add_real_back (depth composed), bit 1 its colour image is composed too
__global__ void real_back_kernel(const uint8_t *__restrict__ rgb, const uint8_t *__restrict__ labels,
                                 const uint16_t *__restrict__ dpt, const uint8_t *__restrict__ back_rgb,
                                 const uint8_t *__restrict__ back_labels, int back_ch,
                                 const uint16_t *__restrict__ back_dpt, const uint8_t *__restrict__ mode, int linemod,
                                 int HW, uint8_t *__restrict__ rgb_out, uint16_t *__restrict__ dpt_out)
{
    const int b = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const size_t i = (size_t)b * HW + p;
    const int m = __ldg(mode + b);
    const int bl = __ldg(back_labels + i * back_ch);
    const bool keep = linemod ? bl < 255 : bl == 0;            // bk_label < 255 (LineMOD), bk_label <= 0 (YCB)
    const bool hole = __ldg(labels + i) == 0;                  // msk_back = labels <= 0
    uint8_t c[3] = {rgb[i * 3], rgb[i * 3 + 1], rgb[i * 3 + 2]};
    if ((m & 3) == 3 && hole) {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) c[ch] = keep ? __ldg(back_rgb + i * 3 + ch) : 0;
    }
    uint16_t d = dpt[i];
    if ((m & 1) && d == 0) d = keep ? __ldg(back_dpt + i) : 0;
    rgb_out[i * 3] = c[0]; rgb_out[i * 3 + 1] = c[1]; rgb_out[i * 3 + 2] = c[2];
    dpt_out[i] = d;
}

static const char *check_record(const double *r)
{
    auto flag = [](double v) { return v == 0.0 || v == 1.0; };
    auto whole = [](double v, double lo, double hi) { return v >= lo && v <= hi && v == (double)(int64_t)v; };
    if (r[R_VERSION] != FFB6D_AUG_VERSION) return "record layout version";
    if (!(whole(r[R_DATASET], 0, 1) && whole(r[R_PASS], 0, 1))) return "dataset / pass";
    if (!(flag(r[R_HSV]) && flag(r[R_SHARPEN]) && flag(r[R_NOISE]) && flag(r[R_FINAL]))) return "stage flag";
    if (!(r[R_SF] >= 0.0 && r[R_SF] <= 256.0 && r[R_VF] >= 0.0 && r[R_VF] <= 256.0)) return "HSV factor";
    if (!whole(r[R_MOTION_A], 0, FFB6D_AUG_MAX_KSIZE)) return "motion kernel size";
    const int g = (int)r[R_GAUSS_K];
    if (!(whole(r[R_GAUSS_K], 0, 5) && (g == 0 || g == 3 || g == 5))) return "Gaussian kernel size";
    int sum = 0;
    for (int i = 0; i < g; ++i) {
        if (!whole(r[R_GAUSS_TAPS + i], 0, 256)) return "Gaussian tap";
        sum += (int)r[R_GAUSS_TAPS + i];
    }
    if (g && sum != 256) return "Gaussian taps (sum != 256)";
    if (!(r[R_NOISE_SIGMA] >= 0.0 && r[R_NOISE_SIGMA] <= 255.0)) return "noise sigma";
    const int a = (int)r[R_MOTION_A];
    for (int i = 0; i < 9; ++i)
        if (!std::isfinite(r[R_SHARPEN_K + i])) return "sharpen kernel";
    for (int i = 0; i < a * a; ++i)
        if (!std::isfinite(r[R_MOTION_K + i])) return "motion kernel";
    return nullptr;
}

// every frame's record, before any launch (ffb6d_rgb_add_noise, ffb6d_rgb_noise_check_records)
static int check_records(const double *plan_host, int64_t B)
{
    for (int64_t b = 0; b < B; ++b) {
        const char *bad = check_record(plan_host + b * FFB6D_AUG_REC_LEN);
        FFB6D_CHECK_ARG(!bad, "rgb_add_noise: frame %lld: bad record (%s)", (long long)b, bad);
    }
    return FFB6D_OK;
}

}  // namespace ffb6d

using namespace ffb6d;

// The 2-D filters put the row tiles in grid.y: H <= 65535 * TY (as ffb6d_fill_depth bounds it)
#define AUG_CHECK_SIZE(tag)                                                                                         \
    FFB6D_CHECK_ARG(B >= 0 && B < 65536 && H >= 32 && W >= 32 && H <= 65535ll * TY && W < (1 << 20) &&              \
                    H * W * 3 < (1ll << 31),                                                                        \
                    tag ": bad size (B=%lld H=%lld W=%lld; H, W >= 32, H <= %lld)", (long long)B, (long long)H,     \
                    (long long)W, 65535ll * TY)

// ffb6d_rgb_add_noise and ffb6d_rgb_add_noise_dseed: the seed by value, or (dseed) read from seed_dev on the device
static int rgb_add_noise(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, const double *plan_host,
                         const double *plan_dev, uint64_t seed, bool dseed, const uint64_t *seed_dev,
                         const double *noise, uint8_t *out, uint8_t *work, ffb6d_stream_t stream)
{
    AUG_CHECK_SIZE("rgb_add_noise");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(rgb && plan_host && plan_dev && out && work && (seed_dev || !dseed), "rgb_add_noise: null pointer");
    FFB6D_CHECK_ARG(work != rgb && work != out, "rgb_add_noise: work must not alias rgb or out");
    FFB6D_CHECK_ARG((uintptr_t)plan_host % 8 == 0 && (uintptr_t)plan_dev % 8 == 0 && (uintptr_t)noise % 8 == 0 &&
                        (uintptr_t)seed_dev % 8 == 0,
                    "rgb_add_noise: misaligned pointer");
    const int rc = check_records(plan_host, B);
    if (rc != FFB6D_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int HW = (int)(H * W);
    const dim3 pgrid((unsigned)ceil_div(HW, 256), (unsigned)B);
    const dim3 tgrid((unsigned)ceil_div(W, TX), (unsigned)ceil_div(H, TY), (unsigned)B), tblock(TX, TY);
    hsv_kernel<<<pgrid, 256, 0, st>>>(rgb, plan_dev, HW, (int)W, out);
    FFB6D_LAUNCH_OK("hsv_kernel");
    filter_kernel<<<tgrid, tblock, 0, st>>>(out, plan_dev, (int)H, (int)W, 0, work);
    FFB6D_LAUNCH_OK("filter_kernel");
    filter_kernel<<<tgrid, tblock, 0, st>>>(work, plan_dev, (int)H, (int)W, 1, out);
    FFB6D_LAUNCH_OK("filter_kernel");
    gauss_kernel<<<tgrid, tblock, 0, st>>>(out, plan_dev, (int)H, (int)W, work);
    FFB6D_LAUNCH_OK("gauss_kernel");
    const uint32_t n_el = (uint32_t)(HW * 3);
    noise_kernel<<<dim3((unsigned)ceil_div(n_el, 256), (unsigned)B), 256, 0, st>>>(work, plan_dev, n_el, seed, seed_dev,
                                                                                noise, (int)B, out);
    FFB6D_LAUNCH_OK("noise_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_rgb_add_noise(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, const double *plan_host,
                                   const double *plan_dev, uint64_t seed, const double *noise, uint8_t *out,
                                   uint8_t *work, ffb6d_stream_t stream)
{
    return rgb_add_noise(rgb, B, H, W, plan_host, plan_dev, seed, false, nullptr, noise, out, work, stream);
}

extern "C" int ffb6d_rgb_add_noise_dseed(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, const double *plan_host,
                                         const double *plan_dev, const uint64_t *seed_dev, const double *noise,
                                         uint8_t *out, uint8_t *work, ffb6d_stream_t stream)
{
    return rgb_add_noise(rgb, B, H, W, plan_host, plan_dev, 0, true, seed_dev, noise, out, work, stream);
}

extern "C" int ffb6d_rgb_noise_check_records(const double *plan_host, int64_t B)
{
    FFB6D_CHECK_ARG(B >= 0 && B < 65536, "rgb_noise_check_records: bad size (B=%lld)", (long long)B);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(plan_host, "rgb_noise_check_records: null pointer");
    FFB6D_CHECK_ARG((uintptr_t)plan_host % 8 == 0, "rgb_noise_check_records: misaligned pointer");
    return check_records(plan_host, B);
}

extern "C" int ffb6d_add_real_back(const uint8_t *rgb, const uint8_t *labels, const uint16_t *dpt,
                                   const uint8_t *back_rgb, const uint8_t *back_labels, int back_label_channels,
                                   const uint16_t *back_dpt, const uint8_t *mode, int dataset, int64_t B, int64_t H,
                                   int64_t W, uint8_t *rgb_out, uint16_t *dpt_out, ffb6d_stream_t stream)
{
    AUG_CHECK_SIZE("add_real_back");
    FFB6D_CHECK_ARG(dataset == FFB6D_AUG_YCB || dataset == FFB6D_AUG_LINEMOD,
                    "add_real_back: dataset must be FFB6D_AUG_YCB or FFB6D_AUG_LINEMOD");
    FFB6D_CHECK_ARG(back_label_channels == 1 || back_label_channels == 3,
                    "add_real_back: back_label_channels must be 1 or 3");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(rgb && labels && dpt && back_rgb && back_labels && back_dpt && mode && rgb_out && dpt_out,
                    "add_real_back: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)dpt | (uintptr_t)back_dpt | (uintptr_t)dpt_out) % 2 == 0,
                    "add_real_back: misaligned pointer");
    const int HW = (int)(H * W);
    real_back_kernel<<<dim3((unsigned)ceil_div(HW, 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
        rgb, labels, dpt, back_rgb, back_labels, back_label_channels, back_dpt, mode, dataset == FFB6D_AUG_LINEMOD,
        HW, rgb_out, dpt_out);
    FFB6D_LAUNCH_OK("real_back_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_aug_noise_field(uint64_t seed, int64_t B, int64_t H, int64_t W, int stage, double *out,
                                     ffb6d_stream_t stream)
{
    AUG_CHECK_SIZE("aug_noise_field");
    FFB6D_CHECK_ARG(stage >= 0 && stage < 4, "aug_noise_field: stage %d outside [0, 4)", stage);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(out, "aug_noise_field: null pointer");
    FFB6D_CHECK_ARG((uintptr_t)out % 8 == 0, "aug_noise_field: misaligned pointer");
    const uint32_t n_el = (uint32_t)(H * W * 3);
    noise_field_kernel<<<dim3((unsigned)ceil_div(n_el, 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
        seed, stage, n_el, out);
    FFB6D_LAUNCH_OK("noise_field_kernel");
    return FFB6D_OK;
}
