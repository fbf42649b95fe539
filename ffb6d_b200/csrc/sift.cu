// sift.cu -- SIFT keypoints of cv2.SIFT_create()'s defaults (sm_90a), DESIGN.md §4.33.
//
// The specification is the header's (ffb6d_sift_detect) and oracle/sift_oracle.py restates it in numpy.  Every float
// operation is an _rn intrinsic in the oracle's order (nvcc never contracts or reorders those), so the outputs are
// bitwise the oracle's.
//
// Frames are processed in chunks of FFB6D_SIFT_CHUNK, octave by octave; the workspace holds one octave-0-sized set of
// layers per frame of a chunk.  Launches per chunk and octave, all with shapes that depend on the arguments only:
//   base     octave 0: grey and the 2x upscale fused; later octaves: layer 3 of the octave before at even pixels;
//   blur     per Gaussian layer a row pass and a column pass (the column pass also writes the DoG layer below it);
//   extrema  per (frame, DoG layer, row) the number of candidates, a per-frame scan of the row counts, then the
//            candidates written in layer then raster order (block scans, no atomics on positions);
//   orient   one warp per candidate, twice: refinement, the orientation histogram and the number of peaks; a
//            per-frame scan of those numbers behind the frame's earlier octaves; then the same computation again,
//            writing each peak's keypoint at its place;
// and per chunk, once every octave is done, one CTA per frame removes duplicates and compacts in order.
#include "common.cuh"

#include <cmath>

namespace ffb6d {
namespace {

constexpr int kGauss = 6, kDog = 5, kLayers = 3;
constexpr int kBorder = 5;
constexpr int kMaxOct = 16;
constexpr int kMaxTaps = 27;          // ks of the largest sigma (3.09)
constexpr int kBins = 36;
constexpr int kThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kDedupThreads = 512;
constexpr int kOriWarps = 4;          // warps per orientation CTA
constexpr int kOriCtas = 256;         // orientation CTAs per frame (grid-stride over the candidates)
constexpr int kMaxWin = 33 * 33;      // window of the largest radius, 16
constexpr int kChunk = FFB6D_SIFT_CHUNK;

struct Geom {
    int n_oct;
    int h[kMaxOct], w[kMaxOct];
    int64_t P;                        // floats of one octave-0 layer
    int ntaps[kGauss];                // [0]: the base blur, [1..5]: the layers
    float taps[kGauss][kMaxTaps];
    int64_t off_cand, off_ncopy, off_rows, off_state;     // byte offsets of a frame's parts
    int64_t frame;                    // workspace bytes of one frame
};

// getGaussianKernel(ks, sigma, CV_32F) with ks = cvRound(8 sigma + 1) | 1, in its bit-exact double form (host)
int gaussian_taps(double sigma, float *out)
{
    const int n = (int)std::nearbyint(sigma * 8 + 1) | 1;
    const double sc = -0.125 / (sigma * sigma);
    double vals[kMaxTaps];
    double s = 0;
    int m = 0;
    for (int x = 1 - n; x < 0; x += 2) {
        vals[m] = std::exp((double)(x * x) * sc);
        s += vals[m++];
    }
    const double mul = 1.0 / (s * 2 + 1.0);
    for (int i = 0; i < m; ++i) out[i] = out[n - 1 - i] = (float)(vals[i] * mul);
    out[m] = (float)mul;
    return n;
}

Geom make_geom(int64_t H, int64_t W)
{
    Geom g;
    g.n_oct = (int)std::nearbyint(std::log((double)std::min(2 * H, 2 * W)) / std::log(2.0) - 2) + 1;
    int h = (int)(2 * H), w = (int)(2 * W);
    for (int o = 0; o < g.n_oct; ++o) {
        g.h[o] = h;
        g.w[o] = w;
        h /= 2;
        w /= 2;
    }
    g.P = (int64_t)g.h[0] * g.w[0];
    const float s = 1.6f;
    g.ntaps[0] = gaussian_taps((double)std::sqrt(std::max(s * s - 0.5f * 0.5f * 4.0f, 0.01f)), g.taps[0]);
    const double k = std::pow(2.0, 1.0 / kLayers);
    for (int i = 1; i < kGauss; ++i) {
        const double prev = std::pow(k, (double)(i - 1)) * 1.6, tot = prev * k;
        g.ntaps[i] = gaussian_taps(std::sqrt(tot * tot - prev * prev), g.taps[i]);
    }
    // per frame: 6 Gaussian + 5 DoG + 1 row-pass layers, candidates and their peak counts (3 P ints each), the row
    // counts (3 h0 + 1 ints) and two ints of per-frame state, each part starting on a 16-byte boundary
    g.off_cand = align_up((size_t)(kGauss + kDog + 1) * g.P * 4, 16);
    g.off_ncopy = g.off_cand + align_up((size_t)3 * g.P * 4, 16);
    g.off_rows = g.off_ncopy + align_up((size_t)3 * g.P * 4, 16);
    g.off_state = g.off_rows + align_up((size_t)(3 * g.h[0] + 1) * 4, 16);
    g.frame = g.off_state + 16;
    return g;
}

struct Args {
    const uint8_t *rgb;
    int64_t H, W;
    int64_t f0;                       // first frame of the chunk
    Geom g;
    uint8_t *ws;
    int32_t *count;
    float *pt, *size, *angle, *resp;
    int32_t *oct;
    int64_t cap;
};

struct Frame {
    float *gauss, *dog, *tmp;
    int32_t *cand, *ncopy, *rows, *state;    // state: [0] candidates of the octave, [1] keypoints before it
};

__device__ __forceinline__ Frame frame_of(const Args &a, int64_t f)
{
    Frame r;
    uint8_t *p = a.ws + f * a.g.frame;
    const int64_t P = a.g.P;
    r.gauss = (float *)p;
    r.dog = r.gauss + kGauss * P;
    r.tmp = r.dog + kDog * P;
    r.cand = (int32_t *)(p + a.g.off_cand);
    r.ncopy = (int32_t *)(p + a.g.off_ncopy);
    r.rows = (int32_t *)(p + a.g.off_rows);
    r.state = (int32_t *)(p + a.g.off_state);
    return r;
}

__device__ __forceinline__ int reflect101(int i, int n)
{
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        if (i >= n) i = 2 * n - 2 - i;
    }
    return i;
}

// OpenCV's column paths of a float blur: 0 fma row and column passes, 1 fma row pass and plain column pass, 2 plain
__device__ __forceinline__ int column_mode(int x, int w)
{
    const int v = w / 8 * 8;
    if (x < v) return 0;
    return (w - v >= 4 && x < v + 4) ? 1 : 2;
}

// octave 0's base before its blur: grey of the frame upscaled 2x (weights 3/4, 1/4, clamped; exact), into tmp
__global__ void __launch_bounds__(kThreads) upscale_kernel(Args a)
{
    const int64_t f = blockIdx.y;
    const int h = a.g.h[0], w = a.g.w[0];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= (int64_t)h * w) return;
    const int y = (int)(i / w), x = (int)(i % w);
    const uint8_t *src = a.rgb + (a.f0 + f) * a.H * a.W * 3;
    auto tap = [](int d, int n, int &s0, int &s1, float &w1) {
        const int s = (d & 1) ? d / 2 : d / 2 - 1;
        w1 = (d & 1) ? 0.25f : 0.75f;
        if (s < 0 || s >= n - 1) w1 = 0.0f;
        s0 = min(max(s, 0), n - 1);
        s1 = min(max(s + 1, 0), n - 1);
    };
    int x0, x1, y0, y1;
    float wx1, wy1;
    tap(x, (int)a.W, x0, x1, wx1);
    tap(y, (int)a.H, y0, y1, wy1);
    auto grey = [&](int yy, int xx) {
        const uint8_t *p = src + ((int64_t)yy * a.W + xx) * 3;
        return (float)((3735 * p[2] + 19235 * p[1] + 9798 * p[0] + (1 << 14)) >> 15);
    };
    const float wx0 = __fsub_rn(1.0f, wx1), wy0 = __fsub_rn(1.0f, wy1);
    const float r0 = __fadd_rn(__fmul_rn(grey(y0, x0), wx0), __fmul_rn(grey(y0, x1), wx1));
    const float r1 = __fadd_rn(__fmul_rn(grey(y1, x0), wx0), __fmul_rn(grey(y1, x1), wx1));
    frame_of(a, f).tmp[i] = __fadd_rn(__fmul_rn(r0, wy0), __fmul_rn(r1, wy1));
}

// a later octave's base: layer 3 of octave o - 1 at even pixels
__global__ void __launch_bounds__(kThreads) downsample_kernel(Args a, int o)
{
    const int64_t f = blockIdx.y;
    const int h = a.g.h[o], w = a.g.w[o], pw = a.g.w[o - 1];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= (int64_t)h * w) return;
    const int y = (int)(i / w), x = (int)(i % w);
    const Frame fr = frame_of(a, f);
    fr.gauss[i] = fr.gauss[3 * a.g.P + (int64_t)(2 * y) * pw + 2 * x];
}

// row pass of Gaussian layer `layer` (0: the base blur of octave 0, reading tmp's upscaled image) into tmp
__global__ void __launch_bounds__(kThreads) row_kernel(Args a, int o, int layer, int from_tmp)
{
    const int64_t f = blockIdx.y;
    const int h = a.g.h[o], w = a.g.w[o];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= (int64_t)h * w) return;
    const int y = (int)(i / w), x = (int)(i % w);
    const Frame fr = frame_of(a, f);
    // octave 0's base blur reads the upscaled image from tmp and writes the dog slot as its scratch
    const float *src = from_tmp ? fr.tmp : fr.gauss + (int64_t)(layer - 1) * a.g.P;
    float *dst = from_tmp ? fr.dog : fr.tmp;
    const float *row = src + (int64_t)y * w;
    const int n = a.g.ntaps[layer], r = n / 2;
    const float *k = a.g.taps[layer];
    const bool fm = column_mode(x, w) <= 1;
    float acc = __fmul_rn(row[reflect101(x - r, w)], k[0]);
    for (int j = 1; j < n; ++j) {
        const float s = row[reflect101(x + j - r, w)];
        acc = fm ? __fmaf_rn(k[j], s, acc) : __fadd_rn(acc, __fmul_rn(k[j], s));
    }
    dst[i] = acc;
}

// column pass of layer `layer` into the Gaussian layer, and the DoG layer below it (layer > 0)
__global__ void __launch_bounds__(kThreads) col_kernel(Args a, int o, int layer, int from_dog)
{
    const int64_t f = blockIdx.y;
    const int h = a.g.h[o], w = a.g.w[o];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= (int64_t)h * w) return;
    const int y = (int)(i / w), x = (int)(i % w);
    const Frame fr = frame_of(a, f);
    const float *src = from_dog ? fr.dog : fr.tmp;
    const int n = a.g.ntaps[layer], r = n / 2;
    const float *k = a.g.taps[layer];
    const bool fm = column_mode(x, w) == 0;
    float acc = __fmul_rn(src[i], k[r]);
    for (int j = 1; j <= r; ++j) {
        const float s = __fadd_rn(src[(int64_t)reflect101(y - j, h) * w + x], src[(int64_t)reflect101(y + j, h) * w + x]);
        acc = fm ? __fmaf_rn(k[r + j], s, acc) : __fadd_rn(acc, __fmul_rn(k[r + j], s));
    }
    fr.gauss[(int64_t)layer * a.g.P + i] = acc;
    if (layer > 0) fr.dog[(int64_t)(layer - 1) * a.g.P + i] = __fsub_rn(acc, fr.gauss[(int64_t)(layer - 1) * a.g.P + i]);
}

// |v| > 1 and v >= (<= for v < 0) each of its 26 neighbours
__device__ __forceinline__ bool is_extremum(const float *D, int64_t P, int layer, int r, int c, int w)
{
    const float *cur = D + layer * P + (int64_t)r * w + c;
    const float v = *cur;
    if (!(fabsf(v) > 1.0f)) return false;
    bool ok = true;
#pragma unroll
    for (int l = -1; l <= 1; ++l)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                if (!l && !dy && !dx) continue;
                const float nb = cur[l * P + dy * w + dx];
                ok = ok && (v > 0.0f ? v >= nb : v <= nb);
            }
    return ok;
}

// exclusive prefix of v over the CTA; total gets the sum.  sh: 32 ints of shared memory.  Ends synchronised.
__device__ __forceinline__ int block_scan(int v, int &total, int *sh)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int s = lane < nw ? sh[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        sh[lane] = s;
    }
    __syncthreads();
    total = sh[nw - 1];
    const int p = (warp ? sh[warp - 1] : 0) + x - v;
    __syncthreads();
    return p;
}

// per (frame, DoG layer 1..3, row): the row's candidates are counted (emit = 0) or written in raster order (emit = 1)
__global__ void __launch_bounds__(kThreads) extrema_kernel(Args a, int o, int emit)
{
    __shared__ int sh[32];
    const int64_t f = blockIdx.z;
    const int layer = blockIdx.y + 1, r = blockIdx.x;
    const int h = a.g.h[o], w = a.g.w[o];
    const Frame fr = frame_of(a, f);
    const int slot = blockIdx.y * h + r;
    if (r < kBorder || r >= h - kBorder || w <= 2 * kBorder) {
        if (!emit && threadIdx.x == 0) fr.rows[slot] = 0;
        return;
    }
    int m = emit ? fr.rows[slot] : 0;
    for (int c0 = kBorder; c0 < w - kBorder; c0 += kThreads) {
        const int c = c0 + threadIdx.x;
        const bool e = c < w - kBorder && is_extremum(fr.dog, a.g.P, layer, r, c, w);
        int tot;
        const int p = block_scan(e, tot, sh);
        if (emit && e) fr.cand[m + p] = (layer << 24) | (r << 12) | c;
        m += tot;
    }
    if (!emit && threadIdx.x == 0) fr.rows[slot] = m;
}

// per frame: exclusive scan of n ints in place; the total into *total (add = 0) or added to it (add = 1), its old
// value into *old when old is not null
__device__ void scan_in_place(int32_t *v, int n, int32_t *total, int add, int32_t *old)
{
    __shared__ int sh[32];
    int m = 0;
    for (int s = 0; s < n; s += blockDim.x) {
        const int i = s + threadIdx.x;
        const int x = i < n ? v[i] : 0;
        int tot;
        const int p = block_scan(x, tot, sh);
        if (i < n) v[i] = m + p;
        m += tot;
    }
    if (threadIdx.x == 0) {
        if (old) *old = *total;
        *total = add ? *total + m : m;
    }
}

__global__ void __launch_bounds__(kScanThreads) scan_rows_kernel(Args a, int o)
{
    const Frame fr = frame_of(a, blockIdx.x);
    scan_in_place(fr.rows, 3 * a.g.h[o], fr.state, 0, nullptr);
}

__global__ void __launch_bounds__(kScanThreads) scan_copies_kernel(Args a)
{
    const int64_t f = blockIdx.x;
    const Frame fr = frame_of(a, f);
    scan_in_place(fr.ncopy, fr.state[0], a.count + a.f0 + f, 1, fr.state + 1);
}

// ------------------------------------------------------------------------------------ refinement and orientation

constexpr float kImgScale = 1.0f / 255.0f;

__device__ __forceinline__ float fms(float a, float b, float c, float d)      // a b - c d as fma(a, b, -(c d))
{
    return __fmaf_rn(a, b, -__fmul_rn(c, d));
}

__device__ __forceinline__ float cof3(float u, float p, float w, float q, float y, float r)
{
    return __fmaf_rn(y, r, __fmaf_rn(u, p, -__fmul_rn(w, q)));
}

struct Refined {
    int layer, r, c;
    float xc, xr, xi, contr;
};

// adjustLocalExtrema: false when rejected
__device__ bool refine(const float *D, int64_t P, int h, int w, int layer, int r, int c, Refined &out)
{
    const float ds = __fmul_rn(kImgScale, 0.5f), cs = __fmul_rn(kImgScale, 0.25f);
    float xi = 0.f, xr = 0.f, xc = 0.f;
    float dD0 = 0.f, dD1 = 0.f, dD2 = 0.f, dxx = 0.f, dyy = 0.f, dxy = 0.f;
    int i = 0;
    auto derivs = [&](float &dss, float &dxs, float &dys) {
        const float *img = D + layer * P + (int64_t)r * w + c, *prv = img - P, *nxt = img + P;
        dD0 = __fmul_rn(__fsub_rn(img[1], img[-1]), ds);
        dD1 = __fmul_rn(__fsub_rn(img[w], img[-w]), ds);
        dD2 = __fmul_rn(__fsub_rn(nxt[0], prv[0]), ds);
        const float v2 = __fmul_rn(img[0], 2.0f);
        dxx = __fmul_rn(__fsub_rn(__fadd_rn(img[1], img[-1]), v2), kImgScale);
        dyy = __fmul_rn(__fsub_rn(__fadd_rn(img[w], img[-w]), v2), kImgScale);
        dss = __fmul_rn(__fsub_rn(__fadd_rn(nxt[0], prv[0]), v2), kImgScale);
        dxy = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(img[w + 1], img[w - 1]), img[-w + 1]), img[-w - 1]), cs);
        dxs = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(nxt[1], nxt[-1]), prv[1]), prv[-1]), cs);
        dys = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(nxt[w], nxt[-w]), prv[w]), prv[-w]), cs);
    };
    for (; i < 5; ++i) {
        float dss, dxs, dys;
        derivs(dss, dxs, dys);
        // Matx33f::solve of H = [[dxx dxy dxs] [dxy dyy dys] [dxs dys dss]], b = dD (Cramer's rule)
        const float a00 = dxx, a01 = dxy, a02 = dxs, a10 = dxy, a11 = dyy, a12 = dys, a20 = dxs, a21 = dys, a22 = dss;
        const float det = cof3(a00, fms(a11, a22, a21, a12), a01, fms(a10, a22, a20, a12), a02, fms(a10, a21, a20, a11));
        float x0 = 0.f, x1 = 0.f, x2 = 0.f;
        if (det != 0.0f) {
            const float d = __fdiv_rn(1.0f, det);
            x0 = __fmul_rn(d, cof3(dD0, fms(a11, a22, a12, a21), a01, fms(dD1, a22, a12, dD2), a02, fms(dD1, a21, a11, dD2)));
            x1 = __fmul_rn(d, cof3(a00, fms(dD1, a22, a12, dD2), dD0, fms(a10, a22, a12, a20), a02, fms(a10, dD2, dD1, a20)));
            x2 = __fmul_rn(d, cof3(a00, fms(a11, dD2, dD1, a21), a01, fms(a10, dD2, dD1, a20), dD0, fms(a10, a21, a11, a20)));
        }
        xi = -x2;
        xr = -x1;
        xc = -x0;
        if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
        const float big = (float)(2147483647 / 3);
        if (fabsf(xi) > big || fabsf(xr) > big || fabsf(xc) > big) return false;
        c += __float2int_rn(xc);
        r += __float2int_rn(xr);
        layer += __float2int_rn(xi);
        if (layer < 1 || layer > kLayers || c < kBorder || c >= w - kBorder || r < kBorder || r >= h - kBorder)
            return false;
    }
    if (i >= 5) return false;
    float dss, dxs, dys;
    derivs(dss, dxs, dys);
    const float t = __fmaf_rn(dD2, xi, __fmaf_rn(dD1, xr, __fmul_rn(dD0, xc)));
    const float contr = __fmaf_rn(D[layer * P + (int64_t)r * w + c], kImgScale, __fmul_rn(t, 0.5f));
    if (__fmul_rn(fabsf(contr), 3.0f) < 0.04f) return false;
    const float tr = __fadd_rn(dxx, dyy);
    const float det = fms(dxx, dyy, dxy, dxy);
    if (det <= 0.0f || __fmul_rn(__fmul_rn(tr, tr), 10.0f) >= __fmul_rn(121.0f, det)) return false;
    out.layer = layer;
    out.r = r;
    out.c = c;
    out.xc = xc;
    out.xr = xr;
    out.xi = xi;
    out.contr = contr;
    return true;
}

__constant__ float c_exp_tab[64];

// exp32 of oracle/sift_oracle.py: OpenCV's table-and-polynomial exp32f in its vector form
__device__ __forceinline__ float exp32(float x)
{
    const float A4 = (float)(1.000000000000002438532970795181890933776 / .9670371139572337719125840413672004409288e-2);
    const float A3 = (float)(.6931471805521448196800669615864773144641 / .9670371139572337719125840413672004409288e-2);
    const float A2 = (float)(.2402265109513301490103372422686535526573 / .9670371139572337719125840413672004409288e-2);
    const float A1 = (float)(.5550339366753125211915322047004666939128e-1 / .9670371139572337719125840413672004409288e-2);
    x = __fmul_rn(fminf(fmaxf(x, -3000.0f), 3000.0f), (float)(1.4426950408889634073599246810019 * 64));
    const int xi = __float2int_rn(x);
    x = __fmul_rn(__fsub_rn(x, (float)xi), 1.0f / 64);
    const int t = min(max((xi >> 6) + 127, 0), 255);
    const float y = __fmul_rn(c_exp_tab[xi & 63], __int_as_float(t << 23));
    const float z = __fmaf_rn(__fmaf_rn(__fmaf_rn(__fadd_rn(x, A1), x, A2), x, A3), x, A4);
    return __fmul_rn(z, y);
}

// atan32: fastAtan2(y, x) in degrees, OpenCV's polynomial in its vector form
__device__ __forceinline__ float atan32(float y, float x)
{
    const float p1 = (float)(0.9997878412794807 * (180 / 3.141592653589793));
    const float p3 = (float)(-0.3258083974640975 * (180 / 3.141592653589793));
    const float p5 = (float)(0.1555786518463281 * (180 / 3.141592653589793));
    const float p7 = (float)(-0.04432655554792128 * (180 / 3.141592653589793));
    const float ax = fabsf(x), ay = fabsf(y);
    const float c = __fdiv_rn(fminf(ax, ay), __fadd_rn(fmaxf(ax, ay), (float)2.220446049250313e-16));
    const float cc = __fmul_rn(c, c);
    float a = __fmul_rn(__fmaf_rn(__fmaf_rn(__fmaf_rn(cc, p7, p5), cc, p3), cc, p1), c);
    if (!(ax >= ay)) a = __fsub_rn(90.0f, a);
    if (x < 0.0f) a = __fsub_rn(180.0f, a);
    if (y < 0.0f) a = __fsub_rn(360.0f, a);
    return a;
}

struct WarpSmem {
    float wm[kMaxWin];                // W mag, rounded (vector part of the window)
    uint8_t bin[kMaxWin];
    float tw[16], tm[16];             // W and mag of the last len mod 16 pixels
    float hist[kBins];
};

// One warp: candidate `ci` of the frame refined and its smoothed orientation histogram built.  Returns the peak mask
// (bit j: bin j is a kept peak), or 0 when the candidate is rejected; `k` and `hist` (in shared memory) describe it.
__device__ uint64_t orient(const Args &a, const Frame &fr, int o, int ci, WarpSmem &s, Refined &k, float &scl)
{
    const int lane = threadIdx.x & 31;
    const int h = a.g.h[o], w = a.g.w[o];
    const int32_t cd = fr.cand[ci];
    if (!refine(fr.dog, a.g.P, h, w, cd >> 24, (cd >> 12) & 4095, cd & 4095, k)) return 0;
    const float y = __fdiv_rn(__fadd_rn((float)k.layer, k.xi), 3.0f);
    const float p = __double2float_rn(exp2((double)y));
    // size before firstOctave's halving is 1.6 p 2^o 2; scl_octv = size 0.5 / 2^o
    scl = __fmul_rn(1.6f, p);
    const int radius = __float2int_rn(__fmul_rn(4.5f, scl));
    const float sig = __fmul_rn(1.5f, scl);
    const float escale = __fdiv_rn(-1.0f, __fmul_rn(__fmul_rn(2.0f, sig), sig));
    const float *img = fr.gauss + (int64_t)k.layer * a.g.P;
    // the window's valid rows and columns: each valid row holds the same valid columns
    const int i0 = max(-radius, 1 - k.r), i1 = min(radius, h - 2 - k.r);
    const int j0 = max(-radius, 1 - k.c), j1 = min(radius, w - 2 - k.c);
    const int nr = max(i1 - i0 + 1, 0), nc = max(j1 - j0 + 1, 0);
    const int len = nr * nc, vec = len / 16 * 16;
    for (int q = lane; q < len; q += 32) {
        const int i = i0 + q / nc, j = j0 + q % nc;
        const float *px = img + (int64_t)(k.r + i) * w + (k.c + j);
        const float dx = __fsub_rn(px[1], px[-1]), dy = __fsub_rn(px[-w], px[w]);
        const float W = exp32(__fmul_rn((float)(i * i + j * j), escale));
        const float ori = atan32(dy, dx);
        const float mag = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
        int b = __float2int_rn(__fmul_rn(0.1f, ori));
        if (b >= kBins) b -= kBins;
        if (b < 0) b += kBins;
        s.bin[q] = (uint8_t)b;
        if (q < vec) {
            s.wm[q] = __fmul_rn(W, mag);
        } else {
            s.tw[q - vec] = W;
            s.tm[q - vec] = mag;
        }
    }
    __syncwarp();
    float h0 = 0.f, h1 = 0.f;           // bins lane and lane + 32, summed in pixel order
    for (int q = 0; q < len; ++q) {
        const int b = s.bin[q];
        if (b == lane || b == lane + 32) {
            const float acc = b == lane ? h0 : h1;
            const float v = q < vec ? __fadd_rn(acc, s.wm[q]) : __fmaf_rn(s.tw[q - vec], s.tm[q - vec], acc);
            if (b == lane) h0 = v; else h1 = v;
        }
    }
    __syncwarp();
    // the 5-tap smoothing over circular bins: vector form for bins < 32, the scalar tail's for 32..35
    auto H = [&](int j) {
        j = (j + kBins) % kBins;
        const float v0 = __shfl_sync(0xffffffffu, h0, j & 31), v1 = __shfl_sync(0xffffffffu, h1, j & 31);
        return j < 32 ? v0 : v1;
    };
    float sm[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int j = lane + 32 * u;
        const float tm2 = H(j - 2), tm1 = H(j - 1), t0 = H(j), tp1 = H(j + 1), tp2 = H(j + 2);
        const float A = __fadd_rn(tm2, tp2), Bv = __fadd_rn(tm1, tp1);
        sm[u] = j < 32 ? __fmaf_rn(A, 1.0f / 16, __fmaf_rn(Bv, 4.0f / 16, __fmul_rn(t0, 6.0f / 16)))
                       : __fmaf_rn(t0, 6.0f / 16, __fadd_rn(__fmul_rn(A, 1.0f / 16), __fmul_rn(Bv, 4.0f / 16)));
    }
    s.hist[lane] = sm[0];
    if (lane < kBins - 32) s.hist[lane + 32] = sm[1];
    __syncwarp();
    float mx = s.hist[0];
    for (int j = 1; j < kBins; ++j) mx = fmaxf(mx, s.hist[j]);
    const float thr = __fmul_rn(mx, 0.8f);
    uint64_t mask = 0;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int j = lane + 32 * u;
        bool pk = false;
        if (j < kBins) {
            const float hl = s.hist[(j + kBins - 1) % kBins], hr = s.hist[(j + 1) % kBins], hj = s.hist[j];
            pk = hj > hl && hj > hr && hj >= thr;
        }
        mask |= (uint64_t)__ballot_sync(0xffffffffu, pk) << (32 * u);
    }
    return mask;
}

__global__ void __launch_bounds__(kOriWarps * 32) orient_kernel(Args a, int o, int write)
{
    __shared__ WarpSmem smem[kOriWarps];
    const int64_t f = blockIdx.y;
    const Frame fr = frame_of(a, f);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    WarpSmem &s = smem[warp];
    const int n = fr.state[0];
    const int64_t base = fr.state[1];
    float *pt = a.pt + (a.f0 + f) * a.cap * 2, *size = a.size + (a.f0 + f) * a.cap;
    float *ang = a.angle + (a.f0 + f) * a.cap, *resp = a.resp + (a.f0 + f) * a.cap;
    int32_t *oc = a.oct + (a.f0 + f) * a.cap;
    for (int ci = blockIdx.x * kOriWarps + warp; ci < n; ci += gridDim.x * kOriWarps) {
        Refined k;
        float scl;
        const uint64_t mask = orient(a, fr, o, ci, s, k, scl);
        if (!write) {
            if (lane == 0) fr.ncopy[ci] = __popcll(mask);
            __syncwarp();
            continue;
        }
        // keypoint j of this candidate goes to base + ncopy[ci] (the scanned offset) + its rank among the peaks
        const int64_t at = base + fr.ncopy[ci];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int j = lane + 32 * u;
            if (j < kBins && ((mask >> j) & 1)) {
                const int64_t idx = at + __popcll(mask & ((1ull << j) - 1));
                if (idx < a.cap) {
                    const float hl = s.hist[(j + kBins - 1) % kBins], hr = s.hist[(j + 1) % kBins], hj = s.hist[j];
                    float b = __fadd_rn((float)j, __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(hl, hr)),
                                                             __fadd_rn(__fsub_rn(hl, __fmul_rn(2.0f, hj)), hr)));
                    b = b < 0.0f ? __fadd_rn(b, (float)kBins) : (b >= (float)kBins ? __fsub_rn(b, (float)kBins) : b);
                    float an = __fsub_rn(360.0f, __fmul_rn(10.0f, b));
                    if (fabsf(__fsub_rn(an, 360.0f)) < 1.1920928955078125e-07f) an = 0.0f;
                    const float sc = __fmul_rn((float)(1 << o), 0.5f);
                    pt[idx * 2] = __fmul_rn(__fadd_rn((float)k.c, k.xc), sc);
                    pt[idx * 2 + 1] = __fmul_rn(__fadd_rn((float)k.r, k.xr), sc);
                    const int q = __double2int_rn(__dmul_rn(__dadd_rn((double)k.xi, 0.5), 255.0));
                    const int packed = o + (k.layer << 8) + (q << 16);
                    oc[idx] = (packed & ~255) | ((o - 1) & 255);
                    size[idx] = __fmul_rn(scl, (float)(1 << o));       // (1.6 p 2^o 2) / 2, exact scalings
                    resp[idx] = fabsf(k.contr);
                    ang[idx] = an;
                }
            }
        }
        __syncwarp();
    }
}

// removeDuplicatedSorted: of keypoints with equal (pt, size, angle) the one of larger (response, packed octave), the
// earlier on ties, is kept; the kept ones are compacted in order.  One CTA per frame, when everything fitted.
__global__ void __launch_bounds__(kDedupThreads) dedup_kernel(Args a)
{
    constexpr int T = kDedupThreads;
    __shared__ float sx[T], sy[T], ss[T], sa[T], sr[T];
    __shared__ int so[T];
    __shared__ int scan_sh[32];
    const int64_t fg = a.f0 + blockIdx.x;
    const int n = a.count[fg];
    if (n > a.cap || n <= 1) return;
    float *pt = a.pt + fg * a.cap * 2, *size = a.size + fg * a.cap, *ang = a.angle + fg * a.cap;
    float *resp = a.resp + fg * a.cap;
    int32_t *oc = a.oct + fg * a.cap;
    // pass 1: mark the dropped ones in bit 31 of the packed octave (the packing stays below 2^24)
    for (int s0 = 0; s0 < n; s0 += T) {
        const int i = s0 + threadIdx.x;
        float x = 0.f, y = 0.f, z = 0.f, an = 0.f, r = 0.f;
        int ob = 0;
        if (i < n) {
            x = pt[2 * i];
            y = pt[2 * i + 1];
            z = size[i];
            an = ang[i];
            r = resp[i];
            ob = oc[i] & 0x7fffffff;
        }
        bool drop = false;
        for (int t0 = 0; t0 < n; t0 += T) {
            __syncthreads();
            const int j = t0 + threadIdx.x;
            if (j < n) {
                sx[threadIdx.x] = pt[2 * j];
                sy[threadIdx.x] = pt[2 * j + 1];
                ss[threadIdx.x] = size[j];
                sa[threadIdx.x] = ang[j];
                sr[threadIdx.x] = resp[j];
                so[threadIdx.x] = oc[j] & 0x7fffffff;
            }
            __syncthreads();
            const int m = min(T, n - t0);
            if (i < n)
                for (int u = 0; u < m; ++u) {
                    const int j2 = t0 + u;
                    if (j2 == i || __float_as_uint(sx[u]) != __float_as_uint(x) ||
                        __float_as_uint(sy[u]) != __float_as_uint(y) || __float_as_uint(ss[u]) != __float_as_uint(z) ||
                        __float_as_uint(sa[u]) != __float_as_uint(an))
                        continue;
                    drop = drop || sr[u] > r || (sr[u] == r && (so[u] > ob || (so[u] == ob && j2 < i)));
                }
        }
        __syncthreads();
        if (i < n && drop) oc[i] = ob | (int)0x80000000;
    }
    __syncthreads();
    int kept = 0;
    for (int s0 = 0; s0 < n; s0 += T) {
        const int i = s0 + threadIdx.x;
        float x = 0.f, y = 0.f, z = 0.f, an = 0.f, r = 0.f;
        int ob = 0;
        bool f = false;
        if (i < n) {
            x = pt[2 * i];
            y = pt[2 * i + 1];
            z = size[i];
            an = ang[i];
            r = resp[i];
            ob = oc[i];
            f = ob >= 0;
        }
        int tot;
        const int p = block_scan(f, tot, scan_sh);      // every read of the chunk happens before this returns
        if (f) {
            pt[2 * (kept + p)] = x;
            pt[2 * (kept + p) + 1] = y;
            size[kept + p] = z;
            ang[kept + p] = an;
            resp[kept + p] = r;
            oc[kept + p] = ob;
        }
        kept += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) a.count[fg] = kept;
}

bool sizes_ok(int64_t B, int64_t H, int64_t W)
{
    return B >= 0 && B <= FFB6D_SIFT_MAX_FRAMES && H >= FFB6D_SIFT_MIN_SIDE && W >= FFB6D_SIFT_MIN_SIDE &&
           H <= FFB6D_SIFT_MAX_SIDE && W <= FFB6D_SIFT_MAX_SIDE;
}

inline bool aligned(const void *p, size_t al) { return ((uintptr_t)p % al) == 0; }

int exp_table_ready()
{
    static std::atomic<unsigned long long> done{0};
    const int dev = current_device() & (kMaxDevices - 1);
    if ((done.load(std::memory_order_relaxed) >> dev) & 1ull) return FFB6D_OK;
    float tab[64];
    for (int i = 0; i < 64; ++i) tab[i] = (float)(std::pow(2.0, i / 64.0) * .9670371139572337719125840413672004409288e-2);
    FFB6D_CUDA(cudaMemcpyToSymbol(c_exp_tab, tab, sizeof(tab)));
    done.fetch_or(1ull << dev, std::memory_order_relaxed);
    return FFB6D_OK;
}

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" int64_t ffb6d_sift_capacity(int64_t H, int64_t W)
{
    if (!sizes_ok(0, H, W)) return 0;
    return std::max<int64_t>(H * W / 16, 256);
}

extern "C" size_t ffb6d_sift_workspace_bytes(int64_t B, int64_t H, int64_t W)
{
    if (!sizes_ok(B, H, W)) return 0;
    return (size_t)std::min<int64_t>(B, kChunk) * (size_t)make_geom(H, W).frame;
}

extern "C" int ffb6d_sift_detect(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, int32_t *count, float *pt,
                                 int32_t *octave, float *size, float *angle, float *response, int64_t cap,
                                 void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(sizes_ok(B, H, W), "sift_detect: bad size (B=%lld H=%lld W=%lld)", (long long)B, (long long)H,
                    (long long)W);
    FFB6D_CHECK_ARG(cap >= 0 && cap <= FFB6D_SIFT_MAX_CAP, "sift_detect: cap=%lld outside [0, %d]", (long long)cap,
                    FFB6D_SIFT_MAX_CAP);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(rgb && count && (cap == 0 || (pt && octave && size && angle && response)),
                    "sift_detect: null pointer");
    FFB6D_CHECK_ARG(aligned(count, 4) && aligned(pt, 4) && aligned(octave, 4) && aligned(size, 4) &&
                    aligned(angle, 4) && aligned(response, 4) && aligned(workspace, 16),
                    "sift_detect: misaligned pointer");
    const size_t need = ffb6d_sift_workspace_bytes(B, H, W);
    if (!workspace || workspace_bytes < need) {
        set_error("sift_detect: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }
    const int rc = exp_table_ready();
    if (rc != FFB6D_OK) return rc;
    Args a;
    a.rgb = rgb;
    a.H = H;
    a.W = W;
    a.g = make_geom(H, W);
    a.ws = (uint8_t *)workspace;
    a.count = count;
    a.pt = pt;
    a.size = size;
    a.angle = angle;
    a.resp = response;
    a.oct = octave;
    a.cap = cap;
    const Geom &g = a.g;
    cudaStream_t st = (cudaStream_t)stream;
    FFB6D_CUDA(cudaMemsetAsync(count, 0, (size_t)B * sizeof(int32_t), st));
    for (int64_t f0 = 0; f0 < B; f0 += kChunk) {
        a.f0 = f0;
        const unsigned C = (unsigned)std::min<int64_t>(B - f0, kChunk);
        for (int o = 0; o < g.n_oct; ++o) {
            const unsigned nb = (unsigned)ceil_div((int64_t)g.h[o] * g.w[o], kThreads);
            if (o == 0) {
                upscale_kernel<<<dim3(nb, C), kThreads, 0, st>>>(a);
                FFB6D_LAUNCH_OK("sift_upscale_kernel");
                row_kernel<<<dim3(nb, C), kThreads, 0, st>>>(a, 0, 0, 1);
                FFB6D_LAUNCH_OK("sift_row_kernel");
                col_kernel<<<dim3(nb, C), kThreads, 0, st>>>(a, 0, 0, 1);
                FFB6D_LAUNCH_OK("sift_col_kernel");
            } else {
                downsample_kernel<<<dim3(nb, C), kThreads, 0, st>>>(a, o);
                FFB6D_LAUNCH_OK("sift_downsample_kernel");
            }
            for (int l = 1; l < kGauss; ++l) {
                row_kernel<<<dim3(nb, C), kThreads, 0, st>>>(a, o, l, 0);
                FFB6D_LAUNCH_OK("sift_row_kernel");
                col_kernel<<<dim3(nb, C), kThreads, 0, st>>>(a, o, l, 0);
                FFB6D_LAUNCH_OK("sift_col_kernel");
            }
            const dim3 rows((unsigned)g.h[o], kLayers, C);
            extrema_kernel<<<rows, kThreads, 0, st>>>(a, o, 0);
            FFB6D_LAUNCH_OK("sift_extrema_kernel");
            scan_rows_kernel<<<C, kScanThreads, 0, st>>>(a, o);
            FFB6D_LAUNCH_OK("sift_scan_rows_kernel");
            extrema_kernel<<<rows, kThreads, 0, st>>>(a, o, 1);
            FFB6D_LAUNCH_OK("sift_extrema_kernel");
            orient_kernel<<<dim3(kOriCtas, C), kOriWarps * 32, 0, st>>>(a, o, 0);
            FFB6D_LAUNCH_OK("sift_orient_kernel");
            scan_copies_kernel<<<C, kScanThreads, 0, st>>>(a);
            FFB6D_LAUNCH_OK("sift_scan_copies_kernel");
            orient_kernel<<<dim3(kOriCtas, C), kOriWarps * 32, 0, st>>>(a, o, 1);
            FFB6D_LAUNCH_OK("sift_orient_kernel");
        }
        dedup_kernel<<<C, kDedupThreads, 0, st>>>(a);
        FFB6D_LAUNCH_OK("sift_dedup_kernel");
    }
    return FFB6D_OK;
}

extern "C" int ffb6d_sift_lift(const int32_t *count, const float *pt, int64_t cap, const float *depth, int64_t B,
                               int64_t H, int64_t W, const double *intrinsics, int intrinsics_per_frame,
                               const double *RTs, int64_t views, float *cloud, int32_t *n_points,
                               ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(sizes_ok(B, H, W), "sift_lift: bad size (B=%lld H=%lld W=%lld)", (long long)B, (long long)H,
                    (long long)W);
    FFB6D_CHECK_ARG(cap >= 0 && cap <= FFB6D_SIFT_MAX_CAP, "sift_lift: cap=%lld outside [0, %d]", (long long)cap,
                    FFB6D_SIFT_MAX_CAP);
    FFB6D_CHECK_ARG(views >= 1 && B % views == 0 && B / views <= FFB6D_SIFT_MAX_FRAMES && views * cap < (1ll << 31),
                    "sift_lift: B=%lld frames must be whole objects of views=%lld, views cap < 2^31", (long long)B,
                    (long long)views);
    FFB6D_CHECK_ARG(intrinsics_per_frame == 0 || intrinsics_per_frame == 1,
                    "sift_lift: intrinsics_per_frame must be 0 or 1");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(count && pt && depth && intrinsics && RTs && cloud && n_points, "sift_lift: null pointer");
    FFB6D_CHECK_ARG(aligned(count, 4) && aligned(pt, 4) && aligned(depth, 4) && aligned(intrinsics, 8) &&
                    aligned(RTs, 8) && aligned(cloud, 4) && aligned(n_points, 4), "sift_lift: misaligned pointer");
    return keypoint_lift_launch(count, pt, cap, depth, B, H, W, intrinsics, intrinsics_per_frame, RTs, views, cloud,
                                n_points, (cudaStream_t)stream);
}
