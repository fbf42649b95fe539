// orb.cu -- ORB keypoints of cv2.ORB_create()'s defaults and their lift onto the mesh (sm_90a), DESIGN.md §4.32.
//
// The specification is the header's (ffb6d_orb_detect, ffb6d_orb_lift) and oracle/orb_oracle.py restates it in numpy.
// Every step is exact integer arithmetic except the Harris response (float32, one _rn intrinsic per operation, as
// OpenCV's scalar loop rounds it) and the lift (float64 _rn intrinsics), so the outputs are bitwise the oracle's.
//
// Launches, all with shapes that depend on the arguments only:
//   memset   count[B] to 0;
//   grey     level 0 of every frame from its RGB pixels;
//   resize   one launch per level 1..7 over all frames, each reading the level before (INTER_LINEAR_EXACT);
//   fast     one launch per level: the FAST score of every pixel into a raw score map;
//   nms      one launch per level: a 32x8 tile of raw scores with a 1-pixel halo in shared memory, strict 3x3
//            non-maximum suppression and the border filter, into the candidate map (0: no candidate);
//   select   one launch per level, one CTA per frame: a 256-bin histogram of the FAST scores gives the first cut,
//            candidates at or above it are compacted in raster order (block scans, no atomics on positions) with
//            their Harris responses, a radix select on order-preserving keys gives the second cut, and the kept
//            points are compacted in place behind the frame's earlier levels.  The launch for level l reads
//            count[b] as the launch for level l-1 left it.
// ffb6d_orb_lift is one launch, one CTA per object, walking its views in order with the same block scan.
#include "common.cuh"

#include <cmath>

namespace ffb6d {
namespace {

constexpr int kLevels = FFB6D_ORB_LEVELS;
constexpr int kBorder = 31;             // ORB's edgeThreshold
constexpr int kFastT = 20;
constexpr int kThreads = 256;
constexpr int kSelThreads = 1024;
constexpr int kTX = 32, kTY = 8;        // fast tile
constexpr int kNFeatures = 500;

struct Geom {
    int h[kLevels], w[kLevels];
    int64_t off[kLevels];               // byte offset of the level in a frame's pyramid
    int64_t frame;                      // bytes of one frame's pyramid
    int64_t cap_off[kLevels + 1];       // capacity bound of the levels before l
    float scale[kLevels];
    int budget[kLevels];
};

// cv::ORB's per-level sizes, scales and budgets, in the float32 arithmetic OpenCV uses (host)
Geom make_geom(int64_t H, int64_t W)
{
    Geom g;
    int64_t off = 0;
    g.cap_off[0] = 0;
    const double sf = (double)1.2f;
    for (int l = 0; l < kLevels; ++l) {
        const float s = (float)std::pow(sf, (double)l);
        const float inv = 1.0f / s;
        g.scale[l] = s;
        g.h[l] = (int)std::nearbyint((float)H * inv);
        g.w[l] = (int)std::nearbyint((float)W * inv);
        g.off[l] = off;
        off += (int64_t)g.h[l] * g.w[l];
        const int64_t rw = std::max(g.w[l] - 2 * kBorder, 0), rh = std::max(g.h[l] - 2 * kBorder, 0);
        g.cap_off[l + 1] = g.cap_off[l] + ((rw + 1) / 2) * ((rh + 1) / 2);
    }
    g.frame = align_up((size_t)off, 16);
    const float factor = (float)(1.0 / sf);
    float nd = (float)kNFeatures * (1.0f - factor) / (1.0f - (float)std::pow((double)factor, (double)kLevels));
    int sum = 0;
    for (int l = 0; l < kLevels - 1; ++l) {
        g.budget[l] = (int)std::nearbyint(nd);
        sum += g.budget[l];
        nd *= factor;
    }
    g.budget[kLevels - 1] = std::max(kNFeatures - sum, 0);
    return g;
}

struct Args {
    const uint8_t *rgb;
    int64_t B;
    Geom g;
    uint8_t *pyr, *raw, *score;
    int32_t *count;
    float *pt, *resp;
    int32_t *oct;
    int64_t cap;
};

__global__ void __launch_bounds__(kThreads) grey_kernel(Args a)
{
    const int64_t b = blockIdx.y, n = (int64_t)a.g.h[0] * a.g.w[0];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= n) return;
    const uint8_t *p = a.rgb + (b * n + i) * 3;
    const int r = p[0], gg = p[1], bl = p[2];
    a.pyr[b * a.g.frame + i] = (uint8_t)((3735 * bl + 19235 * gg + 9798 * r + (1 << 14)) >> 15);
}

// INTER_LINEAR_EXACT taps of destination coordinate d: source index s, and the weight of s + 1 in 1/256
__device__ __forceinline__ void taps(int d, int src, int dst, int &s0, int &s1, int &w1)
{
    const double f = __dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), __ddiv_rn((double)src, (double)dst)), 0.5);
    const double fl = floor(f);
    int s = (int)fl;
    w1 = __double2int_rn(__dmul_rn(__dsub_rn(f, fl), 256.0));
    if (s < 0 || s >= src - 1) {
        s = s < 0 ? 0 : src - 1;
        w1 = 0;
    }
    s0 = s;
    s1 = min(s + 1, src - 1);
}

__global__ void __launch_bounds__(kThreads) resize_kernel(Args a, int l)
{
    const int sh = a.g.h[l - 1], sw = a.g.w[l - 1], dh = a.g.h[l], dw = a.g.w[l];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= (int64_t)dh * dw) return;
    const int y = (int)(i / dw), x = (int)(i % dw);
    const uint8_t *src = a.pyr + blockIdx.y * a.g.frame + a.g.off[l - 1];
    int x0, x1, wx, y0, y1, wy;
    taps(x, sw, dw, x0, x1, wx);
    taps(y, sh, dh, y0, y1, wy);
    const int r0 = src[(int64_t)y0 * sw + x0] * (256 - wx) + src[(int64_t)y0 * sw + x1] * wx;
    const int r1 = src[(int64_t)y1 * sw + x0] * (256 - wx) + src[(int64_t)y1 * sw + x1] * wx;
    const int v = r0 * (256 - wy) + r1 * wy;
    a.pyr[blockIdx.y * a.g.frame + a.g.off[l] + i] = (uint8_t)((v + (1 << 15)) >> 16);
}

// 16-bit mask of the circle pixels p with p - v > t (bright) or v - p > t (dark)
__device__ __forceinline__ bool arc9(unsigned int m)
{
    m |= m << 16;                               // the circle wraps around
    unsigned int r = m;
#pragma unroll
    for (int j = 1; j < 9; ++j) r &= m >> j;
    return (r & 0xffffu) != 0;
}

// FAST-9/16 score of one pixel at least 3 from every edge: the largest t >= 20 for which 9 contiguous circle pixels
// are all brighter than v + t or all darker than v - t (OpenCV's cornerScore, max over arcs of the arc's least
// difference, minus 1), 0 when t = 20 already fails.  corner(t) only weakens as t grows, so a binary search over t
// finds it with comparisons and masks alone (ptxas folds a min / max formulation into three-operand VIMNMX3, which
// gave wrong scores on the H100).
__device__ __forceinline__ int fast_score(const uint8_t *p, int w)
{
    const int cx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    const int cy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
    const int v = p[0];
    int d[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) d[c] = (int)p[cy[c] * w + cx[c]] - v;
    auto corner = [&](int t) {
        unsigned int br = 0, dk = 0;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            br |= (unsigned int)(d[c] > t) << c;
            dk |= (unsigned int)(d[c] < -t) << c;
        }
        return arc9(br) || arc9(dk);
    };
    if (!corner(kFastT)) return 0;
    int lo = kFastT, hi = 255;                  // corner(lo) holds, corner(hi) fails (|d| <= 255)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (corner(mid)) lo = mid; else hi = mid;
    }
    return lo;
}

// raw FAST scores of level l into the score map, one thread per pixel (0 within 3 of an edge)
__global__ void __launch_bounds__(kThreads) fast_kernel(Args a, int l)
{
    const int h = a.g.h[l], w = a.g.w[l];
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= (int64_t)h * w) return;
    const int y = (int)(i / w), x = (int)(i % w);
    const int64_t base = blockIdx.y * a.g.frame + a.g.off[l];
    int s = 0;
    if (y >= 3 && y < h - 3 && x >= 3 && x < w - 3) s = fast_score(a.pyr + base + i, w);
    a.raw[base + i] = (uint8_t)s;
}

// strict 3x3 non-maximum suppression and the border filter of level l: a 32x8 tile of raw scores with a 1-pixel halo
// staged in shared memory; the score map keeps a candidate's score, 0 elsewhere
__global__ void __launch_bounds__(kTX * kTY) nms_kernel(Args a, int l)
{
    constexpr int SX = kTX + 2, SY = kTY + 2;
    __shared__ uint8_t sc[SY][SX];
    const int h = a.g.h[l], w = a.g.w[l];
    const int64_t base = blockIdx.z * a.g.frame + a.g.off[l];
    const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY;
    for (int k = threadIdx.y * kTX + threadIdx.x; k < SX * SY; k += kTX * kTY) {
        const int y = y0 - 1 + k / SX, x = x0 - 1 + k % SX;
        sc[k / SX][k % SX] = (y >= 0 && y < h && x >= 0 && x < w) ? a.raw[base + (int64_t)y * w + x] : 0;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= w || y >= h) return;
    const int s = sc[threadIdx.y + 1][threadIdx.x + 1];
    bool keep = s > 0 && x >= kBorder && x < w - kBorder && y >= kBorder && y < h - kBorder;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx)
            if (dy || dx) keep = keep && s > sc[threadIdx.y + 1 + dy][threadIdx.x + 1 + dx];
    a.score[base + (int64_t)y * w + x] = keep ? (uint8_t)s : 0;
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

__device__ __forceinline__ float harris(const uint8_t *img, int w, int x, int y)
{
    int A = 0, B = 0, C = 0;
    for (int i = -3; i <= 3; ++i) {
        const uint8_t *r = img + (int64_t)(y + i) * w + x;
        for (int j = -3; j <= 3; ++j) {
            const uint8_t *p = r + j;
            const int Ix = (p[1] - p[-1]) * 2 + (p[-w + 1] - p[-w - 1]) + (p[w + 1] - p[w - 1]);
            const int Iy = (p[w] - p[-w]) * 2 + (p[w - 1] - p[-w - 1]) + (p[w + 1] - p[-w + 1]);
            A += Ix * Ix;
            B += Iy * Iy;
            C += Ix * Iy;
        }
    }
    const float scale = __fdiv_rn(1.0f, 7140.0f);       // 1 / ((1 << 2) 7 255)
    const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
    const float fa = __int2float_rn(A), fb = __int2float_rn(B), fc = __int2float_rn(C);
    const float t = __fadd_rn(fa, fb);
    const float r = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, t), t));
    return __fmul_rn(r, s4);
}

// order-preserving key of a float (-0 taken as +0, as the float comparisons of retainBest do)
__device__ __forceinline__ unsigned int fkey(float f)
{
    const unsigned int u = __float_as_uint(f == 0.0f ? 0.0f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(kSelThreads) select_kernel(Args a, int l)
{
    __shared__ int hist[256];
    __shared__ int scan_sh[32];
    __shared__ int cut;
    const int64_t b = blockIdx.x;
    const int h = a.g.h[l], w = a.g.w[l];
    const int rw = w - 2 * kBorder, rh = h - 2 * kBorder;
    if (rw <= 0 || rh <= 0) return;
    const int R = rw * rh;
    const uint8_t *score = a.score + b * a.g.frame + a.g.off[l];
    const uint8_t *img = a.pyr + b * a.g.frame + a.g.off[l];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
        const int s = score[(int64_t)(kBorder + i / rw) * w + kBorder + i % rw];
        if (s) atomicAdd(&hist[s], 1);
    }
    __syncthreads();
    const int n2 = 2 * a.g.budget[l], n1 = a.g.budget[l];
    if (threadIdx.x == 0) {
        int total = 0;
        for (int s = 1; s < 256; ++s) total += hist[s];
        int c = 1;                                      // keep every candidate
        if (total > n2) {
            if (n2 == 0) {
                c = 256;                                // keep none
            } else {
                int cum = 0;
                for (c = 255; c >= 1; --c) {
                    cum += hist[c];
                    if (cum >= n2) break;
                }
            }
        }
        cut = c;
    }
    __syncthreads();
    const int c1 = cut;
    const int64_t base = a.count[b];
    const int64_t o = b * a.cap + base;
    float *pt = a.pt + o * 2;
    float *resp = a.resp + o;
    int32_t *oct = a.oct + o;
    const float sl = a.g.scale[l];
    int m = 0;
    for (int start = 0; start < R; start += blockDim.x) {
        const int i = start + threadIdx.x;
        int x = 0, y = 0;
        bool f = false;
        if (i < R) {
            y = kBorder + i / rw;
            x = kBorder + i % rw;
            const int s = score[(int64_t)y * w + x];
            f = s > 0 && s >= c1;
        }
        int tot;
        const int p = block_scan(f, tot, scan_sh);
        if (f) {
            pt[(m + p) * 2] = __fmul_rn((float)x, sl);
            pt[(m + p) * 2 + 1] = __fmul_rn((float)y, sl);
            resp[m + p] = harris(img, w, x, y);
            oct[m + p] = l;
        }
        m += tot;
    }
    __syncthreads();
    if (m > n1) {
        unsigned int kth = 0;
        if (n1 > 0) {
            unsigned int prefix = 0, mask = 0;
            int rank = n1;
            for (int shift = 24; shift >= 0; shift -= 8) {
                for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
                __syncthreads();
                for (int i = threadIdx.x; i < m; i += blockDim.x) {
                    const unsigned int k = fkey(resp[i]);
                    if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1);
                }
                __syncthreads();
                if (threadIdx.x == 0) {
                    int cum = 0, d = 255;
                    for (; d > 0; --d) {
                        if (cum + hist[d] >= rank) break;
                        cum += hist[d];
                    }
                    cut = d;
                    hist[0] = rank - cum;       // the rank within the chosen digit (hist is cleared next round)
                }
                __syncthreads();
                prefix |= (unsigned int)cut << shift;
                mask |= 255u << shift;
                rank = hist[0];
                __syncthreads();
            }
            kth = prefix;
        } else {
            kth = 0xffffffffu;                  // n1 = 0: keep none (no key exceeds it: keys of floats < 2^32 - 1)
        }
        int kept = 0;
        for (int start = 0; start < m; start += blockDim.x) {
            const int i = start + threadIdx.x;
            float px = 0.f, py = 0.f, r = 0.f;
            bool f = false;
            if (i < m) {
                px = pt[i * 2];
                py = pt[i * 2 + 1];
                r = resp[i];
                f = n1 > 0 && fkey(r) >= kth;
            }
            int tot;
            const int p = block_scan(f, tot, scan_sh);      // every read of the chunk happens before this returns
            if (f) {
                pt[(kept + p) * 2] = px;
                pt[(kept + p) * 2 + 1] = py;
                resp[kept + p] = r;
                oct[kept + p] = l;
            }
            kept += tot;
            __syncthreads();
        }
        m = kept;
    }
    if (threadIdx.x == 0) a.count[b] = (int32_t)(base + m);
}

struct LiftArgs {
    const int32_t *count;
    const float *pt;
    int64_t cap;
    const float *depth;
    int H, W;
    const double *intr;
    int intr_per_frame;
    const double *RTs;
    int64_t views;
    float *cloud;
    int32_t *n_points;
};

__global__ void __launch_bounds__(kThreads) lift_kernel(LiftArgs a)
{
    __shared__ int scan_sh[32];
    const int64_t obj = blockIdx.x;
    float *out = a.cloud + obj * a.views * a.cap * 3;
    int64_t m = 0;
    for (int64_t v = 0; v < a.views; ++v) {
        const int64_t b = obj * a.views + v;
        const int n = a.count[b];
        const float *pt = a.pt + b * a.cap * 2;
        const float *dep = a.depth + b * (int64_t)a.H * a.W;
        const double *k = a.intr + (a.intr_per_frame ? b * 4 : 0);
        const double *rt = a.RTs + b * 12;
        for (int start = 0; start < n; start += kThreads) {
            const int i = start + threadIdx.x;
            bool f = false;
            double q[3];
            if (i < n) {
                const float fx = pt[i * 2], fy = pt[i * 2 + 1];
                if (fx >= 0.f && fy >= 0.f && fx < (float)a.W && fy < (float)a.H) {
                    const int u = (int)fx, w = (int)fy;
                    const double z = (double)dep[(int64_t)w * a.W + u];
                    const double x = __ddiv_rn(__dmul_rn(__dsub_rn((double)u, k[2]), z), k[0]);
                    const double y = __ddiv_rn(__dmul_rn(__dsub_rn((double)w, k[3]), z), k[1]);
                    f = isfinite(x) && z > 1e-8;
                    q[0] = __dsub_rn(x, rt[3]);
                    q[1] = __dsub_rn(y, rt[7]);
                    q[2] = __dsub_rn(z, rt[11]);
                }
            }
            int tot;
            const int p = block_scan(f, tot, scan_sh);
            if (f) {
                float *o = out + (m + p) * 3;
#pragma unroll
                for (int j = 0; j < 3; ++j)
                    o[j] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], rt[j]), __dmul_rn(q[1], rt[4 + j])),
                                                       __dmul_rn(q[2], rt[8 + j])));
            }
            m += tot;
        }
    }
    if (threadIdx.x == 0) a.n_points[obj] = (int32_t)m;
}

bool sizes_ok(int64_t B, int64_t H, int64_t W)
{
    return B >= 0 && B <= FFB6D_ORB_MAX_FRAMES && H >= FFB6D_ORB_MIN_SIDE && W >= FFB6D_ORB_MIN_SIDE &&
           H <= FFB6D_ORB_MAX_SIDE && W <= FFB6D_ORB_MAX_SIDE;
}

inline bool aligned(const void *p, size_t al) { return ((uintptr_t)p % al) == 0; }

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" int64_t ffb6d_orb_capacity(int64_t H, int64_t W)
{
    if (!sizes_ok(0, H, W)) return 0;
    return make_geom(H, W).cap_off[kLevels];
}

// workspace layout: [pyramids][raw FAST scores][candidate scores], each B frame bytes, frame bytes a multiple of 16
extern "C" size_t ffb6d_orb_workspace_bytes(int64_t B, int64_t H, int64_t W)
{
    if (!sizes_ok(B, H, W)) return 0;
    return 3 * (size_t)B * (size_t)make_geom(H, W).frame;
}

extern "C" int ffb6d_orb_detect(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, int32_t *count, float *pt,
                                int32_t *octave, float *response, int64_t cap, void *workspace,
                                size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(sizes_ok(B, H, W), "orb_detect: bad size (B=%lld H=%lld W=%lld)", (long long)B, (long long)H,
                    (long long)W);
    const Geom g = make_geom(H, W);
    FFB6D_CHECK_ARG(cap == g.cap_off[kLevels], "orb_detect: cap=%lld, ffb6d_orb_capacity gives %lld", (long long)cap,
                    (long long)g.cap_off[kLevels]);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(rgb && count && (cap == 0 || (pt && octave && response)), "orb_detect: null pointer");
    FFB6D_CHECK_ARG(aligned(count, 4) && aligned(pt, 4) && aligned(octave, 4) && aligned(response, 4) &&
                    aligned(workspace, 16), "orb_detect: misaligned pointer");
    const size_t need = ffb6d_orb_workspace_bytes(B, H, W);
    if (!workspace || workspace_bytes < need) {
        set_error("orb_detect: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }
    Args a;
    a.rgb = rgb;
    a.B = B;
    a.g = g;
    a.pyr = (uint8_t *)workspace;
    a.raw = a.pyr + (size_t)B * g.frame;
    a.score = a.raw + (size_t)B * g.frame;
    a.count = count;
    a.pt = pt;
    a.resp = response;
    a.oct = octave;
    a.cap = cap;
    cudaStream_t st = (cudaStream_t)stream;
    FFB6D_CUDA(cudaMemsetAsync(count, 0, (size_t)B * sizeof(int32_t), st));
    grey_kernel<<<dim3((unsigned)ceil_div((int64_t)g.h[0] * g.w[0], kThreads), (unsigned)B), kThreads, 0, st>>>(a);
    FFB6D_LAUNCH_OK("orb_grey_kernel");
    for (int l = 1; l < kLevels; ++l) {
        resize_kernel<<<dim3((unsigned)ceil_div((int64_t)g.h[l] * g.w[l], kThreads), (unsigned)B), kThreads, 0, st>>>(
            a, l);
        FFB6D_LAUNCH_OK("orb_resize_kernel");
    }
    for (int l = 0; l < kLevels; ++l) {
        fast_kernel<<<dim3((unsigned)ceil_div((int64_t)g.h[l] * g.w[l], kThreads), (unsigned)B), kThreads, 0, st>>>(
            a, l);
        FFB6D_LAUNCH_OK("orb_fast_kernel");
        nms_kernel<<<dim3((unsigned)ceil_div(g.w[l], kTX), (unsigned)ceil_div(g.h[l], kTY), (unsigned)B),
                     dim3(kTX, kTY), 0, st>>>(a, l);
        FFB6D_LAUNCH_OK("orb_nms_kernel");
    }
    for (int l = 0; l < kLevels; ++l) {
        select_kernel<<<(unsigned)B, kSelThreads, 0, st>>>(a, l);
        FFB6D_LAUNCH_OK("orb_select_kernel");
    }
    return FFB6D_OK;
}

extern "C" int ffb6d_orb_lift(const int32_t *count, const float *pt, int64_t cap, const float *depth, int64_t B,
                              int64_t H, int64_t W, const double *intrinsics, int intrinsics_per_frame,
                              const double *RTs, int64_t views, float *cloud, int32_t *n_points, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(sizes_ok(B, H, W), "orb_lift: bad size (B=%lld H=%lld W=%lld)", (long long)B, (long long)H,
                    (long long)W);
    FFB6D_CHECK_ARG(cap == ffb6d_orb_capacity(H, W), "orb_lift: cap=%lld, ffb6d_orb_capacity gives %lld",
                    (long long)cap, (long long)ffb6d_orb_capacity(H, W));
    FFB6D_CHECK_ARG(views >= 1 && B % views == 0 && B / views <= FFB6D_ORB_MAX_OBJECTS && views * cap < (1ll << 31),
                    "orb_lift: B=%lld frames must be n_obj <= %d objects of views=%lld, views cap < 2^31",
                    (long long)B, FFB6D_ORB_MAX_OBJECTS, (long long)views);
    FFB6D_CHECK_ARG(intrinsics_per_frame == 0 || intrinsics_per_frame == 1,
                    "orb_lift: intrinsics_per_frame must be 0 or 1");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(count && pt && depth && intrinsics && RTs && cloud && n_points, "orb_lift: null pointer");
    FFB6D_CHECK_ARG(aligned(count, 4) && aligned(pt, 4) && aligned(depth, 4) && aligned(intrinsics, 8) &&
                    aligned(RTs, 8) && aligned(cloud, 4) && aligned(n_points, 4), "orb_lift: misaligned pointer");
    LiftArgs a;
    a.count = count;
    a.pt = pt;
    a.cap = cap;
    a.depth = depth;
    a.H = (int)H;
    a.W = (int)W;
    a.intr = intrinsics;
    a.intr_per_frame = intrinsics_per_frame;
    a.RTs = RTs;
    a.views = views;
    a.cloud = cloud;
    a.n_points = n_points;
    lift_kernel<<<(unsigned)(B / views), kThreads, 0, (cudaStream_t)stream>>>(a);
    FFB6D_LAUNCH_OK("orb_lift_kernel");
    return FFB6D_OK;
}
