// vis.cu -- pose and label drawing: the reference's Basic_Utils.project_p3d / draw_p2ds (utils/basic_utils.py:268-295)
// over S point sets at once (ffb6d_project_p3d, ffb6d_draw_p2ds).
//
// Set s is rows start[s] .. start[s] + count[s] of a point table, optionally disabled by enable[s]; outputs are padded
// to [S, max_rows, ...].  A set whose rows leave the table, or with count > max_rows, is empty.
//
// Projection: one thread per (set, row).  Every step is an explicit _rn intrinsic in the order numpy's float64 code
// takes (the pose and intrinsics products as the fma chains of OpenBLAS's Haswell dgemm kernel), so nvcc cannot
// contract or reorder it; the float -> int32 cast is written out as x86's cvttsd2si (NaN, out of range -> INT32_MIN).
//
// Drawing: pass 1, one thread per (set, row), walks OpenCV's integer midpoint circle (cv2.circle, thickness -1,
// LINE_8, shift 0) and takes atomicMax of the key (s << 32 | row) + 1 at every covered pixel of its frame; pass 2,
// one thread per pixel, writes the colour of the winning key.  The largest key is the last draw in (set, row) order,
// so the image is the sequential loop's whatever the scheduling.
#include "common.cuh"

#include <cmath>

namespace ffb6d {
namespace {

constexpr int kThreads = 256;
constexpr int64_t kMaxBlocks = 1 << 16;

static_assert(FFB6D_VIS_MAX_SETS <= (1LL << 31) && FFB6D_VIS_MAX_ROWS <= (1LL << 31), "key layout");

__device__ __forceinline__ int32_t rint_to_i32(double q)
{
    // numpy's astype(np.int32) on x86 (cvttsd2si): NaN and anything outside [-2^31, 2^31) give INT32_MIN
    const double r = rint(q);   // round half to even, as np.around
    if (!(r >= -2147483648.0 && r < 2147483648.0)) return INT32_MIN;
    return (int32_t)r;
}

// The rows [lo, lo + n) of set s, or n = 0 for a disabled set or one whose rows leave the table or exceed max_rows
__device__ __forceinline__ int set_rows(const int32_t *start, const int32_t *count, const unsigned char *enable,
                                        int64_t n_rows, int64_t max_rows, int64_t s, int64_t &lo)
{
    if (enable && !enable[s]) return 0;
    const int64_t a = start[s], n = count[s];
    if (a < 0 || n < 0 || n > max_rows || a + n > n_rows) return 0;
    lo = a;
    return (int)n;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
project_kernel(const T *__restrict__ pts, int64_t n_rows, const int32_t *__restrict__ start,
               const int32_t *__restrict__ count, const unsigned char *__restrict__ enable, int64_t S, int64_t max_rows,
               const double *__restrict__ pose, const double *__restrict__ K, const double *__restrict__ cam_scale,
               int per_set, int2 *__restrict__ p2ds)
{
    const int64_t total = S * max_rows;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = i / max_rows, r = i - s * max_rows;
        int64_t lo = 0;
        const int n = set_rows(start, count, enable, n_rows, max_rows, s, lo);
        if (r >= n) {
            p2ds[i] = make_int2(INT32_MIN, INT32_MIN);
            continue;
        }
        const T *x = pts + (lo + r) * 3;
        const int64_t ps = per_set ? s : 0;
        const double cs = cam_scale[ps];
        double p[3];
        if (pose) {
            // np.dot(mesh, R.T) + t in float64, then p3d * cam_scale in float64
            const double *P = pose + s * 12;
            const double x0 = (double)x[0], x1 = (double)x[1], x2 = (double)x[2];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const double y = __dadd_rn(
                    __fma_rn(x2, P[j * 4 + 2], __fma_rn(x1, P[j * 4 + 1], __dmul_rn(x0, P[j * 4]))), P[j * 4 + 3]);
                p[j] = __dmul_rn(y, cs);
            }
        } else if (sizeof(T) == 4) {
            // float32 points times a Python float stay float32 (numpy's casting), then promote
            const float c = (float)cs;
#pragma unroll
            for (int j = 0; j < 3; ++j) p[j] = (double)__fmul_rn((float)x[j], c);
        } else {
#pragma unroll
            for (int j = 0; j < 3; ++j) p[j] = __dmul_rn((double)x[j], cs);
        }
        // np.dot(p3d, K.T)
        const double *k = K + ps * 9;
        double q[3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
            q[j] = __fma_rn(p[2], k[j * 3 + 2], __fma_rn(p[1], k[j * 3 + 1], __dmul_rn(p[0], k[j * 3])));
        if (q[2] < 1e-8) q[2] = 1.0;   // NaN compares false and stays
        p2ds[i] = make_int2(rint_to_i32(__ddiv_rn(q[0], q[2])), rint_to_i32(__ddiv_rn(q[1], q[2])));
    }
}

// atomicMax of key over the pixels x0 .. x1 (already clipped) of row y
__device__ __forceinline__ void mark_span(unsigned long long *frame_ws, int W, int y, int x0, int x1,
                                          unsigned long long key)
{
    unsigned long long *row = frame_ws + (int64_t)y * W;
    for (int x = x0; x <= x1; ++x) atomicMax(row + x, key);
}

__global__ void __launch_bounds__(kThreads)
draw_mark_kernel(int64_t B, int H, int W, const int2 *__restrict__ p2ds, int64_t S, int64_t max_rows,
                 const int32_t *__restrict__ frame, const int32_t *__restrict__ start,
                 const int32_t *__restrict__ count, const unsigned char *__restrict__ enable, int64_t n_rows,
                 const int32_t *__restrict__ radius, unsigned long long *__restrict__ ws)
{
    const int64_t total = S * max_rows;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = i / max_rows, r = i - s * max_rows;
        int64_t lo = 0;
        const int n = set_rows(start, count, enable, n_rows, max_rows, s, lo);
        const int64_t b = frame[s];
        const int rad = radius[s];
        if (r >= n || b < 0 || b >= B || rad < 0 || rad > FFB6D_VIS_MAX_RADIUS) continue;
        const int2 pt = p2ds[i];
        // np.clip(pt, 0, w) / (0, h): the bounds are inclusive, so a centre on x = W still draws its left part
        const int cx = min(max(pt.x, 0), W), cy = min(max(pt.y, 0), H);
        const unsigned long long key = (((unsigned long long)s << 32) | (unsigned long long)r) + 1ull;
        unsigned long long *fw = ws + b * H * (int64_t)W;
        // OpenCV's Circle() (imgproc/src/drawing.cpp) with fill: each step of the midpoint walk fills the spans
        // rows cy -+ dy over [cx - dx, cx + dx] and rows cy -+ dx over [cx - dy, cx + dy], clipped to the image
        int err = 0, dx = rad, dy = 0, plus = 1, minus = (rad << 1) - 1;
        while (dx >= dy) {
            const int xa0 = max(cx - dx, 0), xa1 = min(cx + dx, W - 1);
            if (xa0 <= xa1) {
                if (cy - dy >= 0 && cy - dy < H) mark_span(fw, W, cy - dy, xa0, xa1, key);
                if (dy != 0 && cy + dy < H) mark_span(fw, W, cy + dy, xa0, xa1, key);
            }
            const int xb0 = max(cx - dy, 0), xb1 = min(cx + dy, W - 1);
            if (xb0 <= xb1 && dx != dy) {   // dx == dy: the same rows and spans as above
                if (cy - dx >= 0 && cy - dx < H) mark_span(fw, W, cy - dx, xb0, xb1, key);
                if (cy + dx < H) mark_span(fw, W, cy + dx, xb0, xb1, key);
            }
            dy++;
            err += plus;
            plus += 2;
            const int mask = (err <= 0) - 1;
            err -= minus & mask;
            dx += mask;
            minus -= mask & 2;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
draw_paint_kernel(unsigned char *__restrict__ img, int64_t n_px, const unsigned long long *__restrict__ ws,
                  int64_t max_rows, const unsigned char *__restrict__ colors, int color_per_row)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_px; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long key = ws[i];
        if (!key) continue;
        const int64_t s = (int64_t)((key - 1ull) >> 32), r = (int64_t)((key - 1ull) & 0xffffffffull);
        const unsigned char *c = colors + (color_per_row ? s * max_rows + r : s) * 3;
        unsigned char *o = img + i * 3;
        o[0] = c[0];
        o[1] = c[1];
        o[2] = c[2];
    }
}

unsigned grid_for(int64_t n) { return (unsigned)std::min<int64_t>(std::max<int64_t>(ceil_div(n, kThreads), 1), kMaxBlocks); }

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_project_p3d(const void *pts, int pts_f64, int64_t n_rows, const int32_t *start,
                                 const int32_t *count, const unsigned char *enable, int64_t S, int64_t max_rows,
                                 const double *pose, const double *K, const double *cam_scale, int per_set,
                                 int32_t *p2ds, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(S >= 0 && S <= FFB6D_VIS_MAX_SETS, "project_p3d: need 0 <= S <= %d, got %lld", FFB6D_VIS_MAX_SETS,
                    (long long)S);
    FFB6D_CHECK_ARG(max_rows >= 1 && max_rows <= FFB6D_VIS_MAX_ROWS, "project_p3d: need 1 <= max_rows <= %d, got %lld",
                    FFB6D_VIS_MAX_ROWS, (long long)max_rows);
    FFB6D_CHECK_ARG(n_rows >= 0 && n_rows <= FFB6D_VIS_MAX_TABLE_ROWS,
                    "project_p3d: need 0 <= n_rows <= %d, got %lld", FFB6D_VIS_MAX_TABLE_ROWS, (long long)n_rows);
    FFB6D_CHECK_ARG(pts_f64 == 0 || pts_f64 == 1, "project_p3d: pts_f64 must be 0 or 1, got %d", pts_f64);
    FFB6D_CHECK_ARG(per_set == 0 || per_set == 1, "project_p3d: per_set must be 0 or 1, got %d", per_set);
    if (S == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG((pts || n_rows == 0) && start && count && K && cam_scale && p2ds, "project_p3d: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)start | (uintptr_t)count) % 4 == 0 && (uintptr_t)pts % (pts_f64 ? 8 : 4) == 0 &&
                        ((uintptr_t)pose | (uintptr_t)K | (uintptr_t)cam_scale | (uintptr_t)p2ds) % 8 == 0,
                    "project_p3d: pointers must be aligned to their element (p2ds to 8 bytes)");
    const cudaStream_t st = (cudaStream_t)stream;
    const int64_t total = S * max_rows;
    if (pts_f64)
        project_kernel<double><<<grid_for(total), kThreads, 0, st>>>((const double *)pts, n_rows, start, count, enable,
                                                                     S, max_rows, pose, K, cam_scale, per_set,
                                                                     (int2 *)p2ds);
    else
        project_kernel<float><<<grid_for(total), kThreads, 0, st>>>((const float *)pts, n_rows, start, count, enable,
                                                                    S, max_rows, pose, K, cam_scale, per_set,
                                                                    (int2 *)p2ds);
    FFB6D_LAUNCH_OK("project_kernel");
    return FFB6D_OK;
}

extern "C" size_t ffb6d_draw_p2ds_workspace_bytes(int64_t B, int64_t H, int64_t W)
{
    if (B < 0 || B > FFB6D_VIS_MAX_FRAMES || H < 1 || H > FFB6D_VIS_MAX_SIDE || W < 1 || W > FFB6D_VIS_MAX_SIDE)
        return 0;
    return (size_t)B * (size_t)H * (size_t)W * sizeof(unsigned long long);
}

extern "C" int ffb6d_draw_p2ds(unsigned char *img, int64_t B, int64_t H, int64_t W, const int32_t *p2ds, int64_t S,
                               int64_t max_rows, const int32_t *frame, const int32_t *start, const int32_t *count,
                               const unsigned char *enable, int64_t n_rows, const int32_t *radius,
                               const unsigned char *colors, int color_per_row, void *workspace, size_t workspace_bytes,
                               ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && B <= FFB6D_VIS_MAX_FRAMES, "draw_p2ds: need 0 <= B <= %d, got %lld", FFB6D_VIS_MAX_FRAMES,
                    (long long)B);
    FFB6D_CHECK_ARG(H >= 1 && H <= FFB6D_VIS_MAX_SIDE && W >= 1 && W <= FFB6D_VIS_MAX_SIDE,
                    "draw_p2ds: need 1 <= H, W <= %d, got %lld x %lld", FFB6D_VIS_MAX_SIDE, (long long)H,
                    (long long)W);
    FFB6D_CHECK_ARG(S >= 0 && S <= FFB6D_VIS_MAX_SETS, "draw_p2ds: need 0 <= S <= %d, got %lld", FFB6D_VIS_MAX_SETS,
                    (long long)S);
    FFB6D_CHECK_ARG(max_rows >= 1 && max_rows <= FFB6D_VIS_MAX_ROWS, "draw_p2ds: need 1 <= max_rows <= %d, got %lld",
                    FFB6D_VIS_MAX_ROWS, (long long)max_rows);
    FFB6D_CHECK_ARG(n_rows >= 0 && n_rows <= FFB6D_VIS_MAX_TABLE_ROWS, "draw_p2ds: need 0 <= n_rows <= %d, got %lld",
                    FFB6D_VIS_MAX_TABLE_ROWS, (long long)n_rows);
    FFB6D_CHECK_ARG(color_per_row == 0 || color_per_row == 1, "draw_p2ds: color_per_row must be 0 or 1, got %d",
                    color_per_row);
    if (B == 0 || S == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(img && p2ds && frame && start && count && radius && colors, "draw_p2ds: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)frame | (uintptr_t)start | (uintptr_t)count | (uintptr_t)radius) % 4 == 0 &&
                        (uintptr_t)p2ds % 8 == 0,
                    "draw_p2ds: pointers must be aligned to their element (p2ds to 8 bytes)");
    FFB6D_CHECK_ARG((uintptr_t)workspace % 8 == 0, "draw_p2ds: workspace must be 8-byte aligned");
    const size_t need = ffb6d_draw_p2ds_workspace_bytes(B, H, W);
    if (!workspace || workspace_bytes < need) {
        set_error("draw_p2ds: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned long long *ws = (unsigned long long *)workspace;
    FFB6D_CUDA(cudaMemsetAsync(ws, 0, need, st));
    draw_mark_kernel<<<grid_for(S * max_rows), kThreads, 0, st>>>(B, (int)H, (int)W, (const int2 *)p2ds, S, max_rows,
                                                                  frame, start, count, enable, n_rows, radius, ws);
    FFB6D_LAUNCH_OK("draw_mark_kernel");
    const int64_t n_px = B * H * W;
    draw_paint_kernel<<<grid_for(n_px), kThreads, 0, st>>>(img, n_px, ws, max_rows, colors, color_per_row);
    FFB6D_LAUNCH_OK("draw_paint_kernel");
    return FFB6D_OK;
}
