// normal.cu -- surface normals from a millimetre depth map on the device (sm_90a), DESIGN.md §4.30.
//
// ffb6d_depth_normal is the least-squares depth-gradient fit of OpenCV's LINEMOD (`accumBilateral`) with the camera's
// fx, fy in place of its fixed focal length and no quantisation.  For pixel (y, x) with d = D[y,x]:
//   d == 0 or d >= distance_threshold                          -> (0, 0, 0)
//   over the 8 offsets (dx, dy) in {-r, 0, r}^2 \ {(0,0)} inside the image, delta = D[y+dy,x+dx] - d, and where
//   |delta| < difference_threshold:  A0 += dx dx, A1 += dx dy, A2 += dy dy, b0 += dx delta, b1 += dy delta
//   det = A0 A2 - A1^2, ddx = A2 b0 - A1 b1, ddy = A0 b1 - A1 b0 (exact integers); det == 0 -> (0, 0, 0)
//   n = (fx ddx, fy ddy, -(det d)) in float64, divided by sqrt((nx nx + ny ny) + nz nz), each rounded once to float32;
//   negated with point_into_surface.
// The sums stay in int32 (|b| <= 6 r 65535 < 2^31 for r <= FFB6D_NRM_MAX_KSIZE), which equals the int64 of the
// specification; the products are int64 and every float64 operation is a separately rounded _rn intrinsic, so the map is
// bitwise oracle/normal_oracle.py's.
//
// Layout: one thread per output pixel, a TX x TY tile per CTA.  The tile and an r-pixel halo of depth are loaded into
// shared memory by consecutive threads along rows (coalesced 2-byte loads).  Each warp is one tile row: its 32 pixels'
// 96 floats go through a shared-memory row and out as three coalesced 128-byte stores, not as stride-3 stores.
//
// ffb6d_depth_to_mm is the YCB dataset's millimetre map of the completed depth, `(dpt_um / 10).astype(np.uint16)`: a
// float32 IEEE division and a truncation.
#include "common.cuh"

namespace ffb6d {
namespace {

constexpr int TX = 32, TY = 8;

__global__ void __launch_bounds__(TX * TY)
depth_normal_kernel(const uint16_t *__restrict__ depth, int H, int W, const double *__restrict__ intr, int intr_per_frame,
                    int r, int dist_thr, int diff_thr, int into, float *__restrict__ nrm)
{
    extern __shared__ uint16_t tile[];              // (TY + 2r) x (TX + 2r) depth, halo included
    __shared__ float stage[TY][3 * TX];
    const int b = blockIdx.z, tx = threadIdx.x, ty = threadIdx.y;
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    const int SW = TX + 2 * r, SH = TY + 2 * r;
    const uint16_t *f = depth + (size_t)b * H * W;

    for (int i = ty * TX + tx; i < SW * SH; i += TX * TY) {
        const int yy = y0 - r + i / SW, xx = x0 - r + i % SW;
        tile[i] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(f + (size_t)yy * W + xx) : (uint16_t)0;
    }
    __syncthreads();

    const int y = y0 + ty, x = x0 + tx;
    float o[3] = {0.0f, 0.0f, 0.0f};
    if (y < H && x < W) {
        const int d = tile[(ty + r) * SW + tx + r];
        if (d != 0 && d < dist_thr) {
            int A0 = 0, A1 = 0, A2 = 0, b0 = 0, b1 = 0;
#pragma unroll
            for (int j = -1; j <= 1; ++j) {
#pragma unroll
                for (int i = -1; i <= 1; ++i) {
                    if (i == 0 && j == 0) continue;
                    const int dx = i * r, dy = j * r;
                    if (y + dy < 0 || y + dy >= H || x + dx < 0 || x + dx >= W) continue;
                    const int delta = (int)tile[(ty + r + dy) * SW + tx + r + dx] - d;
                    if (abs(delta) < diff_thr) {
                        A0 += dx * dx;
                        A1 += dx * dy;
                        A2 += dy * dy;
                        b0 += dx * delta;
                        b1 += dy * delta;
                    }
                }
            }
            const long long det = (long long)A0 * A2 - (long long)A1 * A1;
            if (det != 0) {
                const long long ddx = (long long)A2 * b0 - (long long)A1 * b1;
                const long long ddy = (long long)A0 * b1 - (long long)A1 * b0;
                const double *k = intr + (intr_per_frame ? (size_t)b * 4 : 0);
                const double nx = __dmul_rn(__ldg(k), (double)ddx), ny = __dmul_rn(__ldg(k + 1), (double)ddy);
                const double nz = -(double)(det * d);
                const double s = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
                o[0] = __double2float_rn(__ddiv_rn(nx, s));
                o[1] = __double2float_rn(__ddiv_rn(ny, s));
                o[2] = __double2float_rn(__ddiv_rn(nz, s));
                if (into) {
                    o[0] = -o[0];
                    o[1] = -o[1];
                    o[2] = -o[2];
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) stage[ty][3 * tx + c] = o[c];      // stride 3: no bank conflicts
    __syncwarp();
    if (y >= H) return;
    const int n = 3 * min(TX, W - x0);
    float *row = nrm + ((size_t)b * H * W + (size_t)y * W + x0) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int i = c * TX + tx;
        if (i < n) row[i] = stage[ty][i];
    }
}

__global__ void __launch_bounds__(256)
depth_to_mm_kernel(const float *__restrict__ src, int64_t n, float divisor, uint16_t *__restrict__ dst)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float q = __fdiv_rn(__ldg(src + i), divisor);
        // truncation toward zero (numpy's cast); outside [0, 65535] and NaN, where numpy's cast is undefined, saturate
        dst[i] = (uint16_t)min(__float2uint_rz(q), 65535u);
    }
}

static inline bool aligned(const void *p, size_t a) { return ((uintptr_t)p % a) == 0; }

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_depth_normal(const uint16_t *depth_mm, int64_t B, int64_t H, int64_t W, const double *intrinsics,
                                  int intrinsics_per_frame, int k_size, int distance_threshold,
                                  int difference_threshold, int point_into_surface, float *nrm, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && B <= FFB6D_NRM_MAX_FRAMES && H >= 1 && H <= FFB6D_NRM_MAX_HEIGHT && W >= 1 &&
                    H * W <= FFB6D_NRM_MAX_FRAME_PIXELS, "depth_normal: bad size (B=%lld H=%lld W=%lld)", (long long)B,
                    (long long)H, (long long)W);
    FFB6D_CHECK_ARG(k_size >= 1 && k_size <= FFB6D_NRM_MAX_KSIZE, "depth_normal: k_size=%d outside [1, %d]", k_size,
                    FFB6D_NRM_MAX_KSIZE);
    FFB6D_CHECK_ARG(distance_threshold >= 1 && distance_threshold <= 65536,
                    "depth_normal: distance_threshold=%d outside [1, 65536]", distance_threshold);
    FFB6D_CHECK_ARG(difference_threshold >= 1 && difference_threshold <= 65535,
                    "depth_normal: difference_threshold=%d outside [1, 65535]", difference_threshold);
    FFB6D_CHECK_ARG(intrinsics_per_frame == 0 || intrinsics_per_frame == 1,
                    "depth_normal: intrinsics_per_frame must be 0 or 1");
    FFB6D_CHECK_ARG(point_into_surface == 0 || point_into_surface == 1,
                    "depth_normal: point_into_surface must be 0 or 1");
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(depth_mm && intrinsics && nrm, "depth_normal: null pointer");
    FFB6D_CHECK_ARG(aligned(depth_mm, 2) && aligned(intrinsics, 8) && aligned(nrm, 4), "depth_normal: misaligned pointer");
    const size_t smem = (size_t)(TX + 2 * k_size) * (TY + 2 * k_size) * sizeof(uint16_t);
    const dim3 grid((unsigned)ceil_div(W, TX), (unsigned)ceil_div(H, TY), (unsigned)B);
    depth_normal_kernel<<<grid, dim3(TX, TY), smem, (cudaStream_t)stream>>>(
        depth_mm, (int)H, (int)W, intrinsics, intrinsics_per_frame, k_size, distance_threshold, difference_threshold,
        point_into_surface, nrm);
    FFB6D_LAUNCH_OK("depth_normal_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_depth_to_mm(const float *depth, int64_t n, float divisor, uint16_t *depth_mm,
                                 ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(n >= 0 && n <= FFB6D_NRM_MAX_FRAMES * (int64_t)FFB6D_NRM_MAX_FRAME_PIXELS,
                    "depth_to_mm: bad size n=%lld", (long long)n);
    FFB6D_CHECK_ARG(divisor > 0.0f && divisor < INFINITY, "depth_to_mm: divisor must be positive and finite, got %g",
                    (double)divisor);
    if (n == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(depth && depth_mm, "depth_to_mm: null pointer");
    FFB6D_CHECK_ARG(aligned(depth, 4) && aligned(depth_mm, 2), "depth_to_mm: misaligned pointer");
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(n, 256), 1 << 20);
    depth_to_mm_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(depth, n, divisor, depth_mm);
    FFB6D_LAUNCH_OK("depth_to_mm_kernel");
    return FFB6D_OK;
}
