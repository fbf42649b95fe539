// pose_eval.cu -- ADD and ADD-S of a batch of predicted poses (ffb6d_pose_add_adds): the reference's
// Basic_Utils.cal_add_cuda / cal_adds_cuda (utils/basic_utils.py:651-669) for every object of a test batch at once.
//
// Grid (gt-point tiles, objects).  Each of the 256 threads owns two gt points x_i, transformed by G in registers.  The
// CTA streams the whole mesh, transformed by P, through shared memory in tiles of float4; every warp reads each tile
// element as a broadcast and keeps, per gt point, the NaN-propagating min of |P x_j - G x_i|^2.  ADD's term for x_i is
// |P x_i - G x_i| from the same transform.  Each CTA sums its 512 square roots in fp64 in a fixed order and stores
// them in the workspace; a second kernel adds an object's tiles in tile order, divides once and rounds once.  The
// all-pairs matrices of the reference never exist; HBM sees the mesh once per CTA (L2-resident) and 16 bytes per CTA.
#include "common.cuh"

#include <cmath>

namespace ffb6d {
namespace {

constexpr int kThreads = 256;
constexpr int kGtPerThread = 2;
constexpr int kGtPerCta = kThreads * kGtPerThread;   // 512 gt points per CTA
constexpr int kTile = 512;                           // pred points per shared-memory tile
constexpr int kUnroll = 8;                           // a tile's scanned length is a multiple of this

static_assert(FFB6D_POSE_EVAL_GT_TILE == kGtPerCta && FFB6D_POSE_EVAL_PRED_TILE == kTile, "header tile sizes");

__device__ __forceinline__ float min_nan(float a, float b)
{
    float r;   // FMNMX.NAN: torch.min propagates NaN, fminf drops it
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// R x + t with one fixed instruction sequence (intrinsics are never contracted or reordered), so equal poses give
// equal points bit for bit
__device__ __forceinline__ float3 xform(const float *T, float x, float y, float z)
{
    float3 r;
    r.x = __fadd_rn(__fmaf_rn(T[0], x, __fmaf_rn(T[1], y, __fmul_rn(T[2], z))), T[3]);
    r.y = __fadd_rn(__fmaf_rn(T[4], x, __fmaf_rn(T[5], y, __fmul_rn(T[6], z))), T[7]);
    r.z = __fadd_rn(__fmaf_rn(T[8], x, __fmaf_rn(T[9], y, __fmul_rn(T[10], z))), T[11]);
    return r;
}

__device__ __forceinline__ float sqdist(float ax, float ay, float az, float bx, float by, float bz)
{
    const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
    return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// The points [lo, lo + n) of object m's mesh, or n = 0 when its class id, its offsets or its length is out of range
__device__ __forceinline__ int mesh_range(const int *obj_mesh, const int *mesh_off, int n_meshes, int max_points,
                                          int m, int &lo)
{
    const int c = obj_mesh[m];
    if (c < 0 || c >= n_meshes) return 0;
    lo = mesh_off[c];
    const int hi = mesh_off[c + 1];
    if (lo < 0 || hi < lo || hi - lo > max_points) return 0;
    return hi - lo;
}

__global__ void __launch_bounds__(kThreads)
add_adds_tiles_kernel(const float *__restrict__ pts, const int *__restrict__ mesh_off, int n_meshes, int max_points,
                      const int *__restrict__ obj_mesh, const float *__restrict__ pred_RT,
                      const float *__restrict__ gt_RT, int n_tiles, double2 *__restrict__ part)
{
    __shared__ float4 tile[kTile];
    __shared__ float T[24];                  // pred [3,4], gt [3,4]
    __shared__ double red[kThreads / 32][2];

    const int m = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int lo = 0;
    const int n = mesh_range(obj_mesh, mesh_off, n_meshes, max_points, m, lo);
    const int g0 = blockIdx.x * kGtPerCta;
    if (g0 >= n) return;                     // n = 0 (a NaN row) or a tile past this mesh: the finalize reads neither

    float v = 0.f;
    if (tid < 12) v = pred_RT[(size_t)m * 12 + tid];
    else if (tid < 24) v = gt_RT[(size_t)m * 12 + tid - 12];
    if (tid < 24) T[tid] = v;
    const bool bad_pose = __syncthreads_or(tid < 24 && !isfinite(v));
    const float *P = T, *G = T + 12;
    const float *mp = pts + (size_t)lo * 3;

    double s_add = 0.0, s_adds = 0.0;
    if (bad_pose) {
        s_add = s_adds = (double)NAN;
    } else {
        float gx[kGtPerThread], gy[kGtPerThread], gz[kGtPerThread], best[kGtPerThread];
        bool own[kGtPerThread], fin[kGtPerThread];
#pragma unroll
        for (int k = 0; k < kGtPerThread; ++k) {
            const int i = g0 + tid + k * kThreads;
            own[k] = i < n;
            float x = 0.f, y = 0.f, z = 0.f;
            if (own[k]) { x = mp[(size_t)i * 3]; y = mp[(size_t)i * 3 + 1]; z = mp[(size_t)i * 3 + 2]; }
            const float3 g = xform(G, x, y, z);
            gx[k] = g.x; gy[k] = g.y; gz[k] = g.z;
            best[k] = INFINITY;
            fin[k] = finite3(x, y, z);               // a non-finite point makes its object's row NaN
            if (own[k]) {
                const float3 p = xform(P, x, y, z);     // the diagonal term: ADD
                s_add += fin[k] ? (double)sqrtf(sqdist(p.x, p.y, p.z, g.x, g.y, g.z)) : (double)NAN;
            }
        }
        for (int base = 0; base < n; base += kTile) {
            const int len = min(kTile, n - base);
            const int len_u = (len + kUnroll - 1) / kUnroll * kUnroll;
            __syncthreads();                 // the previous tile has been read
            for (int j = tid; j < len_u; j += kThreads) {
                float4 q = make_float4(INFINITY, INFINITY, INFINITY, 0.f);   // padding: never the min of a finite row
                if (j < len) {
                    const float *s = mp + (size_t)(base + j) * 3;
                    const float3 p = xform(P, s[0], s[1], s[2]);
                    q = make_float4(p.x, p.y, p.z, 0.f);
                }
                tile[j] = q;
            }
            __syncthreads();
            for (int j = 0; j < len_u; j += kUnroll) {
#pragma unroll
                for (int u = 0; u < kUnroll; ++u) {
                    const float4 q = tile[j + u];
#pragma unroll
                    for (int k = 0; k < kGtPerThread; ++k)
                        best[k] = min_nan(best[k], sqdist(q.x, q.y, q.z, gx[k], gy[k], gz[k]));
                }
            }
        }
#pragma unroll
        for (int k = 0; k < kGtPerThread; ++k)
            if (own[k]) s_adds += fin[k] ? (double)sqrtf(best[k]) : (double)NAN;
    }

#pragma unroll
    for (int o = 16; o; o >>= 1) {
        s_add += __shfl_down_sync(0xffffffffu, s_add, o);
        s_adds += __shfl_down_sync(0xffffffffu, s_adds, o);
    }
    if (lane == 0) { red[warp][0] = s_add; red[warp][1] = s_adds; }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) { a += red[w][0]; b += red[w][1]; }
        part[(size_t)m * n_tiles + blockIdx.x] = make_double2(a, b);
    }
}

__global__ void add_adds_finalize_kernel(const int *__restrict__ mesh_off, int n_meshes, int max_points,
                                         const int *__restrict__ obj_mesh, int M, int n_tiles,
                                         const double2 *__restrict__ part, float *__restrict__ add,
                                         float *__restrict__ adds)
{
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    int lo = 0;
    const int n = mesh_range(obj_mesh, mesh_off, n_meshes, max_points, m, lo);
    if (n == 0) {
        add[m] = adds[m] = NAN;
        return;
    }
    double a = 0.0, b = 0.0;
    const int used = (n + kGtPerCta - 1) / kGtPerCta;
    for (int t = 0; t < used; ++t) {
        const double2 p = part[(size_t)m * n_tiles + t];
        a += p.x;
        b += p.y;
    }
    add[m] = (float)(a / n);
    adds[m] = (float)(b / n);
}

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" size_t ffb6d_pose_add_adds_workspace_bytes(int64_t M, int64_t max_points)
{
    if (M < 0 || max_points < 1 || M > FFB6D_POSE_EVAL_MAX_OBJECTS || max_points > FFB6D_POSE_EVAL_MAX_POINTS)
        return 0;
    return (size_t)M * (size_t)ceil_div(max_points, kGtPerCta) * sizeof(double2);
}

extern "C" int ffb6d_pose_add_adds(const float *mesh_pts, const int32_t *mesh_off, int64_t n_meshes,
                                   int64_t max_points, const int32_t *obj_mesh, const float *pred_RT,
                                   const float *gt_RT, int64_t M, float *add, float *adds, void *workspace,
                                   size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(M >= 0 && M <= FFB6D_POSE_EVAL_MAX_OBJECTS, "pose_add_adds: need 0 <= M <= %d, got %lld",
                    FFB6D_POSE_EVAL_MAX_OBJECTS, (long long)M);
    FFB6D_CHECK_ARG(max_points >= 1 && max_points <= FFB6D_POSE_EVAL_MAX_POINTS,
                    "pose_add_adds: need 1 <= max_points <= %d, got %lld", FFB6D_POSE_EVAL_MAX_POINTS,
                    (long long)max_points);
    FFB6D_CHECK_ARG(n_meshes >= 0 && n_meshes <= FFB6D_POSE_EVAL_MAX_MESHES,
                    "pose_add_adds: need 0 <= n_meshes <= %d, got %lld", FFB6D_POSE_EVAL_MAX_MESHES,
                    (long long)n_meshes);
    if (M == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(n_meshes >= 1, "pose_add_adds: n_meshes is 0 but M = %lld objects are scored", (long long)M);
    FFB6D_CHECK_ARG(mesh_pts && mesh_off && obj_mesh && pred_RT && gt_RT && add && adds, "pose_add_adds: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)mesh_pts | (uintptr_t)mesh_off | (uintptr_t)obj_mesh | (uintptr_t)pred_RT |
                     (uintptr_t)gt_RT | (uintptr_t)add | (uintptr_t)adds) % 4 == 0,
                    "pose_add_adds: pointers must be 4-byte aligned");
    FFB6D_CHECK_ARG((uintptr_t)workspace % 16 == 0, "pose_add_adds: workspace must be 16-byte aligned");
    const size_t need = ffb6d_pose_add_adds_workspace_bytes(M, max_points);
    if (!workspace || workspace_bytes < need) {
        set_error("pose_add_adds: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }

    const int n_tiles = (int)ceil_div(max_points, kGtPerCta);
    const cudaStream_t st = (cudaStream_t)stream;
    double2 *part = (double2 *)workspace;
    add_adds_tiles_kernel<<<dim3((unsigned)n_tiles, (unsigned)M), kThreads, 0, st>>>(
        mesh_pts, mesh_off, (int)n_meshes, (int)max_points, obj_mesh, pred_RT, gt_RT, n_tiles, part);
    FFB6D_LAUNCH_OK("add_adds_tiles_kernel");
    add_adds_finalize_kernel<<<(unsigned)ceil_div(M, 128), 128, 0, st>>>(mesh_off, (int)n_meshes, (int)max_points,
                                                                         obj_mesh, (int)M, n_tiles, part, add, adds);
    FFB6D_LAUNCH_OK("add_adds_finalize_kernel");
    return FFB6D_OK;
}
