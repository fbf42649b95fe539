// pose_eval.cu -- ADD and ADD-S of a batch of predicted poses (ffb6d_pose_add_adds): the reference's
// Basic_Utils.cal_add_cuda / cal_adds_cuda (utils/basic_utils.py:651-669) for every object of a test batch at once.
//
// Grid (gt-point tiles, objects).  Each of the 256 threads owns two gt points x_i, transformed by G in registers.  The
// CTA streams the whole mesh, transformed by P, through shared memory in tiles of float4; every warp reads each tile
// element as a broadcast and keeps, per gt point, the NaN-propagating min of |P x_j - G x_i|^2.  ADD's term for x_i is
// |P x_i - G x_i| from the same transform.  Each CTA sums its 512 square roots in fp64 in a fixed order and stores
// them in the workspace; a second kernel adds an object's tiles in tile order, divides once and rounds once.  The
// all-pairs matrices of the reference never exist; HBM sees the mesh once per CTA (L2-resident) and 16 bytes per CTA.
//
// The test run's record and summary (ffb6d_eval_record, ffb6d_eval_auc; DESIGN.md §4.29): the reference's TorchEval
// lists (utils/pvn3d_eval_utils_kpls.py:326-505) as a device table of fixed-slot rows, and its cal_auc / cal_lm_add
// (utils/basic_utils.py:642-649) over that table, with CUB's radix sort and fixed-order fp64 sums.
#include "common.cuh"

#include <cmath>
#include <cub/cub.cuh>

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

// ------------------------------------------------------------------------------------------------ the test record
namespace ffb6d {
namespace {

constexpr int kRecThreads = 256;
constexpr int kAucThreads = 256;
constexpr int kW = FFB6D_EVAL_ROW_WORDS;
static_assert(kW == 20, "row layout");

// One CTA: the state is read, the batch placed and the state advanced by the same block, so no other block races it.
__global__ void __launch_bounds__(kRecThreads)
eval_record_kernel(const int32_t *__restrict__ cls_ids, const uint8_t *__restrict__ valid,
                   const uint8_t *__restrict__ present, const float *__restrict__ kps,
                   const double *__restrict__ poses, const float *__restrict__ gt_kps,
                   const float *__restrict__ pred_RT, const float *__restrict__ add, const float *__restrict__ adds,
                   int B, int n_obj, int n_cls, int R, int n_kps, int obj_id, int32_t *__restrict__ rows,
                   long long capacity, long long *__restrict__ state, double *__restrict__ frame_poses,
                   uint8_t *__restrict__ frame_flags, long long frame_capacity)
{
    __shared__ long long base_s, fbase_s;
    __shared__ int ok_s;
    const int tid = threadIdx.x;
    const long long n_rows = (long long)B * n_obj;
    if (tid == 0) {
        const long long base = state[0], fbase = state[1];
        const bool fits = base >= 0 && base <= capacity && n_rows <= capacity - base &&
                          (!frame_flags || (fbase >= 0 && fbase <= frame_capacity && B <= frame_capacity - fbase));
        if (!fits) state[2] = 1;      // the table is left as it is
        base_s = base;
        fbase_s = fbase;
        ok_s = fits;
    }
    __syncthreads();
    if (!ok_s) return;
    const long long base = base_s, fbase = fbase_s;

    for (long long r = tid; r < n_rows; r += kRecThreads) {
        const int b = (int)(r / n_obj), j = (int)(r % n_obj);
        const bool frame_ok = !valid || valid[b];
        int cls = -1;
        if (frame_ok) {
            if (obj_id > 0) {
                cls = j == 0 ? obj_id : -1;               // LineMOD: slot 0 is the object
            } else {
                cls = cls_ids[r];
                for (int q = 0; q < j && cls != -1; ++q)      // YCB: slots from the first zero id on are skipped
                    if (cls_ids[(long long)b * n_obj + q] == 0) cls = -1;
                if (cls == 0) cls = -1;
            }
        }
        int32_t w[kW];
#pragma unroll
        for (int k = 0; k < kW; ++k) w[k] = 0;
        w[0] = cls;
        w[1] = (int32_t)(fbase + b);
        if (cls != -1) {
            const long long s = obj_id > 0 ? b : r;      // the scored object: [B] (LineMOD) or [B, n_obj] (YCB)
            const int pc = obj_id > 0 ? 1 : cls;          // its row of the vote
            const bool pres = pc >= 0 && pc < n_cls && present[(long long)b * n_cls + pc];
            float err = 0.f;
            if (obj_id == 0) {
                // mean_k |gt_kp - pred_kp| in f32, pred_kp = 0 for a class that was not predicted; the vote's kps
                // row holds the centre last, which the reference drops
                const float *g = gt_kps + r * n_kps * 3;
                const float *p = pres ? kps + ((long long)b * n_cls + pc) * R * 3 : nullptr;
                float sum = 0.f;
                for (int k = 0; k < n_kps; ++k) {
                    const float dx = __fsub_rn(g[3 * k], p ? p[3 * k] : 0.f);
                    const float dy = __fsub_rn(g[3 * k + 1], p ? p[3 * k + 1] : 0.f);
                    const float dz = __fsub_rn(g[3 * k + 2], p ? p[3 * k + 2] : 0.f);
                    const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)),
                                                         __fmul_rn(dz, dz)));
                    sum = k == 0 ? n : __fadd_rn(sum, n);
                }
                err = __fdiv_rn(sum, (float)n_kps);
            }
            w[2] = pres;
            w[3] = __float_as_int(add[s]);
            w[4] = __float_as_int(adds[s]);
            w[5] = __float_as_int(err);
#pragma unroll
            for (int k = 0; k < 12; ++k) w[6 + k] = __float_as_int(pred_RT[s * 12 + k]);
        }
        int32_t *o = rows + (base + r) * kW;
#pragma unroll
        for (int k = 0; k < kW; ++k) o[k] = w[k];
    }
    if (frame_flags) {
        const long long n_f = (long long)B * n_cls;
        for (long long e = tid; e < n_f; e += kRecThreads) {
            const int b = (int)(e / n_cls);
            const bool frame_ok = !valid || valid[b];
            frame_flags[fbase * n_cls + e] = (uint8_t)((present[e] ? 1 : 0) | (frame_ok ? 2 : 0));
        }
        for (long long e = tid; e < n_f * 12; e += kRecThreads) frame_poses[fbase * n_cls * 12 + e] = poses[e];
    }
    __syncthreads();
    if (tid == 0) {
        state[0] = base + n_rows;
        state[1] = fbase + B;
    }
}

__device__ __forceinline__ float row_f(const int32_t *row, int k) { return __int_as_float(row[k]); }

__device__ __forceinline__ unsigned int order_bits(float v)
{
    const unsigned int u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float unorder_bits(unsigned int k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Per row, six keys (ADD, ADD-S, ADD(-S)) x (its class, class 0): segment m * n_cls + c in the high word, the
// distance's order bits in the low word.  Distances > 0.1 (misses) and NaN sort past every segment as padding;
// the segment counters are integer atomics, so the counts do not depend on the order.
__global__ void eval_auc_keys_kernel(const int32_t *__restrict__ rows, const long long *__restrict__ state,
                                     long long capacity, int n_cls, const uint8_t *__restrict__ sym, double lm_thr,
                                     unsigned long long *__restrict__ keys, int *__restrict__ n_seg,
                                     int *__restrict__ f_seg, int *__restrict__ nan_seg, int *__restrict__ below)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= capacity) return;
    const long long count = min(max(state[0], 0ll), capacity);
    const int32_t *row = rows + r * kW;
    const int cls = r < count ? row[0] : -1;
    const bool ok = cls >= 1 && cls < n_cls;
    unsigned long long *k6 = keys + r * 6;
    if (!ok) {
#pragma unroll
        for (int i = 0; i < 6; ++i) k6[i] = ~0ull;
        return;
    }
    const float a = row_f(row, 3), s = row_f(row, 4);
    const float v3[3] = {a, s, (sym && sym[cls]) ? s : a};
#pragma unroll
    for (int m = 0; m < 3; ++m) {
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int seg = m * n_cls + (t == 0 ? cls : 0);
            unsigned long long key = ~0ull;
            atomicAdd(&n_seg[seg], 1);
            if (isnan(v3[m])) {
                atomicOr(&nan_seg[seg], 1);
            } else if (!((double)v3[m] > 0.1)) {
                atomicAdd(&f_seg[seg], 1);
                key = ((unsigned long long)seg << 32) | order_bits(v3[m]);
            }
            k6[m * 2 + t] = key;
        }
    }
    if ((double)a < lm_thr) { atomicAdd(&below[cls], 1); atomicAdd(&below[0], 1); }
    if ((double)s < lm_thr) { atomicAdd(&below[n_cls + cls], 1); atomicAdd(&below[n_cls], 1); }
}

__device__ double block_sum(double v, double *red)
{
    const int tid = threadIdx.x;
    red[tid] = v;
    __syncthreads();
    for (int h = kAucThreads / 2; h; h >>= 1) {       // a fixed tree: the same sum on every run
        if (tid < h) red[tid] += red[tid + h];
        __syncthreads();
    }
    const double out = red[0];
    __syncthreads();
    return out;
}

// Block s < 3 n_cls: cal_auc of segment s from its sorted distances (VOCap's area, times 10, in percent).  Block
// 3 n_cls: the keypoint-error sum and count over the counted rows.
__global__ void __launch_bounds__(kAucThreads)
eval_auc_final_kernel(const int32_t *__restrict__ rows, const long long *__restrict__ state, long long capacity,
                      int n_cls, const unsigned long long *__restrict__ sorted, const int *__restrict__ n_seg,
                      const int *__restrict__ f_seg, const int *__restrict__ nan_seg, const int *__restrict__ below,
                      double *__restrict__ auc, double *__restrict__ pct, double *__restrict__ kp)
{
    __shared__ double red[kAucThreads];
    __shared__ long long start_s;
    const int s = blockIdx.x, tid = threadIdx.x, S = 3 * n_cls;
    if (s == S) {
        const long long count = min(max(state[0], 0ll), capacity);
        double sum = 0.0, cnt = 0.0;
        for (long long r = tid; r < count; r += kAucThreads) {
            const int32_t *row = rows + r * kW;
            if (row[0] >= 1 && row[0] < n_cls) {
                sum += (double)row_f(row, 5);
                cnt += 1.0;
            }
        }
        sum = block_sum(sum, red);
        cnt = block_sum(cnt, red);
        if (tid == 0) { kp[0] = sum; kp[1] = cnt; }
        return;
    }
    if (tid == 0) {
        long long st = 0;
        for (int q = 0; q < s; ++q) st += f_seg[q];
        start_s = st;
    }
    __syncthreads();
    const int n = n_seg[s], f = f_seg[s];
    if (s < n_cls && tid == 0) {          // np.mean(dist < 0.1 diameter) * 100; an empty class gives NaN
        pct[s] = (double)below[s] / (double)n * 100.0;
        pct[n_cls + s] = (double)below[n_cls + s] / (double)n * 100.0;
    }
    if (nan_seg[s] || f == 0) {
        if (tid == 0) auc[s] = nan_seg[s] ? (double)NAN : 0.0;
        return;
    }
    const unsigned long long *d = sorted + start_s;
    // sum_i (r_i - r_{i-1}) acc_i over the distances <= 0.1 (r_{-1} = 0), closed by (0.1 - r_{f-1}) acc_{f-1}; acc_i
    // is the float32 (i + 1) / n of the reference's cumulative count
    double part = 0.0;
    for (int i = tid; i < f; i += kAucThreads) {
        const double r = (double)unorder_bits((unsigned int)d[i]);
        const double r0 = i ? (double)unorder_bits((unsigned int)d[i - 1]) : 0.0;
        const double acc = (double)__fdiv_rn((float)(i + 1), (float)n);
        part += (r - r0) * acc;
        if (i == f - 1) part += (0.1 - r) * acc;
    }
    const double area = block_sum(part, red);
    if (tid == 0) auc[s] = area * 10 * 100;
}

struct AucLayout {
    size_t keys_in, keys_out, counters, temp, temp_bytes, total;
};

static AucLayout auc_layout(long long capacity, int n_cls)
{
    AucLayout L{};
    const size_t n_keys = (size_t)capacity * 6;
    size_t tb = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tb, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                   (int)n_keys, 0, 64, (cudaStream_t)0);
    L.keys_in = 0;
    L.keys_out = align_up(L.keys_in + n_keys * 8, 256);
    L.counters = align_up(L.keys_out + n_keys * 8, 256);
    L.temp = align_up(L.counters + (size_t)(3 * 3 * n_cls + 2 * n_cls) * sizeof(int), 256);
    L.temp_bytes = tb;
    L.total = L.temp + tb;
    return L;
}

}  // namespace
}  // namespace ffb6d

extern "C" int ffb6d_eval_record(const int32_t *cls_ids, const uint8_t *valid, const uint8_t *present,
                                 const float *kps, const double *poses, const float *gt_kps, const float *pred_RT,
                                 const float *add, const float *adds, int64_t B, int64_t n_obj, int64_t n_cls,
                                 int64_t R, int64_t n_kps, int64_t obj_id, int32_t *rows, int64_t capacity,
                                 int64_t *state, double *frame_poses, uint8_t *frame_flags, int64_t frame_capacity,
                                 ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && n_obj >= 1 && B * n_obj <= FFB6D_POSE_EVAL_MAX_OBJECTS,
                    "eval_record: need B >= 1, n_obj >= 1 and B * n_obj <= %d, got B = %lld, n_obj = %lld",
                    FFB6D_POSE_EVAL_MAX_OBJECTS, (long long)B, (long long)n_obj);
    FFB6D_CHECK_ARG(n_cls >= 1 && n_cls <= FFB6D_VOTE_MAX_CLASSES, "eval_record: need 1 <= n_cls <= %d, got %lld",
                    FFB6D_VOTE_MAX_CLASSES, (long long)n_cls);
    FFB6D_CHECK_ARG(capacity >= 1 && capacity <= FFB6D_EVAL_MAX_ROWS, "eval_record: need 1 <= capacity <= %d, got %lld",
                    FFB6D_EVAL_MAX_ROWS, (long long)capacity);
    FFB6D_CHECK_ARG(obj_id >= 0 && obj_id < (1ll << 31), "eval_record: obj_id %lld outside [0, 2^31)",
                    (long long)obj_id);
    FFB6D_CHECK_ARG(obj_id > 0 || (n_kps >= 1 && n_kps <= FFB6D_VOTE_MAX_KPS && R >= n_kps + 1 &&
                                   R <= FFB6D_VOTE_MAX_KPS + 1),
                    "eval_record: need 1 <= n_kps <= %d and n_kps + 1 <= R <= %d, got n_kps = %lld, R = %lld",
                    FFB6D_VOTE_MAX_KPS, FFB6D_VOTE_MAX_KPS + 1, (long long)n_kps, (long long)R);
    FFB6D_CHECK_ARG(obj_id == 0 || n_cls >= 2, "eval_record: LineMOD needs the two-class vote, got n_cls = %lld",
                    (long long)n_cls);
    FFB6D_CHECK_ARG(present && pred_RT && add && adds && rows && state, "eval_record: null pointer");
    FFB6D_CHECK_ARG(obj_id > 0 || (cls_ids && kps && gt_kps), "eval_record: null pointer (YCB reads cls_ids, kps and "
                    "gt_kps)");
    FFB6D_CHECK_ARG((frame_poses == nullptr) == (frame_flags == nullptr), "eval_record: frame_poses and frame_flags "
                    "go together");
    FFB6D_CHECK_ARG(!frame_flags || (poses && frame_capacity >= 1 && frame_capacity <= FFB6D_EVAL_MAX_ROWS),
                    "eval_record: the frame table needs poses and 1 <= frame_capacity <= %d, got %lld",
                    FFB6D_EVAL_MAX_ROWS, (long long)frame_capacity);
    FFB6D_CHECK_ARG(((uintptr_t)cls_ids | (uintptr_t)kps | (uintptr_t)gt_kps | (uintptr_t)pred_RT | (uintptr_t)add |
                     (uintptr_t)adds | (uintptr_t)rows) % 4 == 0 &&
                    ((uintptr_t)state | (uintptr_t)poses | (uintptr_t)frame_poses) % 8 == 0,
                    "eval_record: misaligned pointer");
    eval_record_kernel<<<1, kRecThreads, 0, (cudaStream_t)stream>>>(
        cls_ids, valid, present, kps, poses, gt_kps, pred_RT, add, adds, (int)B, (int)n_obj, (int)n_cls, (int)R,
        (int)n_kps, (int)obj_id, rows, (long long)capacity, (long long *)state, frame_poses, frame_flags,
        (long long)frame_capacity);
    FFB6D_LAUNCH_OK("eval_record_kernel");
    return FFB6D_OK;
}

extern "C" size_t ffb6d_eval_auc_workspace_bytes(int64_t capacity, int64_t n_cls)
{
    if (capacity < 1 || capacity > FFB6D_EVAL_MAX_ROWS || n_cls < 1 || n_cls > FFB6D_VOTE_MAX_CLASSES) return 0;
    return auc_layout(capacity, (int)n_cls).total;
}

extern "C" int ffb6d_eval_auc(const int32_t *rows, const int64_t *state, int64_t capacity, int64_t n_cls,
                              const uint8_t *sym, double lm_thr, double *auc, double *pct, double *kp,
                              void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(capacity >= 1 && capacity <= FFB6D_EVAL_MAX_ROWS, "eval_auc: need 1 <= capacity <= %d, got %lld",
                    FFB6D_EVAL_MAX_ROWS, (long long)capacity);
    FFB6D_CHECK_ARG(n_cls >= 1 && n_cls <= FFB6D_VOTE_MAX_CLASSES, "eval_auc: need 1 <= n_cls <= %d, got %lld",
                    FFB6D_VOTE_MAX_CLASSES, (long long)n_cls);
    FFB6D_CHECK_ARG(!std::isnan(lm_thr), "eval_auc: lm_thr is NaN");
    FFB6D_CHECK_ARG(rows && state && auc && pct && kp, "eval_auc: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)rows % 4 | (uintptr_t)state % 8 | (uintptr_t)auc % 8 | (uintptr_t)pct % 8 |
                     (uintptr_t)kp % 8) == 0, "eval_auc: misaligned pointer");
    FFB6D_CHECK_ARG((uintptr_t)workspace % 256 == 0, "eval_auc: workspace must be 256-byte aligned");
    const AucLayout L = auc_layout(capacity, (int)n_cls);
    if (!workspace || workspace_bytes < L.total) {
        set_error("eval_auc: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
        return FFB6D_ERR_WORKSPACE;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    unsigned long long *keys_in = (unsigned long long *)(ws + L.keys_in);
    unsigned long long *keys_out = (unsigned long long *)(ws + L.keys_out);
    const int K = (int)n_cls, S = 3 * K;
    int *n_seg = (int *)(ws + L.counters), *f_seg = n_seg + S, *nan_seg = f_seg + S, *below = nan_seg + S;
    FFB6D_CUDA(cudaMemsetAsync(n_seg, 0, (size_t)(3 * S + 2 * K) * sizeof(int), st));
    eval_auc_keys_kernel<<<(unsigned)ceil_div(capacity, 256), 256, 0, st>>>(
        rows, (const long long *)state, (long long)capacity, K, sym, lm_thr, keys_in, n_seg, f_seg, nan_seg, below);
    FFB6D_LAUNCH_OK("eval_auc_keys_kernel");
    size_t tb = L.temp_bytes;
    FFB6D_CUDA(cub::DeviceRadixSort::SortKeys(ws + L.temp, tb, keys_in, keys_out, (int)(capacity * 6), 0, 64, st));
    count_launch();
    eval_auc_final_kernel<<<(unsigned)(S + 1), kAucThreads, 0, st>>>(
        rows, (const long long *)state, (long long)capacity, K, keys_out, n_seg, f_seg, nan_seg, below, auc, pct, kp);
    FFB6D_LAUNCH_OK("eval_auc_final_kernel");
    return FFB6D_OK;
}
