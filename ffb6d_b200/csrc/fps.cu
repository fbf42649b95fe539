// fps.cu -- batched farthest point sampling (ffb6d_farthest_point_sampling), the keypoint selection of the
// reference's object-info tool (utils/dataset_tools/fps/src/farthest_point_sampling.cpp, behind
// utils/dataset_tools/gen_obj_info.py:86-88).
//
// One thread-block cluster per cloud.  Each of its C CTAs keeps a contiguous chunk of the cloud in shared memory
// as float4 (x, y, z, min_dist) for the whole run, so HBM is read once.  A round updates min_dist with the point
// chosen last and takes the arg-max in three levels: warp shuffles, the block (one __syncthreads), then the
// cluster, where every warp reads the C block winners through distributed shared memory after one cluster barrier.
// The block winners live in two slots used in alternate rounds: a CTA writing round r + 2's slot has passed round
// r + 1's barrier, which no CTA reaches before it has finished reading round r's slots.
//
// Tie contract, the reference's find_max_dist_idx (:56-73): the first index with a strictly greater value, from
// max_idx = 0, max_d = 0.f.  A candidate is encoded as (float bits of a min_dist > 0) << 32 | ~index, so the
// largest key is the largest distance and, among equal ones, the lowest index; no candidate (every remaining
// distance 0 or NaN) is key 0, which decodes to index 0 -- the reference's re-selection of point 0.
#include "common.cuh"

#include <cfloat>
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace ffb6d {
namespace {

constexpr int kThreads = 1024;
constexpr int kPtsPerCta = FFB6D_FPS_MAX_POINTS / FFB6D_FPS_MAX_CLUSTER;   // 14336 x 16 B = 224 KB
constexpr float kSelected = -1.f;    // min_dist of a selected point: never < a distance, never a candidate

struct __align__(16) Slot {
    unsigned long long key;
    float x, y, z;
};

__device__ __forceinline__ unsigned long long cand_key(float d, int i)
{
    return d > 0.f ? ((unsigned long long)__float_as_uint(d) << 32) | (0xFFFFFFFFu - (unsigned)i) : 0ull;
}

__device__ __forceinline__ int key_index(unsigned long long k) { return k ? (int)(0xFFFFFFFFu - (unsigned)k) : 0; }

__device__ __forceinline__ unsigned long long warp_max(unsigned long long k)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, k, o);
        k = v > k ? v : k;
    }
    return k;
}

// std::max(a, b) / std::min(a, b) as max_vec3 / min_vec3 call them (:107-120): b replaces a only on a strict
// comparison, so NaN never enters and -FLT_MAX / FLT_MAX survive an axis without finite values.
__device__ __forceinline__ float ref_max(float a, float b) { return a < b ? b : a; }
__device__ __forceinline__ float ref_min(float a, float b) { return b < a ? b : a; }

__global__ void __launch_bounds__(kThreads, 1)
fps_kernel(const float *__restrict__ pts, const int *__restrict__ counts, int P, int S, int chunk,
           const int *__restrict__ start, int init_center, int *__restrict__ idx_out)
{
    extern __shared__ float4 sm[];                 // [chunk] (x, y, z, min_dist)
    __shared__ unsigned long long warp_key[kThreads / 32];
    __shared__ float warp_box[kThreads / 32][6];
    __shared__ float box[6];                       // this CTA's (max x, y, z, min x, y, z)
    __shared__ Slot slot[2];

    cg::cluster_group cluster = cg::this_cluster();
    const int C = (int)cluster.num_blocks();
    const int rank = (int)cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int g = blockIdx.y;
    const float *cp = pts + (size_t)g * P * 3;
    int *out = idx_out + (size_t)g * S;

    // Every CTA of the cluster reads the same count and start, so all of them leave here together.
    const int n = counts ? counts[g] : P;
    int cur = 0;
    bool bad = n < 1 || n > P;
    if (!bad && !init_center) {
        cur = start[g];
        bad = cur < 0 || cur >= n;
    }
    if (bad) {
        if (rank == 0)
            for (int s = tid; s < S; s += blockDim.x) out[s] = -1;
        return;
    }

    const int lo = rank * chunk;
    const int m = max(min(lo + chunk, n) - lo, 0);
    for (int i = tid; i < m; i += blockDim.x) {
        const float *q = cp + (size_t)(lo + i) * 3;
        sm[i] = make_float4(q[0], q[1], q[2], FLT_MAX);
    }
    const float p0x = cp[0], p0y = cp[1], p0z = cp[2];

    // the cluster's arg-max of the block candidates; returns the winner and its coordinates
    int par = 0;
    float cx, cy, cz;
    auto select = [&](unsigned long long best) {
        best = warp_max(best);
        if (lane == 0) warp_key[warp] = best;
        __syncthreads();
        if (warp == 0) {
            unsigned long long k = lane < nwarps ? warp_key[lane] : 0ull;
            k = warp_max(k);
            if (lane == 0) {
                Slot s{k, 0.f, 0.f, 0.f};
                if (k) {
                    const float4 p = sm[key_index(k) - lo];
                    s.x = p.x; s.y = p.y; s.z = p.z;
                }
                slot[par] = s;
            }
        }
        cluster.sync();
        Slot r{0ull, 0.f, 0.f, 0.f};
        if (lane < C) r = *cluster.map_shared_rank(&slot[par], lane);
        const unsigned long long k = warp_max(r.key);
        par ^= 1;
        if (!k) {
            cx = p0x; cy = p0y; cz = p0z;
            return 0;
        }
        const int src = __ffs(__ballot_sync(0xffffffffu, lane < C && r.key == k)) - 1;
        cx = __shfl_sync(0xffffffffu, r.x, src);
        cy = __shfl_sync(0xffffffffu, r.y, src);
        cz = __shfl_sync(0xffffffffu, r.z, src);
        return key_index(k);
    };

    if (init_center) {
        // sample_farthest_points_init_center (:122-149): min_dist = min(|p - (max + min) * 0.5f|^2, FLT_MAX),
        // max / min per axis over the whole cloud, then the first arg-max
        float b[6] = {-FLT_MAX, -FLT_MAX, -FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX};
        for (int i = tid; i < m; i += blockDim.x) {
            const float4 p = sm[i];
            b[0] = ref_max(b[0], p.x); b[1] = ref_max(b[1], p.y); b[2] = ref_max(b[2], p.z);
            b[3] = ref_min(b[3], p.x); b[4] = ref_min(b[4], p.y); b[5] = ref_min(b[5], p.z);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
#pragma unroll
            for (int a = 0; a < 6; ++a) {
                const float v = __shfl_xor_sync(0xffffffffu, b[a], o);
                b[a] = a < 3 ? ref_max(b[a], v) : ref_min(b[a], v);
            }
        }
        if (lane == 0)
            for (int a = 0; a < 6; ++a) warp_box[warp][a] = b[a];
        __syncthreads();
        if (tid < 6) {
            float v = warp_box[0][tid];
            for (int w = 1; w < nwarps; ++w) v = tid < 3 ? ref_max(v, warp_box[w][tid]) : ref_min(v, warp_box[w][tid]);
            box[tid] = v;
        }
        cluster.sync();
        float c[3];
        for (int a = 0; a < 3; ++a) {
            float mx = -FLT_MAX, mn = FLT_MAX;
            for (int r = 0; r < C; ++r) {
                const float *rb = cluster.map_shared_rank(box, r);
                mx = ref_max(mx, rb[a]);
                mn = ref_min(mn, rb[3 + a]);
            }
            c[a] = __fmul_rn(__fadd_rn(mx, mn), 0.5f);      // (max + min) / 2.f = * (1.f / 2.f), :20, :138
        }
        unsigned long long best = 0ull;
        for (int i = tid; i < m; i += blockDim.x) {
            const float4 p = sm[i];
            const float d = ref_sqdist(p.x, p.y, p.z, c[0], c[1], c[2]);
            const float md = FLT_MAX < d ? FLT_MAX : d;     // std::min(d, FLT_MAX): a NaN d is kept
            sm[i].w = md;
            best = best > cand_key(md, lo + i) ? best : cand_key(md, lo + i);
        }
        cur = select(best);
    } else {
        cx = cp[(size_t)cur * 3]; cy = cp[(size_t)cur * 3 + 1]; cz = cp[(size_t)cur * 3 + 2];
    }

    // sample_farthest_points (:76-105): select cur, then min_dist = min(min_dist, |p - cur|^2) over the points
    // not yet selected and the next arg-max
    for (int s = 0; s < S; ++s) {
        if (rank == 0 && tid == 0) out[s] = cur;
        if (s == S - 1) break;
        unsigned long long best = 0ull;
        for (int i = tid; i < m; i += blockDim.x) {
            const float4 p = sm[i];
            float md = p.w;
            if (lo + i == cur) {
                md = kSelected;
            } else {
                const float d = ref_sqdist(p.x, p.y, p.z, cx, cy, cz);
                if (d < md) md = d;
            }
            sm[i].w = md;
            const unsigned long long k = cand_key(md, lo + i);
            best = k > best ? k : best;
        }
        cur = select(best);
    }
    cluster.sync();   // no CTA leaves while another may still read its slots
}

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" size_t ffb6d_farthest_point_sampling_workspace_bytes(int64_t G, int64_t P, int64_t S)
{
    (void)G; (void)P; (void)S;
    return 0;
}

extern "C" int ffb6d_farthest_point_sampling(const float *pts, const int *n_points_per_cloud, int64_t G, int64_t P,
                                             int64_t S, const int *start, int init_center, int *idx_out, void *ws,
                                             size_t ws_bytes, ffb6d_stream_t stream)
{
    (void)ws; (void)ws_bytes;
    FFB6D_CHECK_ARG(G >= 1 && G <= FFB6D_FPS_MAX_CLOUDS, "farthest_point_sampling: need 1 <= G <= %d, got %lld",
                    FFB6D_FPS_MAX_CLOUDS, (long long)G);
    FFB6D_CHECK_ARG(P >= 1 && P <= FFB6D_FPS_MAX_POINTS, "farthest_point_sampling: need 1 <= P <= %d, got %lld",
                    FFB6D_FPS_MAX_POINTS, (long long)P);
    FFB6D_CHECK_ARG(S >= 1 && S <= FFB6D_FPS_MAX_SAMPLES, "farthest_point_sampling: need 1 <= S <= %d, got %lld",
                    FFB6D_FPS_MAX_SAMPLES, (long long)S);
    FFB6D_CHECK_ARG(init_center == 0 || init_center == 1, "farthest_point_sampling: init_center must be 0 or 1");
    FFB6D_CHECK_ARG(pts && idx_out, "farthest_point_sampling: null pointer");
    FFB6D_CHECK_ARG(init_center || start, "farthest_point_sampling: start is required without init_center");
    FFB6D_CHECK_ARG(((uintptr_t)pts | (uintptr_t)idx_out | (uintptr_t)start | (uintptr_t)n_points_per_cloud) % 4 == 0,
                    "farthest_point_sampling: pointers must be 4-byte aligned");

    const int C = (int)ceil_div(P, kPtsPerCta);
    const int chunk = (int)ceil_div(P, C);
    const int threads = (int)std::min<int64_t>(kThreads, ceil_div(chunk, 32) * 32);
    const size_t smem = (size_t)chunk * sizeof(float4);
    FFB6D_CHECK_ARG(smem <= (size_t)device_info().max_smem_optin,
                    "farthest_point_sampling: %zu bytes of shared memory per CTA exceed this device's %d", smem,
                    device_info().max_smem_optin);
    FFB6D_OPTIN_SMEM(fps_kernel, (size_t)kPtsPerCta * sizeof(float4));

    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)C, (unsigned)G, 1);
    cfg.blockDim = dim3((unsigned)threads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    FFB6D_CUDA(cudaLaunchKernelEx(&cfg, fps_kernel, pts, n_points_per_cloud, (int)P, (int)S, chunk, start, init_center,
                                  idx_out));
    FFB6D_LAUNCH_OK("fps_kernel");
    return FFB6D_OK;
}
