// knn_brute.cu -- tiled all-pairs exact KNN (sm_90a).
//
// One thread owns one query and keeps its K best (distance, index) pairs sorted
// in registers; the support cloud streams through shared memory in float4
// tiles that every thread reads as a broadcast.  Distances use the reference's
// unfused fp32 arithmetic (common.cuh: ref_sqdist); candidates are visited in
// ascending support index and inserted behind equal distances, which is the
// "stable ascending sort, first K" order the reference produces on tie-free
// input (NN/nanoflann.hpp:115-139, SURVEY.md App. B).
//
// This is the path for small supports (where building a search grid costs more
// than scanning) and the cross-check for the grid search in knn_grid.cu.
#include "common.cuh"
#include "knn_common.cuh"

namespace ffb6d {

template <int KCAP, int THREADS, int TILE, typename IdxT>
__global__ void __launch_bounds__(THREADS)
knn_brute_kernel(const float *__restrict__ support, const float *__restrict__ query, int S, int Q,
                 int K, IdxT *__restrict__ idx_out)
{
    __shared__ float4 tile[TILE];
    const int b = blockIdx.y;
    const float *sup = support + (size_t)b * S * 3;
    const int q = blockIdx.x * THREADS + threadIdx.x;
    const bool active = q < Q;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (active) {
        const float *qp = query + ((size_t)b * Q + q) * 3;
        qx = qp[0];
        qy = qp[1];
        qz = qp[2];
    }
    TopK<KCAP> top;
    top.init();

    for (int s0 = 0; s0 < S; s0 += TILE) {
        const int n = min(TILE, S - s0);
        __syncthreads();
        // stage 3n contiguous floats -> float4 per point
        const float *src = sup + (size_t)s0 * 3;
        for (int t = threadIdx.x; t < 3 * n; t += THREADS)
            reinterpret_cast<float *>(tile)[(t / 3) * 4 + (t % 3)] = __ldg(src + t);
        __syncthreads();
        if (active) {
#pragma unroll 4
            for (int t = 0; t < n; ++t) {
                const float4 p = tile[t];
                const float d = ref_sqdist(qx, qy, qz, p.x, p.y, p.z);
                if (d < top.worst()) top.push_ordered(d, s0 + t);
            }
        }
    }
    if (active) {
        IdxT *o = idx_out + ((size_t)b * Q + q) * K;
#pragma unroll
        for (int j = 0; j < KCAP; ++j)
            if (j < K) o[j] = (IdxT)top.i[j];
    }
}

template <int KCAP, typename IdxT>
static int launch_brute_t(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                          int K, void *idx_out, cudaStream_t st)
{
    constexpr int THREADS = (KCAP >= 32) ? 64 : 128;
    constexpr int TILE = 1024;
    dim3 grid((unsigned)ceil_div(Q, THREADS), (unsigned)B);
    knn_brute_kernel<KCAP, THREADS, TILE, IdxT>
        <<<grid, THREADS, 0, st>>>(support, query, (int)S, (int)Q, K, (IdxT *)idx_out);
    FFB6D_LAUNCH_OK("knn_brute_kernel");
    return FFB6D_OK;
}

template <typename IdxT>
static int launch_brute_k(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                          int K, void *idx_out, cudaStream_t st)
{
    if (K == 1) return launch_brute_t<1, IdxT>(support, query, B, S, Q, K, idx_out, st);
    if (K <= 4) return launch_brute_t<4, IdxT>(support, query, B, S, Q, K, idx_out, st);
    if (K <= 8) return launch_brute_t<8, IdxT>(support, query, B, S, Q, K, idx_out, st);
    if (K <= 16) return launch_brute_t<16, IdxT>(support, query, B, S, Q, K, idx_out, st);
    if (K <= 32) return launch_brute_t<32, IdxT>(support, query, B, S, Q, K, idx_out, st);
    return launch_brute_t<64, IdxT>(support, query, B, S, Q, K, idx_out, st);
}

int knn_brute_launch(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                     int K, void *idx_out, int idx_is_i64, cudaStream_t st)
{
    if (idx_is_i64)
        return launch_brute_k<long long>(support, query, B, S, Q, K, idx_out, st);
    return launch_brute_k<int>(support, query, B, S, Q, K, idx_out, st);
}

}  // namespace ffb6d
