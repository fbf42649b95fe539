// knn_common.cuh -- per-thread sorted top-K list kept in registers.
#pragma once
#include "common.cuh"

namespace ffb6d {

// Sorted ascending by (distance, index).  Empty slots hold (+inf, 0): a support
// smaller than K therefore leaves index 0 in the trailing slots, which is what
// the reference's value-initialised out_ids show (NN/knn_.cxx:120-121).
template <int KCAP>
struct TopK {
    float d[KCAP];
    int i[KCAP];

    __device__ __forceinline__ void init()
    {
#pragma unroll
        for (int j = 0; j < KCAP; ++j) {
            d[j] = __int_as_float(0x7f800000);
            i[j] = 0;
        }
    }
    __device__ __forceinline__ float worst() const { return d[KCAP - 1]; }
    // distance of the K-th entry (1 <= K <= KCAP) without dynamic register indexing
    __device__ __forceinline__ float kth(int K) const
    {
        float v = d[KCAP - 1];
#pragma unroll
        for (int j = KCAP - 2; j >= 0; --j) v = (j >= K - 1) ? d[j] : v;
        return v;
    }
    __device__ __forceinline__ int worst_idx() const { return i[KCAP - 1]; }

    // Candidates arrive in ascending index order: a candidate goes behind every
    // entry with distance <= its own (strict '>' like KNNResultSet::addPoint,
    // NN/nanoflann.hpp:118-129).  Caller guarantees dist < worst().
    __device__ __forceinline__ void push_ordered(float dist, int id)
    {
#pragma unroll
        for (int j = KCAP - 1; j > 0; --j) {
            const bool shift = d[j - 1] > dist;      // entry j-1 moves to j
            const bool here = !shift && (d[j] > dist);  // candidate lands in j
            const float nd = shift ? d[j - 1] : (here ? dist : d[j]);
            const int ni = shift ? i[j - 1] : (here ? id : i[j]);
            d[j] = nd;
            i[j] = ni;
        }
        if (d[0] > dist) {
            d[0] = dist;
            i[0] = id;
        }
    }

    // true when (dist,id) sorts before the current worst entry
    __device__ __forceinline__ bool accepts(float dist, int id) const
    {
        return dist < d[KCAP - 1] || (dist == d[KCAP - 1] && id < i[KCAP - 1]);
    }

    // Candidates in arbitrary order: total order (distance, index).  Caller
    // guarantees accepts(dist,id).
    __device__ __forceinline__ void push_any(float dist, int id)
    {
#pragma unroll
        for (int j = KCAP - 1; j > 0; --j) {
            const bool shift = d[j - 1] > dist || (d[j - 1] == dist && i[j - 1] > id);
            const bool after = d[j] > dist || (d[j] == dist && i[j] > id);
            const bool here = !shift && after;
            const float nd = shift ? d[j - 1] : (here ? dist : d[j]);
            const int ni = shift ? i[j - 1] : (here ? id : i[j]);
            d[j] = nd;
            i[j] = ni;
        }
        if (d[0] > dist || (d[0] == dist && i[0] > id)) {
            d[0] = dist;
            i[0] = id;
        }
    }
};

// entry points of the two search algorithms (knn_brute.cu, knn_grid.cu)
int knn_brute_launch(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                     int K, void *idx_out, int idx_is_i64, cudaStream_t st);
size_t knn_grid_workspace_bytes(int64_t B, int64_t S, int64_t Q, int K);   // 0: the grid declines
int knn_grid_launch(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                    int K, void *idx_out, int idx_is_i64, void *workspace, size_t workspace_bytes,
                    cudaStream_t st);
// build once, query many times (knn_grid.cu)
void knn_grid_tune(float cell_scale, int quantile);
void knn_grid_tune_k1(float cell_scale_k1);
size_t knn_grid_store_bytes(int64_t B, int64_t S);
size_t knn_grid_query_bytes(int64_t B, int64_t Q);
int knn_grid_build(const float *support, int64_t B, int64_t S, int K, void *grid_mem,
                   size_t grid_bytes, cudaStream_t st);
int knn_grid_query(const float *support, const float *query, int64_t B, int64_t S, int64_t Q, int K,
                   void *idx_out, int idx_is_i64, const void *grid_mem, size_t grid_bytes,
                   void *scratch, size_t scratch_bytes, cudaStream_t st, int64_t query_width = 0);

}  // namespace ffb6d
