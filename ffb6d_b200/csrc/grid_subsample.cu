// grid_subsample.cu -- voxel-grid barycentre subsampling on the GPU (sm_90a).
//
// Replaces grid_subsampling() (GS/cpp_subsampling/grid_subsampling/grid_subsampling.cpp:5-106),
// which walks the cloud once and accumulates per-voxel sums in an unordered_map.  The GPU
// version keeps the reference's arithmetic bit for bit:
//   1. min/max of the cloud (reduction)            -> origin, NX, NY exactly as :27-31
//   2. voxel key per point, same fp32 expression   -> key = iX + NX*iY + NX*NY*iZ   (:53-56)
//   3. STABLE radix sort of (key, point index)     -> each voxel's points contiguous and still in
//                                                     input order (cub::DeviceRadixSort, the
//                                                     toolkit's library sort: this op is not on
//                                                     the FFB6D fusion path, SURVEY.md §0)
//   4. one thread per voxel adds its points IN INPUT ORDER in fp32, like the reference's
//      `point += p` / `features += f` (grid_subsampling.h:42-79), then
//      barycentre = sum * (float)(1.0 / count), mean feature = sum / (float)count   (:87-94)
//   5. labels: (voxel, label) pairs sorted, longest run wins, smallest label on ties
//      (the reference takes the first maximum in hash-map order, :99-101).
// Rows come out by ascending voxel key.
#include "common.cuh"

#include <algorithm>
#include <cub/cub.cuh>
#include <math.h>

namespace ffb6d {

__global__ void __launch_bounds__(1024)
gs_minmax_kernel(const float *__restrict__ pts, size_t N, float *__restrict__ out6)
{
    // single CTA: N is a pre-processing sized cloud, the reduction is not the bottleneck
    const float INF = __int_as_float(0x7f800000);
    float mn[3] = {INF, INF, INF}, mx[3] = {-INF, -INF, -INF};
    for (size_t i = threadIdx.x; i < N; i += blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = pts[3 * i + a];
            // the reference compares with '<' / '>' starting from point 0 (cloud.cpp:27-67)
            mn[a] = v < mn[a] ? v : mn[a];
            mx[a] = v > mx[a] ? v : mx[a];
        }
    }
    __shared__ float red[6][32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if (lane == 0) {
            red[a][wid] = mn[a];
            red[3 + a][wid] = mx[a];
        }
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        float v = red[threadIdx.x][0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            v = threadIdx.x < 3 ? fminf(v, red[threadIdx.x][w]) : fmaxf(v, red[threadIdx.x][w]);
        out6[threadIdx.x] = v;
    }
}

__global__ void __launch_bounds__(256)
gs_key_kernel(const float *__restrict__ pts, size_t N, float ox, float oy, float oz, float dl,
              unsigned long long NX, unsigned long long NY, unsigned long long *__restrict__ keys,
              unsigned int *__restrict__ order)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    // (size_t)floor((p.x - origin.x) / sampleDl), fp32, IEEE division      (:53-55)
    const unsigned long long iX = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(pts[3 * i + 0], ox), dl));
    const unsigned long long iY = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(pts[3 * i + 1], oy), dl));
    const unsigned long long iZ = (unsigned long long)floorf(__fdiv_rn(__fsub_rn(pts[3 * i + 2], oz), dl));
    keys[i] = iX + NX * iY + NX * NY * iZ;
    order[i] = (unsigned int)i;
}

__global__ void __launch_bounds__(256)
gs_heads_kernel(const unsigned long long *__restrict__ keys, size_t N, unsigned int *__restrict__ head)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

// rank[i] = inclusive scan of head -> voxel number + 1; starts[v] = first sorted position of voxel v
__global__ void __launch_bounds__(256)
gs_starts_kernel(const unsigned int *__restrict__ head, const unsigned int *__restrict__ rank, size_t N,
                 unsigned int *__restrict__ starts)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    if (head[i]) starts[rank[i] - 1] = (unsigned int)i;
}

__global__ void __launch_bounds__(128)
gs_reduce_kernel(const float *__restrict__ pts, const float *__restrict__ feats, size_t fdim,
                 const unsigned int *__restrict__ order, const unsigned int *__restrict__ starts,
                 size_t M, size_t N, float *__restrict__ sub_pts, float *__restrict__ sub_feats)
{
    const size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= M) return;
    const size_t a = starts[v], b = (v + 1 < M) ? starts[v + 1] : N;
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (size_t t = a; t < b; ++t) {   // input order inside the voxel (stable sort)
        const size_t i = order[t];
        sx = __fadd_rn(sx, pts[3 * i + 0]);
        sy = __fadd_rn(sy, pts[3 * i + 1]);
        sz = __fadd_rn(sz, pts[3 * i + 2]);
    }
    const int count = (int)(b - a);
    const float r = (float)(1.0 / (double)count);   // `point * (1.0 / count)`: double reciprocal (:87)
    sub_pts[3 * v + 0] = __fmul_rn(sx, r);
    sub_pts[3 * v + 1] = __fmul_rn(sy, r);
    sub_pts[3 * v + 2] = __fmul_rn(sz, r);
    const float fc = (float)count;
    for (size_t f = 0; f < fdim; ++f) {
        float acc = 0.f;
        for (size_t t = a; t < b; ++t) acc = __fadd_rn(acc, feats[(size_t)order[t] * fdim + f]);
        sub_feats[v * fdim + f] = __fdiv_rn(acc, fc);   // f / count                     (:90-94)
    }
}

__global__ void __launch_bounds__(256)
gs_label_key_kernel(const int *__restrict__ classes, size_t ldim, size_t l,
                    const unsigned int *__restrict__ order, const unsigned int *__restrict__ rank,
                    size_t N, unsigned long long *__restrict__ lkeys)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= N) return;
    const unsigned int lab = (unsigned int)classes[(size_t)order[t] * ldim + l] ^ 0x80000000u;   // order-preserving
    lkeys[t] = ((unsigned long long)(rank[t] - 1) << 32) | lab;
}

__global__ void __launch_bounds__(128)
gs_label_vote_kernel(const unsigned long long *__restrict__ lkeys, const unsigned int *__restrict__ starts,
                     size_t M, size_t N, size_t ldim, size_t l, int *__restrict__ sub_classes)
{
    const size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= M) return;
    const size_t a = starts[v], b = (v + 1 < M) ? starts[v + 1] : N;
    unsigned int best = (unsigned int)(lkeys[a] & 0xffffffffu), cur = best;
    size_t best_n = 0, run = 0;
    for (size_t t = a; t < b; ++t) {
        const unsigned int lab = (unsigned int)(lkeys[t] & 0xffffffffu);
        run = (t > a && lab == cur) ? run + 1 : 1;
        cur = lab;
        if (run > best_n) {   // strict: the smallest label wins a tie
            best_n = run;
            best = lab;
        }
    }
    sub_classes[v * ldim + l] = (int)(best ^ 0x80000000u);
}

struct DevBuf {   // frees on scope exit
    void *p = nullptr;
    ~DevBuf()
    {
        if (p) cudaFree(p);
    }
    cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 16); }
    template <typename T>
    T *as()
    {
        return (T *)p;
    }
};

}  // namespace ffb6d

using namespace ffb6d;

#define GS_LAUNCH(name)          \
    do {                         \
        FFB6D_LAUNCH_OK(name);   \
    } while (0)

extern "C" int ffb6d_grid_subsample_host(const float *points, size_t N, const float *features,
                                         size_t fdim, const int *classes, size_t ldim,
                                         float sampleDl, float *sub_points, float *sub_features,
                                         int *sub_classes, size_t *M_out)
{
    FFB6D_CHECK_ARG(points && sub_points && M_out, "grid_subsample: null pointer");
    FFB6D_CHECK_ARG(N >= 1 && N < (1ull << 31), "grid_subsample: N=%zu outside [1, 2^31) (32-bit item counts of the sort / scan)", N);
    FFB6D_CHECK_ARG(sampleDl > 0.f, "grid_subsample: sampleDl must be positive");
    FFB6D_CHECK_ARG(fdim == 0 || (features && sub_features), "grid_subsample: null features");
    FFB6D_CHECK_ARG(ldim == 0 || (classes && sub_classes), "grid_subsample: null classes");
    if (ffb6d_device_count() == 0) {
        set_error("grid_subsample: no CUDA device visible");
        return FFB6D_ERR_NO_DEVICE;
    }
    cudaStream_t st = 0;
    DevBuf d_pts, d_feat, d_cls, d_mm, d_keys, d_keys2, d_ord, d_ord2, d_head, d_rank, d_starts, d_tmp,
        d_sp, d_sf, d_sc, d_lk, d_lk2;
    FFB6D_CUDA(d_pts.alloc(N * 3 * sizeof(float)));
    FFB6D_CUDA(cudaMemcpyAsync(d_pts.p, points, N * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
    if (fdim) {
        FFB6D_CUDA(d_feat.alloc(N * fdim * sizeof(float)));
        FFB6D_CUDA(cudaMemcpyAsync(d_feat.p, features, N * fdim * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    if (ldim) {
        FFB6D_CUDA(d_cls.alloc(N * ldim * sizeof(int)));
        FFB6D_CUDA(cudaMemcpyAsync(d_cls.p, classes, N * ldim * sizeof(int), cudaMemcpyHostToDevice, st));
    }
    // 1. limits of the cloud
    FFB6D_CUDA(d_mm.alloc(6 * sizeof(float)));
    gs_minmax_kernel<<<1, 1024, 0, st>>>(d_pts.as<float>(), N, d_mm.as<float>());
    GS_LAUNCH("gs_minmax_kernel");
    float mm[6];
    FFB6D_CUDA(cudaMemcpyAsync(mm, d_mm.p, sizeof(mm), cudaMemcpyDeviceToHost, st));
    FFB6D_CUDA(cudaStreamSynchronize(st));
    // grid_subsampling.cpp:27-31 -- host fp32, x86-64 has no FMA contraction here
    volatile float inv = 1 / sampleDl;
    float org[3];
    for (int a = 0; a < 3; ++a) {
        volatile float t = mm[a] * inv;
        volatile float f = floorf(t);
        org[a] = f * sampleDl;
    }
    volatile float ex = (mm[3] - org[0]) / sampleDl, ey = (mm[4] - org[1]) / sampleDl;
    const unsigned long long NX = (unsigned long long)floorf(ex) + 1;
    const unsigned long long NY = (unsigned long long)floorf(ey) + 1;

    // 2. keys, 3. stable sort by key
    FFB6D_CUDA(d_keys.alloc(N * 8));
    FFB6D_CUDA(d_keys2.alloc(N * 8));
    FFB6D_CUDA(d_ord.alloc(N * 4));
    FFB6D_CUDA(d_ord2.alloc(N * 4));
    const unsigned nb = (unsigned)ceil_div((int64_t)N, 256);
    gs_key_kernel<<<nb, 256, 0, st>>>(d_pts.as<float>(), N, org[0], org[1], org[2], sampleDl, NX, NY,
                                      d_keys.as<unsigned long long>(), d_ord.as<unsigned int>());
    GS_LAUNCH("gs_key_kernel");
    size_t tmp_bytes = 0, tb2 = 0, tb3 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_keys.as<unsigned long long>(),
                                    d_keys2.as<unsigned long long>(), d_ord.as<unsigned int>(),
                                    d_ord2.as<unsigned int>(), (int)N, 0, 64, st);
    cub::DeviceScan::InclusiveSum(nullptr, tb2, (unsigned int *)nullptr, (unsigned int *)nullptr, (int)N, st);
    cub::DeviceRadixSort::SortKeys(nullptr, tb3, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                   (int)N, 0, 64, st);
    tmp_bytes = std::max(tmp_bytes, std::max(tb2, tb3));
    FFB6D_CUDA(d_tmp.alloc(tmp_bytes));
    FFB6D_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp.p, tmp_bytes, d_keys.as<unsigned long long>(),
                                               d_keys2.as<unsigned long long>(), d_ord.as<unsigned int>(),
                                               d_ord2.as<unsigned int>(), (int)N, 0, 64, st));
    count_launch(4);
    // voxel heads and ranks
    FFB6D_CUDA(d_head.alloc(N * 4));
    FFB6D_CUDA(d_rank.alloc(N * 4));
    gs_heads_kernel<<<nb, 256, 0, st>>>(d_keys2.as<unsigned long long>(), N, d_head.as<unsigned int>());
    GS_LAUNCH("gs_heads_kernel");
    FFB6D_CUDA(cub::DeviceScan::InclusiveSum(d_tmp.p, tmp_bytes, d_head.as<unsigned int>(),
                                             d_rank.as<unsigned int>(), (int)N, st));
    count_launch(2);
    unsigned int M32 = 0;
    FFB6D_CUDA(cudaMemcpyAsync(&M32, d_rank.as<unsigned int>() + (N - 1), 4, cudaMemcpyDeviceToHost, st));
    FFB6D_CUDA(cudaStreamSynchronize(st));
    const size_t M = M32;
    FFB6D_CUDA(d_starts.alloc(M * 4));
    gs_starts_kernel<<<nb, 256, 0, st>>>(d_head.as<unsigned int>(), d_rank.as<unsigned int>(), N,
                                         d_starts.as<unsigned int>());
    GS_LAUNCH("gs_starts_kernel");
    // 4. per-voxel sums in input order
    FFB6D_CUDA(d_sp.alloc(M * 3 * sizeof(float)));
    if (fdim) FFB6D_CUDA(d_sf.alloc(M * fdim * sizeof(float)));
    const unsigned mb = (unsigned)ceil_div((int64_t)M, 128);
    gs_reduce_kernel<<<mb, 128, 0, st>>>(d_pts.as<float>(), d_feat.as<float>(), fdim, d_ord2.as<unsigned int>(),
                                         d_starts.as<unsigned int>(), M, N, d_sp.as<float>(), d_sf.as<float>());
    GS_LAUNCH("gs_reduce_kernel");
    // 5. labels
    if (ldim) {
        FFB6D_CUDA(d_sc.alloc(M * ldim * sizeof(int)));
        FFB6D_CUDA(d_lk.alloc(N * 8));
        FFB6D_CUDA(d_lk2.alloc(N * 8));
        for (size_t l = 0; l < ldim; ++l) {
            gs_label_key_kernel<<<nb, 256, 0, st>>>(d_cls.as<int>(), ldim, l, d_ord2.as<unsigned int>(),
                                                    d_rank.as<unsigned int>(), N, d_lk.as<unsigned long long>());
            GS_LAUNCH("gs_label_key_kernel");
            FFB6D_CUDA(cub::DeviceRadixSort::SortKeys(d_tmp.p, tmp_bytes, d_lk.as<unsigned long long>(),
                                                      d_lk2.as<unsigned long long>(), (int)N, 0, 64, st));
            count_launch(4);
            gs_label_vote_kernel<<<mb, 128, 0, st>>>(d_lk2.as<unsigned long long>(), d_starts.as<unsigned int>(),
                                                     M, N, ldim, l, d_sc.as<int>());
            GS_LAUNCH("gs_label_vote_kernel");
        }
    }
    FFB6D_CUDA(cudaMemcpyAsync(sub_points, d_sp.p, M * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (fdim)
        FFB6D_CUDA(cudaMemcpyAsync(sub_features, d_sf.p, M * fdim * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (ldim)
        FFB6D_CUDA(cudaMemcpyAsync(sub_classes, d_sc.p, M * ldim * sizeof(int), cudaMemcpyDeviceToHost, st));
    FFB6D_CUDA(cudaStreamSynchronize(st));
    *M_out = M;
    return FFB6D_OK;
}
