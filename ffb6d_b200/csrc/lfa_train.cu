// lfa_train.cu -- the attentive pooling of RandLA's Building_block in training, forward and backward (sm_90a).
//
// Reference (models/RandLA/RandLANet.py:200-212, 243-248), per point n with its K = 16 neighbours idx[n, :]:
//     x_k   = cat(feature[:, idx[n, k]], f_xyz[:, n, k])                  [d = 2 * d/2 channels]
//     f_agg = sum_k x_k * softmax_k(W_fc . x_k)                           [B, d, N]
// The per-op training path materialises the gathered neighbours [B, d/2, N, 16] and the logits [B, d, N, 16] and
// keeps both alive for the backward.  Here a warp owns a point (the layout of lfa_fused.cu): it gathers x into its
// slice of shared memory, forms the logits with warp_mac16, takes the softmax over the 16 neighbours (max
// subtracted, as torch) and the weighted sum in registers.  The forward writes f_agg only.
//
// The backward recomputes x, the logits and the softmax s from the saved inputs, then per position
//     dlogit = s * g * (x - f_agg)              (g = dL/df_agg of the point's channel)
//     dx     = g * s + W_fc^T . dlogit
// and writes dx: its f_xyz half to grad_f_xyz [B, d/2, N, 16], its feature half to an edge buffer [B, d/2, N*16],
// the gradient of the per-op path's K = 1 neighbour gather, which the caller scatters onto the points with that
// gather's own backward.  dW_fc = sum dlogit . x^T without atomics: the CTAs walk fixed tiles of points in a fixed
// order; after each tile the CTA adds the tile's product into its own [d, d] partial in the workspace (every entry
// owned by one thread), and lfa_wgrad_reduce_kernel sums the partials in CTA order in fp64, rounded once.  The
// partition depends on the shape and on the device's SM count and occupancy, never on timing, so dW_fc is
// bit-identical from run to run.
#include "common.cuh"
#include "lfa_warp.cuh"

#include <algorithm>

namespace ffb6d {

struct LfaTrainParams {
    const float *feature;    // [B, DH, N]   features whose neighbours are gathered
    const void *idx;         // [B, N, 16]
    const float *f_xyz;      // [B, DH, N, 16]
    const float *w_fc;       // [D, D]
    const float *grad_agg;   // [B, D, N]            (backward)
    float *f_agg;            // [B, D, N]            (forward)
    float *grad_edge;        // [B, DH, N * 16]      (backward)
    float *grad_xyz;         // [B, DH, N, 16]       (backward)
    float *part;             // [gridDim.x][D][D]    (backward: one dW_fc partial per CTA)
    long long total;         // B * N
    int N, idx_is_i64;
};

// X[c][k] = x_k[c] of point p = (b, n): the gathered neighbour features (channels < DH) and f_xyz (channels >= DH)
template <int D>
__device__ __forceinline__ void lfa_load_x(const LfaTrainParams &P, long long p, int b, int n, float *X, int lane)
{
    constexpr int DH = D / 2;
    const int k = lane & 15, h = lane >> 4;
    int nb = 0;
    if (lane < LK)
        nb = P.idx_is_i64 ? (int)__ldg(reinterpret_cast<const long long *>(P.idx) + p * LK + lane)
                          : __ldg(reinterpret_cast<const int *>(P.idx) + p * LK + lane);
    const int col = __shfl_sync(0xffffffffu, nb, k);
    const float *fb = P.feature + (size_t)b * DH * P.N + col;
    const float *xb = P.f_xyz + ((size_t)b * DH * P.N + n) * LK + k;
#pragma unroll 4
    for (int c = h; c < DH; c += 2) {
        X[c * LD + k] = __ldg(fb + (size_t)c * P.N);
        X[(DH + c) * LD + k] = __ldg(xb + (size_t)c * P.N * LK);
    }
}

// logits in acc -> softmax over the 16 positions in acc (a lane holds 8, its partner lane ^ 16 the other 8), and
// agg[i] = sum_k X[c][k] * s[c][k] for the lane's channels c = CPL * (lane % 16) + i
template <int D>
__device__ __forceinline__ void lfa_softmax_pool(float (&acc)[D / 16][8], const float *X, int lane, float (&agg)[D / 16])
{
    constexpr int CPL = D / 16;
    const int l = lane & 15, k0 = (lane >> 4) * 8;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
        float mx = acc[i][0];
#pragma unroll
        for (int k = 1; k < 8; ++k) mx = fmaxf(mx, acc[i][k]);
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 16));
        float den = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            acc[i][k] = expf(acc[i][k] - mx);
            den += acc[i][k];
        }
        den += __shfl_xor_sync(0xffffffffu, den, 16);
        float f[8];
        lds_vec<8>(X + (CPL * l + i) * LD + k0, f);
        float num = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            acc[i][k] = acc[i][k] / den;
            num = fmaf(f[k], acc[i][k], num);
        }
        agg[i] = num + __shfl_xor_sync(0xffffffffu, num, 16);
    }
}

template <int D, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
lfa_train_fwd_kernel(const LfaTrainParams P)
{
    constexpr int CPL = D / 16;
    extern __shared__ __align__(16) float sm[];
    float *Wt = sm;                                                    // Wt[j][c] = w_fc[c][j]
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) Wt[(i % D) * D + i / D] = __ldg(P.w_fc + i);
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, l = lane & 15;
    float *X = sm + D * D + (size_t)wid * D * LD;
    for (long long p = (long long)blockIdx.x * WARPS + wid; p < P.total; p += (long long)gridDim.x * WARPS) {
        const int b = (int)(p / P.N), n = (int)(p % P.N);
        lfa_load_x<D>(P, p, b, n, X, lane);
        __syncwarp();
        float acc[CPL][8], agg[CPL];
        warp_mac16<D>(Wt, D, X, lane, acc);
        lfa_softmax_pool<D>(acc, X, lane, agg);
        if (lane < 16)
#pragma unroll
            for (int i = 0; i < CPL; ++i) P.f_agg[((size_t)b * D + CPL * l + i) * P.N + n] = agg[i];
        __syncwarp();
    }
}

// part[c][j] (+)= sum over the tile's nv points w and positions k of G_w[c][k] * X_w[j][k].  Thread t owns the
// entries j = t % D, c = t / D + NG * q: its X row is read once per point with conflict-free 128-bit loads (row
// stride LD), the dlogit rows are warp-wide broadcasts.  `first`: the CTA's first tile stores instead of adding.
template <int D, int WARPS>
__device__ __forceinline__ void lfa_wgrad_tile(const float *tiles, int nv, float *part, bool first)
{
    constexpr int THREADS = WARPS * 32, NG = THREADS / D, E = D / NG, CH = E < 16 ? E : 16;
    static_assert(THREADS % D == 0 && E % CH == 0, "dW_fc entries must split evenly over the CTA");
    const int j = threadIdx.x % D, cg = threadIdx.x / D;
    for (int q0 = 0; q0 < E; q0 += CH) {
        float acc[CH];
#pragma unroll
        for (int q = 0; q < CH; ++q) acc[q] = first ? 0.f : part[(size_t)(cg + NG * (q0 + q)) * D + j];
        for (int w = 0; w < nv; ++w) {
            const float *X = tiles + (size_t)w * 2 * D * LD, *G = X + D * LD;
            float x[16];
            lds_vec<16>(X + j * LD, x);
#pragma unroll
            for (int q = 0; q < CH; ++q) {
                float gq[16];
                lds_vec<16>(G + (cg + NG * (q0 + q)) * LD, gq);
#pragma unroll
                for (int k = 0; k < 16; ++k) acc[q] = fmaf(gq[k], x[k], acc[q]);
            }
        }
#pragma unroll
        for (int q = 0; q < CH; ++q) part[(size_t)(cg + NG * (q0 + q)) * D + j] = acc[q];
    }
}

template <int D, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
lfa_train_bwd_kernel(const LfaTrainParams P)
{
    constexpr int DH = D / 2, CPL = D / 16;
    extern __shared__ __align__(16) float sm[];
    float *Wt = sm;                 // Wt[j][c] = w_fc[c][j]  (logits)
    float *Wn = sm + D * D;         // Wn[c][j] = w_fc[c][j]  (W_fc^T . dlogit)
    float *tiles = Wn + D * D;      // per warp: X [D][LD], then G = dlogit [D][LD]
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
        const float v = __ldg(P.w_fc + i);
        Wt[(i % D) * D + i / D] = v;
        Wn[i] = v;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, l = lane & 15, k0 = (lane >> 4) * 8;
    float *X = tiles + (size_t)wid * 2 * D * LD, *G = X + D * LD;
    float *part = P.part + (size_t)blockIdx.x * D * D;
    const long long ntiles = (P.total + WARPS - 1) / WARPS;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const long long p = t * WARPS + wid;
        if (p < P.total) {
            const int b = (int)(p / P.N), n = (int)(p % P.N);
            lfa_load_x<D>(P, p, b, n, X, lane);
            __syncwarp();
            float s[CPL][8], agg[CPL];
            warp_mac16<D>(Wt, D, X, lane, s);
            lfa_softmax_pool<D>(s, X, lane, agg);
            // dlogit = s * g * (x - f_agg) into G; s becomes g * s, the direct term of dx
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                const int c = CPL * l + i;
                const float g = __ldg(P.grad_agg + ((size_t)b * D + c) * P.N + n);
                float f[8], d[8];
                lds_vec<8>(X + c * LD + k0, f);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    d[k] = s[i][k] * (g * (f[k] - agg[i]));
                    s[i][k] *= g;
                }
                *reinterpret_cast<float4 *>(G + c * LD + k0) = make_float4(d[0], d[1], d[2], d[3]);
                *reinterpret_cast<float4 *>(G + c * LD + k0 + 4) = make_float4(d[4], d[5], d[6], d[7]);
            }
            __syncwarp();
            float dx[CPL][8];
            warp_mac16<D>(Wn, D, G, lane, dx);
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                const int c = CPL * l + i;     // a lane's channels lie all in one half (CPL divides DH)
                float *dst = c < DH ? P.grad_edge + (((size_t)b * DH + c) * P.N + n) * LK
                                    : P.grad_xyz + (((size_t)b * DH + c - DH) * P.N + n) * LK;
                reinterpret_cast<float4 *>(dst + k0)[0] =
                    make_float4(dx[i][0] + s[i][0], dx[i][1] + s[i][1], dx[i][2] + s[i][2], dx[i][3] + s[i][3]);
                reinterpret_cast<float4 *>(dst + k0)[1] =
                    make_float4(dx[i][4] + s[i][4], dx[i][5] + s[i][5], dx[i][6] + s[i][6], dx[i][7] + s[i][7]);
            }
        }
        __syncthreads();
        const int nv = (int)std::min<long long>(WARPS, P.total - t * WARPS);
        lfa_wgrad_tile<D, WARPS>(tiles, nv, part, t == blockIdx.x);
        __syncthreads();
    }
}

// out[e] = sum over the partials i in ascending order of part[i][e], in fp64, rounded once
__global__ void lfa_wgrad_reduce_kernel(const float *__restrict__ part, int nparts, int DD, float *__restrict__ out)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= DD) return;
    double s = 0.0;
    for (int i = 0; i < nparts; ++i) s += (double)part[(size_t)i * DD + e];
    out[e] = (float)s;
}

template <int D, int WARPS>
static size_t lfa_train_fwd_smem() { return sizeof(float) * ((size_t)D * D + (size_t)WARPS * D * LD); }
template <int D, int WARPS>
static size_t lfa_train_bwd_smem() { return sizeof(float) * ((size_t)2 * D * D + (size_t)WARPS * 2 * D * LD); }

// Persistent grid: as many CTAs as fit on the device at once, at most one per tile of WARPS points.  The backward's
// partial count is this grid, so the workspace query and the launch both come through here.  One instantiation per
// kernel: FFB6D_OPTIN_SMEM keeps its once-per-device flag in a static of the function it expands in.
template <int D, int WARPS, bool BWD>
static int lfa_train_grid(long long total, unsigned *grid)
{
    auto kern = BWD ? lfa_train_bwd_kernel<D, WARPS> : lfa_train_fwd_kernel<D, WARPS>;
    const size_t smem = BWD ? lfa_train_bwd_smem<D, WARPS>() : lfa_train_fwd_smem<D, WARPS>();
    FFB6D_OPTIN_SMEM(kern, smem);
    int per_sm = 1;
    FFB6D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, WARPS * 32, smem));
    per_sm = std::max(1, per_sm);
    *grid = (unsigned)std::min<long long>(ceil_div(total, WARPS), (long long)per_sm * num_sms());
    return FFB6D_OK;
}

template <int D, int WARPS>
static int lfa_train_fwd_launch(const LfaTrainParams &P, cudaStream_t st)
{
    unsigned grid = 0;
    const int rc = lfa_train_grid<D, WARPS, false>(P.total, &grid);
    if (rc != FFB6D_OK) return rc;
    lfa_train_fwd_kernel<D, WARPS><<<grid, WARPS * 32, lfa_train_fwd_smem<D, WARPS>(), st>>>(P);
    FFB6D_LAUNCH_OK("lfa_train_fwd_kernel");
    return FFB6D_OK;
}

// Backward CTA shapes: 8 warps for d/2 = 16, 32; 4 for d/2 = 64 (two [128][128] weight copies and 4 warps' tiles
// take 208 KB of shared memory)
template <int D>
constexpr int lfa_bwd_warps() { return D == 128 ? 4 : 8; }

static int lfa_train_bwd_parts(int64_t Dh, long long total, unsigned *grid)
{
    if (Dh == 16) return lfa_train_grid<32, lfa_bwd_warps<32>(), true>(total, grid);
    if (Dh == 32) return lfa_train_grid<64, lfa_bwd_warps<64>(), true>(total, grid);
    return lfa_train_grid<128, lfa_bwd_warps<128>(), true>(total, grid);
}

template <int D>
static int lfa_train_bwd_launch(const LfaTrainParams &P, unsigned grid, float *grad_w, cudaStream_t st)
{
    constexpr int W = lfa_bwd_warps<D>();
    lfa_train_bwd_kernel<D, W><<<grid, W * 32, lfa_train_bwd_smem<D, W>(), st>>>(P);
    FFB6D_LAUNCH_OK("lfa_train_bwd_kernel");
    lfa_wgrad_reduce_kernel<<<(unsigned)ceil_div(D * D, 256), 256, 0, st>>>(P.part, (int)grid, D * D, grad_w);
    FFB6D_LAUNCH_OK("lfa_wgrad_reduce_kernel");
    return FFB6D_OK;
}

static bool lfa_train_sizes_ok(int64_t B, int64_t N) { return B >= 0 && N >= 0 && B < 65536 && N < (1ll << 31); }

}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_lfa_train_fwd(const float *feature, const void *idx, int idx_is_i64, const float *f_xyz,
                                   const float *w_fc, int64_t B, int64_t N, int K, int64_t Dh, float *f_agg,
                                   ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(lfa_train_sizes_ok(B, N), "lfa_train_fwd: bad size B=%lld N=%lld", (long long)B, (long long)N);
    FFB6D_CHECK_ARG(K == LK, "lfa_train_fwd: K=%d, only K = 16 is fused", K);
    FFB6D_CHECK_ARG(Dh == 16 || Dh == 32 || Dh == 64, "lfa_train_fwd: d/2=%lld, fused for 16, 32, 64", (long long)Dh);
    FFB6D_CHECK_ARG(idx_is_i64 == 0 || idx_is_i64 == 1, "lfa_train_fwd: idx_is_i64=%d", idx_is_i64);
    if (B == 0 || N == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(feature && idx && f_xyz && w_fc && f_agg, "lfa_train_fwd: null pointer");
    LfaTrainParams P = {};
    P.feature = feature; P.idx = idx; P.f_xyz = f_xyz; P.w_fc = w_fc; P.f_agg = f_agg;
    P.total = (long long)B * N; P.N = (int)N; P.idx_is_i64 = idx_is_i64;
    cudaStream_t st = (cudaStream_t)stream;
    if (Dh == 16) return lfa_train_fwd_launch<32, 8>(P, st);
    if (Dh == 32) return lfa_train_fwd_launch<64, 8>(P, st);
    return lfa_train_fwd_launch<128, 8>(P, st);
}

extern "C" size_t ffb6d_lfa_train_bwd_workspace_bytes(int64_t B, int64_t N, int K, int64_t Dh)
{
    if (!lfa_train_sizes_ok(B, N) || K != LK || (Dh != 16 && Dh != 32 && Dh != 64) || B == 0 || N == 0) return 0;
    unsigned grid = 0;
    if (lfa_train_bwd_parts(Dh, (long long)B * N, &grid) != FFB6D_OK) return 0;
    return (size_t)grid * 4 * Dh * Dh * sizeof(float);
}

extern "C" int ffb6d_lfa_train_bwd(const float *feature, const void *idx, int idx_is_i64, const float *f_xyz,
                                   const float *w_fc, const float *grad_agg, int64_t B, int64_t N, int K, int64_t Dh,
                                   float *grad_edge, float *grad_f_xyz, float *grad_w_fc, void *workspace,
                                   size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(lfa_train_sizes_ok(B, N), "lfa_train_bwd: bad size B=%lld N=%lld", (long long)B, (long long)N);
    FFB6D_CHECK_ARG(K == LK, "lfa_train_bwd: K=%d, only K = 16 is fused", K);
    FFB6D_CHECK_ARG(Dh == 16 || Dh == 32 || Dh == 64, "lfa_train_bwd: d/2=%lld, fused for 16, 32, 64", (long long)Dh);
    FFB6D_CHECK_ARG(idx_is_i64 == 0 || idx_is_i64 == 1, "lfa_train_bwd: idx_is_i64=%d", idx_is_i64);
    FFB6D_CHECK_ARG(grad_w_fc, "lfa_train_bwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (B == 0 || N == 0) {   // no positions: dW_fc = 0
        FFB6D_CUDA(cudaMemsetAsync(grad_w_fc, 0, sizeof(float) * 4 * Dh * Dh, st));
        return FFB6D_OK;
    }
    FFB6D_CHECK_ARG(feature && idx && f_xyz && w_fc && grad_agg && grad_edge && grad_f_xyz,
                    "lfa_train_bwd: null pointer");
    FFB6D_CHECK_ARG(((uintptr_t)grad_edge | (uintptr_t)grad_f_xyz) % 16 == 0,
                    "lfa_train_bwd: grad_edge and grad_f_xyz must be 16-byte aligned");
    const long long total = (long long)B * N;
    unsigned grid = 0;
    const int rc = lfa_train_bwd_parts(Dh, total, &grid);
    if (rc != FFB6D_OK) return rc;
    const size_t need = (size_t)grid * 4 * Dh * Dh * sizeof(float);
    if (!workspace || workspace_bytes < need || (uintptr_t)workspace % 16 != 0) {
        set_error("lfa_train_bwd: workspace of %zu bytes at %p, need %zu bytes, 16-byte aligned", workspace_bytes,
                  workspace, need);
        return FFB6D_ERR_WORKSPACE;
    }
    LfaTrainParams P = {};
    P.feature = feature; P.idx = idx; P.f_xyz = f_xyz; P.w_fc = w_fc; P.grad_agg = grad_agg;
    P.grad_edge = grad_edge; P.grad_xyz = grad_f_xyz; P.part = (float *)workspace;
    P.total = total; P.N = (int)N; P.idx_is_i64 = idx_is_i64;
    if (Dh == 16) return lfa_train_bwd_launch<32>(P, grid, grad_w_fc, st);
    if (Dh == 32) return lfa_train_bwd_launch<64>(P, grid, grad_w_fc, st);
    return lfa_train_bwd_launch<128>(P, grid, grad_w_fc, st);
}
