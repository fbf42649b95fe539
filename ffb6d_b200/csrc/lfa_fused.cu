// lfa_fused.cu -- RandLA local feature aggregation, one fused kernel per attentive pooling (sm_90a).
//
// Reference (models/RandLA/RandLANet.py:196-250), per point n with its K neighbours idx[n, :]:
//     f_xyz  = mlp1(relative_pos_encoding(xyz, idx))                 [B, d/2, N, K]     (:197-199, 216-223)
//     f_xyz' = mlp2(f_xyz)                  (second pooling only)                       (:207)
//     f_cat  = cat(gather_neighbour(feature, idx), f_xyz or f_xyz')   [B, d, N, K]       (:200-205, 208-212)
//     att    = softmax_K(fc(f_cat));  f_agg = sum_K f_cat * att;  out = mlp(f_agg)      (:243-250)
// as separate torch ops, every [B, *, N, K] tensor a round trip through HBM.  The unfused kernels of this
// repository kept those round trips (56.6 MB/frame of gathers alone, SURVEY.md App. A.2; ~5 GB per 32-frame step
// at level 0 counting all intermediates).  Here ONE warp owns a point: the position encoding of its 16
// neighbours, the 10 -> d/2 (-> d/2) encoding MLP(s), the neighbour feature gather, the d x d attention
// product, the softmax over K, the weighted sum and the output MLP all happen in registers and the warp's
// slice of shared memory; HBM sees xyz, the indices, the [B, d/2, N] feature map and the [B, d_out, N] result.
// Weights (BatchNorm folded, transposed so that a warp reads consecutive output channels) live in shared
// memory for the lifetime of a persistent CTA.
//
// This is dense fp32 FMA work on tiny matrices (d = 32 ... 128) with a softmax in the middle; it runs on the
// CUDA cores: per position 10*d/2 + (d/2)^2 + d^2 multiply-adds, 16 independent accumulators per lane and
// weight element (register reuse across the K neighbours), activations broadcast from shared memory with
// 128-bit loads.  fp32 summation order differs from cuDNN's; results agree with the reference modules to
// < 1e-5 of the output scale (tests/test_gpu_lfa.py).
#include "common.cuh"
#include "lfa_warp.cuh"

#include <algorithm>

namespace ffb6d {

__device__ __forceinline__ float leaky(float v, float slope) { return v > 0.f ? v : v * slope; }

// out[c][k] = leaky(scale[c] * (Wt^T in)[c][k] + shift[c]) for c < COUT, k < 16 (shared memory, row stride LD)
template <int COUT>
__device__ __forceinline__ void warp_dense16(const float *__restrict__ Wt, int cin, const float *__restrict__ in,
                                             float *__restrict__ out, const float *__restrict__ scale,
                                             const float *__restrict__ shift, float slope, int lane)
{
    constexpr int CPL = COUT / 16;
    float acc[CPL][8];
    warp_mac16<COUT>(Wt, cin, in, lane, acc);
    const int l = lane & 15, k0 = (lane >> 4) * 8;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
        const int c = CPL * l + i;
        const float sc = scale[c], sh = shift[c];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            float4 v;
            v.x = leaky(fmaf(acc[i][4 * q], sc, sh), slope); v.y = leaky(fmaf(acc[i][4 * q + 1], sc, sh), slope);
            v.z = leaky(fmaf(acc[i][4 * q + 2], sc, sh), slope); v.w = leaky(fmaf(acc[i][4 * q + 3], sc, sh), slope);
            *reinterpret_cast<float4 *>(out + c * LD + k0 + 4 * q) = v;
        }
    }
}

struct LfaParams {
    const float *xyz;        // [B, N, 3]
    const void *idx;         // [B, N, 16]
    const float *feature;    // [B, DH, N]   features whose neighbours are gathered
    const float *w_x1, *s_x1, *t_x1;   // mlp1: [DH, 10], folded BN scale / shift [DH]
    const float *w_x2, *s_x2, *t_x2;   // mlp2: [DH, DH] or null
    const float *w_fc;                 // [D, D]
    const float *w_o, *s_o, *t_o;      // output mlp: [DO, D], [DO]
    float *out;              // [B, DO, N]
    long long total;         // B * N
    int N, idx_is_i64, DO;
    float slope;
};

// D = d = 2 * DH channels of the concatenated neighbourhood features; WARPS warps (= points in flight) per CTA
template <int D, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
lfa_att_pool_fused_kernel(const LfaParams P)
{
    constexpr int DH = D / 2;
    extern __shared__ __align__(16) float sm[];
    // ---- CTA-resident weights, transposed [in][out]
    float *Wfc = sm;                           // [D][D]
    float *Wo = Wfc + D * D;                   // [D][DO]  (DO <= D)
    float *Wx1 = Wo + D * D;                   // [10][DH]
    float *Wx2 = Wx1 + 10 * DH;                // [DH][DH]
    float *aff = Wx2 + DH * DH;                // s_x1, t_x1, s_x2, t_x2 [DH each], s_o, t_o [D each]
    float *warp_mem = aff + 4 * DH + 2 * D;
    const int DO = P.DO;
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) Wfc[(i % D) * D + i / D] = __ldg(P.w_fc + i);          // Wfc[j][c] = w[c][j]
    for (int i = threadIdx.x; i < DO * D; i += blockDim.x) Wo[(i % D) * DO + i / D] = __ldg(P.w_o + i);           // Wo[j][o]
    for (int i = threadIdx.x; i < DH * 10; i += blockDim.x) Wx1[(i % 10) * DH + i / 10] = __ldg(P.w_x1 + i);
    if (P.w_x2)
        for (int i = threadIdx.x; i < DH * DH; i += blockDim.x) Wx2[(i % DH) * DH + i / DH] = __ldg(P.w_x2 + i);
    for (int i = threadIdx.x; i < DH; i += blockDim.x) {
        aff[i] = __ldg(P.s_x1 + i);
        aff[DH + i] = __ldg(P.t_x1 + i);
        aff[2 * DH + i] = P.w_x2 ? __ldg(P.s_x2 + i) : 1.f;
        aff[3 * DH + i] = P.w_x2 ? __ldg(P.t_x2 + i) : 0.f;
    }
    for (int i = threadIdx.x; i < DO; i += blockDim.x) {
        aff[4 * DH + i] = __ldg(P.s_o + i);
        aff[4 * DH + D + i] = __ldg(P.t_o + i);
    }
    __syncthreads();
    // ---- per-warp scratch: R [10][16] (padded to 12 rows), X [DH][16], FC [D][16] (gathered | encoded), A [D]
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    constexpr int WARP_FLOATS = 12 * LD + DH * LD + D * LD + D;
    float *R = warp_mem + (size_t)wid * WARP_FLOATS;
    float *X = R + 12 * LD;
    float *FC = X + DH * LD;
    float *A = FC + D * LD;
    const float slope = P.slope;
    for (long long p = (long long)blockIdx.x * WARPS + wid; p < P.total; p += (long long)gridDim.x * WARPS) {
        const int b = (int)(p / P.N), n = (int)(p % P.N);
        // ---- relative position encoding of the 16 neighbours (RandLANet.py:216-223), one neighbour per lane pair
        int nb = 0;
        if (lane < LK) {
            nb = P.idx_is_i64 ? (int)__ldg(reinterpret_cast<const long long *>(P.idx) + p * LK + lane)
                              : __ldg(reinterpret_cast<const int *>(P.idx) + p * LK + lane);
            const float *pc = P.xyz + (size_t)p * 3, *pn = P.xyz + ((size_t)b * P.N + nb) * 3;
            const float cx = __ldg(pc), cy = __ldg(pc + 1), cz = __ldg(pc + 2);
            const float nx = __ldg(pn), ny = __ldg(pn + 1), nz = __ldg(pn + 2);
            const float dx = __fsub_rn(cx, nx), dy = __fsub_rn(cy, ny), dz = __fsub_rn(cz, nz);
            const float ss = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            R[0 * LD + lane] = __fsqrt_rn(ss);
            R[1 * LD + lane] = dx; R[2 * LD + lane] = dy; R[3 * LD + lane] = dz;
            R[4 * LD + lane] = cx; R[5 * LD + lane] = cy; R[6 * LD + lane] = cz;
            R[7 * LD + lane] = nx; R[8 * LD + lane] = ny; R[9 * LD + lane] = nz;
        }
        // ---- neighbours' features: FC[c][k] = feature[b, c, idx[k]]  (lane = (k, half), channels c = half + 2i)
        {
            const int k = lane & 15, h = lane >> 4;
            const int col = __shfl_sync(0xffffffffu, nb, k);
            const float *fb = P.feature + (size_t)b * DH * P.N + col;
#pragma unroll 4
            for (int c = h; c < DH; c += 2) FC[c * LD + k] = __ldg(fb + (size_t)c * P.N);
        }
        __syncwarp();
        // ---- encoding MLP(s): f_xyz = mlp1(R) [-> mlp2], written as the second half of FC
        if (P.w_x2) {
            warp_dense16<DH>(Wx1, 10, R, X, aff, aff + DH, slope, lane);
            __syncwarp();
            warp_dense16<DH>(Wx2, DH, X, FC + DH * LD, aff + 2 * DH, aff + 3 * DH, slope, lane);
        } else {
            warp_dense16<DH>(Wx1, 10, R, FC + DH * LD, aff, aff + DH, slope, lane);
        }
        __syncwarp();
        // ---- attention scores fc(f_cat) [D][16], softmax over the neighbours, weighted sum: a lane holds CPL channels x 8
        // positions in registers; the other 8 positions of a channel sit in the partner lane (lane ^ 16)
        {
            constexpr int CPL = D / 16;
            float acc[CPL][8];
            warp_mac16<D>(Wfc, D, FC, lane, acc);
            const int l = lane & 15, k0 = (lane >> 4) * 8;
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                const int c = CPL * l + i;
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
                lds_vec<8>(FC + c * LD + k0, f);
                float num = 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k) num += f[k] * (acc[i][k] / den);
                num += __shfl_xor_sync(0xffffffffu, num, 16);
                if (lane < 16) A[c] = num;
            }
        }
        __syncwarp();
        // ---- output MLP on the pooled vector: out[o] = leaky(s * sum_j Wo[j][o] * A[j] + t)
        for (int o = lane; o < DO; o += 32) {
            float acc = 0.f;
#pragma unroll 8
            for (int j = 0; j < D; ++j) acc = fmaf(Wo[j * DO + o], A[j], acc);
            P.out[((size_t)b * DO + o) * P.N + n] = leaky(fmaf(acc, aff[4 * DH + o], aff[4 * DH + D + o]), slope);
        }
        __syncwarp();
    }
}

template <int D, int WARPS>
static size_t lfa_smem_bytes()
{
    constexpr int DH = D / 2;
    return sizeof(float) * ((size_t)2 * D * D + 10 * DH + DH * DH + 4 * DH + 2 * D + (size_t)WARPS * (12 * LD + DH * LD + D * LD + D));
}

template <int D, int WARPS>
static int lfa_launch(const LfaParams &P, cudaStream_t st)
{
    auto kern = lfa_att_pool_fused_kernel<D, WARPS>;
    const size_t smem = lfa_smem_bytes<D, WARPS>();
    FFB6D_OPTIN_SMEM(kern, smem);
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, WARPS * 32, smem);
    per_sm = std::max(1, per_sm);
    const long long want = ceil_div(P.total, WARPS);
    const unsigned grid = (unsigned)std::min<long long>(want, (long long)per_sm * num_sms());   // persistent CTAs
    kern<<<grid, WARPS * 32, smem, st>>>(P);
    FFB6D_LAUNCH_OK("lfa_att_pool_fused_kernel");
    return FFB6D_OK;
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_lfa_att_pool_fused(const float *xyz, const void *idx, int idx_is_i64, const float *feature,
                                        const float *w_x1, const float *scale_x1, const float *shift_x1, const float *w_x2,
                                        const float *scale_x2, const float *shift_x2, const float *w_fc, const float *w_out,
                                        const float *scale_out, const float *shift_out, int64_t B, int64_t N, int K, int64_t Dh,
                                        int64_t Do, float negative_slope, float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && N >= 0 && B < 65536 && N < (1ll << 31), "lfa_att_pool_fused: bad size");
    FFB6D_CHECK_ARG(K == LK, "lfa_att_pool_fused: K=%d, only K = 16 is fused", K);
    FFB6D_CHECK_ARG(Dh == 16 || Dh == 32 || Dh == 64, "lfa_att_pool_fused: d/2=%lld, fused for 16, 32, 64", (long long)Dh);
    FFB6D_CHECK_ARG(Do >= 1 && Do <= 2 * Dh, "lfa_att_pool_fused: d_out=%lld outside [1, d]", (long long)Do);
    if (B == 0 || N == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(xyz && idx && feature && w_x1 && scale_x1 && shift_x1 && w_fc && w_out && scale_out && shift_out && out &&
                        (!w_x2 || (scale_x2 && shift_x2)),
                    "lfa_att_pool_fused: null pointer");
    LfaParams P;
    P.xyz = xyz; P.idx = idx; P.feature = feature;
    P.w_x1 = w_x1; P.s_x1 = scale_x1; P.t_x1 = shift_x1;
    P.w_x2 = w_x2; P.s_x2 = scale_x2; P.t_x2 = shift_x2;
    P.w_fc = w_fc; P.w_o = w_out; P.s_o = scale_out; P.t_o = shift_out;
    P.out = out; P.total = (long long)B * N; P.N = (int)N; P.idx_is_i64 = idx_is_i64; P.DO = (int)Do; P.slope = negative_slope;
    cudaStream_t st = (cudaStream_t)stream;
    if (Dh == 16) return lfa_launch<32, 8>(P, st);
    if (Dh == 32) return lfa_launch<64, 8>(P, st);
    return lfa_launch<128, 4>(P, st);
}
