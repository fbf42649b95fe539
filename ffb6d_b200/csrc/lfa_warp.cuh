// lfa_warp.cuh -- the warp-per-point building blocks shared by the attentive-pooling kernels: lfa_fused.cu
// (inference, one kernel per pooling) and lfa_train.cu (training, forward and recomputing backward).
#pragma once
#include "common.cuh"

namespace ffb6d {

constexpr int LK = 16;   // neighbours per point (the only K FFB6D uses, datasets/ycb/ycb_dataset.py:276)

constexpr int LD = 20;   // shared-memory row stride of a [channels][16 positions] tile: 80 bytes, so that the 128-bit
                         // row accesses of lanes one row apart fall into distinct banks (a 64-byte stride is 4-way conflicted)

template <int N>
__device__ __forceinline__ void lds_vec(const float *p, float (&w)[N])   // N consecutive floats, N-float aligned
{
    if constexpr (N == 1) {
        w[0] = p[0];
    } else if constexpr (N == 2) {
        const float2 v = *reinterpret_cast<const float2 *>(p);
        w[0] = v.x; w[1] = v.y;
    } else {
#pragma unroll
        for (int q = 0; q < N / 4; ++q) {
            const float4 v = *reinterpret_cast<const float4 *>(p + 4 * q);
            w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
        }
    }
}

// acc[i][k] = sum_j Wt[j][CPL*l + i] * in[j][8*half + k]: the warp's 16 x COUT product, lane (l = lane % 16, half =
// lane / 16) owning CPL = COUT / 16 consecutive output channels and 8 of the 16 positions.  Per j: two broadcast
// 128-bit activation loads and ONE weight load of CPL floats feed 8 * CPL FMAs.
template <int COUT>
__device__ __forceinline__ void warp_mac16(const float *__restrict__ Wt, int cin, const float *__restrict__ in, int lane,
                                           float (&acc)[COUT / 16][8])
{
    constexpr int CPL = COUT / 16;
    const int l = lane & 15, k0 = (lane >> 4) * 8;
#pragma unroll
    for (int i = 0; i < CPL; ++i)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[i][k] = 0.f;
#pragma unroll 2
    for (int j = 0; j < cin; ++j) {
        float f[8], w[CPL];
        lds_vec<8>(in + j * LD + k0, f);
        lds_vec<CPL>(Wt + j * COUT + CPL * l, w);
#pragma unroll
        for (int i = 0; i < CPL; ++i)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[i][k] = fmaf(w[i], f[k], acc[i][k]);
    }
}

}  // namespace ffb6d
