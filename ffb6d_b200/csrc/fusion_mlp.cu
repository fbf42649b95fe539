// fusion_mlp.cu -- the 1x1 fusion MLP of FFB6D on Hopper tensor cores (sm_90a, wgmma).
//
// Reference: pt_utils.Conv2d(in, out, kernel_size=(1,1), bn=True) = conv(bias=False) ->
// BatchNorm2d -> ReLU (models/pytorch_utils.py:75-129, 168-201), 28 instances built at
// models/ffb6d.py:55-80, 104-129 and applied to torch.cat((a, b), dim=1) (:246-262, 282-298).
// With frozen (eval) statistics the layer is, per frame,
//     out[co, p] = relu( scale[co] * sum_ci W[co, ci] * X[ci, p] + shift[co] ),   X = [X1; X2]
// i.e. a dense GEMM D[Co x P] = W[Co x Ci] * X[Ci x P] with a per-row affine + ReLU epilogue.
//
// Kernels in this file (DESIGN.md 4.4):
//   fusion_mlp_packed_kernel  the product path: weights pre-split once (ffb6d_fusion_mlp_pack) and
//                             fetched by bulk-async copies (TMA engine, mbarrier completion), the
//                             activations staged by the CTA's threads
//   fusion_wgrad_kernel       the weight gradient of training, same tile machinery
//
// All of them fuse the concat (two K ranges read from two tensors), the GEMM, BN and ReLU:
//   * wgmma.mma_async m64n128k8 .tf32, two warpgroups per CTA (rows 0-63 and 64-127 of a 128 x 128
//     tile), accumulators in registers
//   * fp32 fidelity through 3xTF32: every fp32 operand is split into hi = tf32(x) and
//     lo = tf32(x - hi) while it is staged, and D += Ahi*Bhi + Alo*Bhi + Ahi*Blo (the dropped lo*lo
//     term is 2^-22 relative): results agree with the fp32 cuDNN path to ~1e-6 relative, inside the
//     1e-5 contract of BASELINE.json
//   * operands are staged into the canonical K-major no-swizzle layout: 8-row x 16-byte core
//     matrices, 128 B between 8-row groups (SBO), 2048 B between 16-byte K chunks (LBO); X is
//     transposed on the fly (it is point-major in memory)
//   * three stages and one CTA barrier per k-tile: the MMAs of k-tile kt run asynchronously while
//     the threads load k-tile kt + 1 from global memory; a stage is rewritten only after every
//     warpgroup has waited for the MMAs that read it (wgmma.wait_group 1 before the barrier)
//   * the tensor core's fp32 accumulation truncates, a bias that grows with every MMA into the same
//     accumulator (chunks of 128 = 48 MMAs: ~4e-6 relative, enough to show in whole-network training
//     gradients); K is therefore accumulated one k-tile (12 MMAs) at a time and every chunk is added
//     into round-to-nearest fp32 register sums
//   * epilogue: scale/shift/activation in registers, stores along the point axis (NCHW output)
#include "common.cuh"
#include "psp.cuh"

#include <algorithm>
#include <stdlib.h>

namespace ffb6d {

constexpr int TM = 128, TN = 128, TK = 32;            // CTA tile
constexpr int CHUNK_BYTES = TM * 16;                  // one 16-byte K chunk of all 128 rows
constexpr int TILE_BYTES = (TK / 4) * CHUNK_BYTES;    // 16 KB
constexpr int STAGE_BYTES = 4 * TILE_BYTES;           // A_hi, A_lo, B_hi, B_lo
constexpr int NST = 3;                                // stages
constexpr int CH = 1;                                 // k-tiles per accumulation chunk (K = 32, 12 MMAs)
constexpr int MLP_THREADS = 256;                      // two warpgroups
constexpr int MLP_SMEM = NST * STAGE_BYTES + 64;      // stages + mbarriers: 192 KB, one CTA per SM

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// round-to-nearest (ties away) to TF32's 10-bit mantissa with two full-rate integer ops; identical to
// cvt.rna.tf32.f32 for finite inputs below (2 - 2^-11) * 2^127 in magnitude (that conversion runs on the quarter-rate
// conversion pipe).  Above, in the bit patterns 0x7F7FF000 .. 0x7F7FFFFF of either sign, the rounding carries into the
// exponent and gives +-inf.
__device__ __forceinline__ float to_tf32(float x)
{
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}

// to_tf32 with the top band truncated instead, so that a finite x has a finite tf32: the sum is clamped to 0x7F7FFFFF
// as an int32 (the positive band) and to 0xFF7FFFFF as a uint32 (the negative band); each clamp leaves the other sign
// alone, and below the band neither fires.  ptxas fuses the add and the int32 clamp into one VIADDMNMX, so this costs
// one integer op more than to_tf32.
__device__ __forceinline__ float to_tf32_finite(float x)
{
    const uint32_t r = __float_as_uint(x) + 0x1000u;
    return __uint_as_float(min((uint32_t)min((int)r, 0x7F7FFFFF), 0xFF7FFFFFu) & 0xFFFFE000u);
}

// x = hi + lo, to 2^-22 |x| + 2^-137 for every finite x (oracle/tf32_oracle.py restates it bit for bit).  Only hi needs
// the truncated band: |x - hi| <= 2^-10 |x| never reaches it.  For a non-finite x, to_tf32_finite gives a finite value
// or +-0 (for NaNs near 0x7FFFFFFF, the NaN the GPU's own arithmetic produces, the integer add wraps), and x - hi is
// NaN or +-inf: an upstream NaN would vanish from the layer.  hi = fma(x - hi, 0, hi) restores it (one FMA-pipe op;
// hi itself for finite x), so a NaN input comes out NaN, and so does +-inf.
__device__ __forceinline__ void split1(float x, float &hi, float &lo)
{
    const float h = to_tf32_finite(x), d = x - h;
    lo = to_tf32(d);
    hi = __fmaf_rn(d, 0.f, h);
}

__device__ __forceinline__ void split4(const float4 v, float4 &hi, float4 &lo)
{
    split1(v.x, hi.x, lo.x);
    split1(v.y, hi.y, lo.y);
    split1(v.z, hi.z, lo.z);
    split1(v.w, hi.w, lo.w);
}

// K-major, no-swizzle (layout type 0) wgmma shared-memory matrix descriptor: start address, LBO = next
// 16-byte K chunk, SBO = next 8-row group, all in 16-byte units
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr)
{
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(CHUNK_BYTES >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
}

// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, fp32 accumulate, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t a, uint64_t b, int accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
        "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, "
        "%43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
}

// keeps the compiler from moving reads or writes of the accumulators across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(float (&d)[64])
{
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int N>
__device__ __forceinline__ void wgmma_wait()
{
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// the 12 MMAs of one k-tile (4 k-steps x 3 split products) for warpgroup `wg` (rows 64 wg .. 64 wg + 63),
// committed as one group; `first`: the k-tile opens an accumulation chunk.  The small lo products go first,
// while the accumulator is small too, so that only the 4 hi * hi MMAs truncate at the full magnitude.
__device__ __forceinline__ void mma_ktile(float (&d)[64], uint32_t s0, int wg, bool first)
{
    const uint64_t a_hi = gmma_desc(s0 + wg * 8 * 128), a_lo = gmma_desc(s0 + TILE_BYTES + wg * 8 * 128);
    const uint64_t b_hi = gmma_desc(s0 + 2 * TILE_BYTES), b_lo = gmma_desc(s0 + 3 * TILE_BYTES);
    acc_fence(d);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int j = 0; j < TK / 8; ++j) {
        const uint64_t off = (uint64_t)(j * ((2 * CHUNK_BYTES) >> 4));
        wgmma_tf32(d, a_lo + off, b_hi + off, (first && j == 0) ? 0 : 1);
        wgmma_tf32(d, a_hi + off, b_lo + off, 1);
    }
#pragma unroll
    for (int j = 0; j < TK / 8; ++j) {
        const uint64_t off = (uint64_t)(j * ((2 * CHUNK_BYTES) >> 4));
        wgmma_tf32(d, a_hi + off, b_hi + off, 1);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    acc_fence(d);
}

// waits for every MMA of this warpgroup and adds the finished chunk into the round-to-nearest sums
__device__ __forceinline__ void drain(float (&d)[64], float (&sum)[64])
{
    wgmma_wait<0>();
    acc_fence(d);
#pragma unroll
    for (int i = 0; i < 64; ++i) sum[i] = __fadd_rn(sum[i], d[i]);
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t done = 0;
    for (int spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, P1;\n\t}\n"
            : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1 << 26)) __trap();   // never hang the GPU on a protocol bug
    }
}

// ===================================================================== packed-weight kernel
// The weights are constants at inference: their hi/lo split is computed once
// (fusion_mlp_pack_kernel) and written in exactly the shared-memory image the A operand needs, one
// contiguous 32 KB block per (128-row tile, 32-column k-tile): [A_hi | A_lo], each 8 chunks x 128
// rows x 16 B.  Thread 0 brings the block of k-tile kt + 1 with one cp.async.bulk while the MMAs of
// k-tile kt run; its mbarrier counts the transaction bytes.
constexpr int PACK_BLOCK_BYTES = 2 * TILE_BYTES;                 // A_hi + A_lo of one k-tile

// Optional extras of the epilogue (all null / 0 for the plain layer):
//   addend [B, NA, Co] (channels-last) + idx [B, P]: out = act(scale * (W x + addend[b, idx[b, p], :]) + shift)
//   out_nsc: the result is stored channels-last, [B, P, Co]
struct MlpEpilogue {
    const float *addend;
    const void *idx;
    int NA;
    int idx_is_i64;
    int out_nsc;
};

__global__ void __launch_bounds__(256)
fusion_mlp_pack_kernel(const float *__restrict__ w, int Co, int Ci, int nk, int nblocks, float4 *__restrict__ packed)
{
    const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one (block, chunk, row) each
    if (o >= (long long)nblocks * 1024) return;
    const int blk = (int)(o >> 10), r = (int)(o & 1023), c = r >> 7, m = r & 127;
    const int gm = (blk / nk) * TM + m, gk = (blk % nk) * TK + 4 * c;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gm < Co) {
        const float *src = w + (size_t)gm * Ci + gk;
        if (gk + 0 < Ci) v.x = __ldg(src + 0);
        if (gk + 1 < Ci) v.y = __ldg(src + 1);
        if (gk + 2 < Ci) v.z = __ldg(src + 2);
        if (gk + 3 < Ci) v.w = __ldg(src + 3);
    }
    float4 hi, lo;
    split4(v, hi, lo);
    float4 *dst = packed + (size_t)blk * (PACK_BLOCK_BYTES / 16);
    dst[r] = hi;
    dst[TILE_BYTES / 16 + r] = lo;
}

// The product of the packed-weight kernels (fusion_mlp_packed_kernel here, and the PSP head's kernels of psp.cu):
// sum = this warpgroup's 64 x 128 part of the CTA tile W[m0 .., :] * [X1; X2][:, n0 ..] of one frame, rounded as
// described at the top of the file.  xb1 / xb2: the frame's inputs (NCHW, [C1, P] and [C2, P]); wsrc: the packed
// blocks of the CTA's 128-row tile; vec: 16-byte vector loads are allowed (P % 4 == 0, inputs aligned).  Uses the
// whole dynamic shared memory (MLP_SMEM); a caller that reuses it afterwards synchronises the CTA first.
__device__ __forceinline__ void packed_mainloop(unsigned char *smem, const float *__restrict__ xb1, int C1,
                                                const float *__restrict__ xb2, int C2,
                                                const unsigned char *__restrict__ wsrc, int P, int n0, bool vec,
                                                float (&sum)[64])
{
    uint64_t *full_a = reinterpret_cast<uint64_t *>(smem + NST * STAGE_BYTES);
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int Ci = C1 + C2;
    const int nk = (Ci + TK - 1) / TK;
    auto fetch_a = [&](int kt) {
        const int st = kt % NST;
        const uint32_t bar = smem_u32(full_a + st);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(PACK_BLOCK_BYTES) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"(smem_u32(smem + st * STAGE_BYTES)), "l"(wsrc + (size_t)kt * PACK_BLOCK_BYTES),
                        "r"(PACK_BLOCK_BYTES), "r"(bar) : "memory");
    };
    if (tid == 0) {
        for (int i = 0; i < NST; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(full_a + i)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) fetch_a(0);

    // X tile (32 k x 128 n): warp -> K chunk kg (4 k rows), lane -> 4 n (128-bit loads); a thread ends up
    // with whole 16-byte (n; k..k+3) slots of the K-major layout
    const int kg = wid, nl = 4 * lane;
    // fast path: whole tile inside the tensors, vector loads, and a 4-row K chunk never straddles the
    // concat boundary -> one base pointer per tile, four loads at a row stride
    const bool fast = vec && ((C1 & 3) == 0) && (n0 + TN <= P);
    auto load_b = [&](int kt, float4 (&rb)[4]) {
        const int gk0 = kt * TK + 4 * kg;
        if (fast && gk0 + 3 < Ci) {
            const float *p0 = ((gk0 < C1) ? xb1 + (size_t)gk0 * P : xb2 + (size_t)(gk0 - C1) * P) + (n0 + nl);
#pragma unroll
            for (int j = 0; j < 4; ++j) rb[j] = __ldg(reinterpret_cast<const float4 *>(p0 + (size_t)j * P));
            return;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int gk = gk0 + j, gn = n0 + nl;
            float e[4] = {0.f, 0.f, 0.f, 0.f};
            if (gk < Ci) {
                const float *row = (gk < C1) ? xb1 + (size_t)gk * P : xb2 + (size_t)(gk - C1) * P;
                if (vec && gn + 3 < P) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(row + gn));
                    e[0] = v.x;
                    e[1] = v.y;
                    e[2] = v.z;
                    e[3] = v.w;
                } else {
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        if (gn + u < P) e[u] = __ldg(row + gn + u);
                }
            }
            rb[j] = make_float4(e[0], e[1], e[2], e[3]);
        }
    };
    auto store_b = [&](int st, const float4 (&rb)[4]) {
        unsigned char *sB_hi = smem + st * STAGE_BYTES + 2 * TILE_BYTES, *sB_lo = sB_hi + TILE_BYTES;
        unsigned char *bh = sB_hi + kg * CHUNK_BYTES + nl * 16, *bl = sB_lo + kg * CHUNK_BYTES + nl * 16;
        const float4 t0 = make_float4(rb[0].x, rb[1].x, rb[2].x, rb[3].x);   // n = nl + 0, k = 4kg .. 4kg+3
        const float4 t1 = make_float4(rb[0].y, rb[1].y, rb[2].y, rb[3].y);
        const float4 t2 = make_float4(rb[0].z, rb[1].z, rb[2].z, rb[3].z);
        const float4 t3 = make_float4(rb[0].w, rb[1].w, rb[2].w, rb[3].w);
        float4 hi, lo;
#pragma unroll
        for (int i = 0; i < 4; ++i) {   // rotated slots: every quarter-warp covers all 32 banks
            const int x = (i + (lane >> 1)) & 3;
            const float4 tx = (x == 0) ? t0 : (x == 1) ? t1 : (x == 2) ? t2 : t3;
            split4(tx, hi, lo);
            *reinterpret_cast<float4 *>(bh + 16 * x) = hi;
            *reinterpret_cast<float4 *>(bl + 16 * x) = lo;
        }
    };

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = sum[i] = 0.f;
    float4 rb[4];
    load_b(0, rb);
    for (int kt = 0; kt < nk; ++kt) {
        const int st = kt % NST;
        store_b(st, rb);   // stage st was last read by the MMAs of k-tile kt - 3: complete (see the loop end)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the MMA
        __syncthreads();   // every warpgroup has passed its wait for the MMAs of k-tile kt - 2
        if (tid == 0 && kt + 1 < nk) fetch_a(kt + 1);   // into the stage of k-tile kt - 2
        if (kt + 1 < nk) load_b(kt + 1, rb);            // in flight during this k-tile's MMAs
        mbar_wait(smem_u32(full_a + st), (uint32_t)((kt / NST) & 1));
        if (kt % CH == 0 && kt > 0) drain(acc, sum);
        mma_ktile(acc, smem_u32(smem + st * STAGE_BYTES), wg, kt % CH == 0);
        wgmma_wait<1>();   // the MMAs of k-tile kt - 1 are done
    }
    drain(acc, sum);
}

__global__ void __launch_bounds__(MLP_THREADS, 1)
fusion_mlp_packed_kernel(const float *__restrict__ x1, int C1, const float *__restrict__ x2, int C2,
                         const unsigned char *__restrict__ wpack, const float *__restrict__ scale,
                         const float *__restrict__ shift, float *__restrict__ out, int Co, int P, int act,
                         float slope, MlpEpilogue ep)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int b = blockIdx.z, m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
    const int nk = (C1 + C2 + TK - 1) / TK;
    const float *xb1 = x1 + (size_t)b * C1 * P;
    const float *xb2 = x2 ? x2 + (size_t)b * C2 * P : nullptr;
    const bool vec = ((P & 3) == 0) && ((reinterpret_cast<uintptr_t>(xb1) & 15) == 0) &&
                     (!xb2 || (reinterpret_cast<uintptr_t>(xb2) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    float sum[64];
    packed_mainloop(smem, xb1, C1, xb2, C2, wpack + (size_t)blockIdx.y * nk * PACK_BLOCK_BYTES, P, n0, vec, sum);

    // accumulator fragment of m64n128: register 4i + 2h + c holds row 16 w + lane / 4 + 8 h,
    // column 8 i + 2 (lane % 4) + c of the warpgroup's 64 x 128 tile
    const int row0 = m0 + 64 * wg + 16 * (wid & 3) + (lane >> 2), col0 = n0 + 2 * (lane & 3);
    const int *idx32 = (ep.addend && !ep.idx_is_i64) ? reinterpret_cast<const int *>(ep.idx) + (size_t)b * P : nullptr;
    const long long *idx64 = (ep.addend && ep.idx_is_i64) ? reinterpret_cast<const long long *>(ep.idx) + (size_t)b * P : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int gm = row0 + 8 * h;
        if (gm >= Co) continue;
        const float sc = __ldg(scale + gm), sh = __ldg(shift + gm);
        float *orow = out + ((size_t)b * Co + gm) * P;
        // optional epilogue extras (MlpEpilogue): a gathered addend in front of the affine -- the second half
        // of a concat-GEMM restructured as W1*x + (W2*p)[idx] -- and a channels-last store
        const float *add_row = ep.addend ? ep.addend + (size_t)b * ep.NA * Co + gm : nullptr;
        float *ocol = ep.out_nsc ? out + (size_t)b * P * Co + gm : nullptr;
#pragma unroll
        for (int i = 0; i < TN / 8; ++i) {
            const int gn = col0 + 8 * i;
            float y[2] = {sum[4 * i + 2 * h], sum[4 * i + 2 * h + 1]};
            if (add_row) {   // the addend row is channels-last: the 8 rows of a warp read 32 contiguous bytes
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int a = (gn + u < P) ? (idx32 ? __ldg(idx32 + gn + u) : (int)__ldg(idx64 + gn + u)) : 0;
                    y[u] = __fadd_rn(y[u], __ldg(add_row + (size_t)a * Co));
                }
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                y[u] = __fadd_rn(__fmul_rn(y[u], sc), sh);
                if (act == 1) y[u] = max_nan(y[u], 0.f);
                else if (act == 2) y[u] = (y[u] > 0.f) ? y[u] : __fmul_rn(y[u], slope);
            }
            if (ocol) {
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (gn + u < P) ocol[(size_t)(gn + u) * Co] = y[u];
            } else if (vec && gn + 1 < P) {
                *reinterpret_cast<float2 *>(orow + gn) = make_float2(y[0], y[1]);
            } else {
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (gn + u < P) orow[gn + u] = y[u];
            }
        }
    }
}

// ===================================================================== PSP head (eval, DESIGN.md 4.17)
// Bottleneck of PSPModule restructured (models/cnn/pspnet.py:24-31):
//     out = relu( W_f * f + bias + sum_s up_s(T_s) ),   T_s = (W_s C_s) pool_s(f),   s = 1, 2, 3, 6
// The product W_f * f is the packed main loop over the C feature channels only; the epilogue adds the
// align_corners=False bilinear taps of the four prior tables T (channels-last, [B, s*s, Co] per scale, one after the
// other), the bias and the ReLU.  The upsampled priors and the 5C-channel concat are never written.
constexpr int PSP_NS = 4;
__constant__ int c_psp_size[PSP_NS] = {1, 2, 3, 6};
__constant__ int c_psp_off[PSP_NS] = {0, 1, 5, 14};   // first bin of each scale among the 50

// psp_tap (psp.cuh): one output coordinate's two source taps along one axis, shared with the adjoint in psp.cu

__global__ void __launch_bounds__(MLP_THREADS, 1)
psp_bottleneck_kernel(const float *__restrict__ x, int C, const unsigned char *__restrict__ wpack,
                      const float *__restrict__ bias, const float *__restrict__ table, float *__restrict__ out, int Co,
                      int H, int W, int B)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int b = blockIdx.z, m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
    const int P = H * W;
    const int nk = (C + TK - 1) / TK;
    const float *xb = x + (size_t)b * C * P;
    const bool vec = ((P & 3) == 0) && ((reinterpret_cast<uintptr_t>(xb) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    float sum[64];
    packed_mainloop(smem, xb, C, nullptr, 0, wpack + (size_t)blockIdx.y * nk * PACK_BLOCK_BYTES, P, n0, vec, sum);
    __syncthreads();   // both warpgroups are past their last MMA: the stages are free

    // taps of every output row (scale-major, [4][H]) and column ([4][W])
    PspTap *tap_y = reinterpret_cast<PspTap *>(smem), *tap_x = tap_y + PSP_NS * H;
    for (int t = tid; t < PSP_NS * (H + W); t += MLP_THREADS) {
        if (t < PSP_NS * H)
            tap_y[t] = psp_tap(t % H, H, c_psp_size[t / H]);
        else
            tap_x[t - PSP_NS * H] = psp_tap((t - PSP_NS * H) % W, W, c_psp_size[(t - PSP_NS * H) / W]);
    }
    __syncthreads();

    const int row0 = m0 + 64 * wg + 16 * (wid & 3) + (lane >> 2), col0 = n0 + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < TN / 8; ++i) {
        const int gn0 = col0 + 8 * i;
        if (gn0 >= P) continue;
        // the two pixels of this fragment column pair: their four scales' tap rows and columns
        int oy0[2][PSP_NS], oy1[2][PSP_NS], ox0[2][PSP_NS], ox1[2][PSP_NS];
        float ly0[2][PSP_NS], ly1[2][PSP_NS], lx0[2][PSP_NS], lx1[2][PSP_NS];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int gn = min(gn0 + u, P - 1), py = gn / W, px = gn - py * W;
#pragma unroll
            for (int k = 0; k < PSP_NS; ++k) {
                const PspTap ty = tap_y[k * H + py], tx = tap_x[k * W + px];
                const int s = c_psp_size[k];
                // bin (iy, ix) of scale k, frame b: row (B * off_k + b * s * s + iy * s + ix) of the table
                const int base = B * c_psp_off[k] + b * s * s;
                oy0[u][k] = base + ty.i0 * s;
                oy1[u][k] = base + ty.i1 * s;
                ox0[u][k] = tx.i0;
                ox1[u][k] = tx.i1;
                ly0[u][k] = ty.l0;
                ly1[u][k] = ty.l1;
                lx0[u][k] = tx.l0;
                lx1[u][k] = tx.l1;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int gm = row0 + 8 * h;
            if (gm >= Co) continue;
            const float bs = __ldg(bias + gm);
            const float *tc = table + gm;   // channels-last: the 8 rows of a warp read 32 contiguous bytes
            float y[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                float prior = 0.f;
#pragma unroll
                for (int k = 0; k < PSP_NS; ++k) {
                    // torch's order: h0lambda * (w0lambda * t00 + w1lambda * t01) + h1lambda * (...); every tap is
                    // read, so a NaN at a zero-weight tap propagates as it does in torch
                    const float t00 = __ldg(tc + (size_t)(oy0[u][k] + ox0[u][k]) * Co);
                    const float t01 = __ldg(tc + (size_t)(oy0[u][k] + ox1[u][k]) * Co);
                    const float t10 = __ldg(tc + (size_t)(oy1[u][k] + ox0[u][k]) * Co);
                    const float t11 = __ldg(tc + (size_t)(oy1[u][k] + ox1[u][k]) * Co);
                    const float r0 = __fadd_rn(__fmul_rn(lx0[u][k], t00), __fmul_rn(lx1[u][k], t01));
                    const float r1 = __fadd_rn(__fmul_rn(lx0[u][k], t10), __fmul_rn(lx1[u][k], t11));
                    prior = __fadd_rn(prior, __fadd_rn(__fmul_rn(ly0[u][k], r0), __fmul_rn(ly1[u][k], r1)));
                }
                y[u] = max_nan(__fadd_rn(__fadd_rn(sum[4 * i + 2 * h + u], prior), bs), 0.f);
            }
            float *orow = out + ((size_t)b * Co + gm) * P;
            if (vec && gn0 + 1 < P) {
                *reinterpret_cast<float2 *>(orow + gn0) = make_float2(y[0], y[1]);
            } else {
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (gn0 + u < P) orow[gn0 + u] = y[u];
            }
        }
    }
}

// `final` of PSPNet (models/cnn/pspnet.py:108-112): 1x1 conv + bias + LogSoftmax over the channels, Co <= 128, so every
// channel of a pixel is in the CTA's one 128-row tile.  The max and the sum of exponentials over the channels are
// reduced in the epilogue (registers -> shuffles across the 8 rows of a warp -> shared memory across the 8 warps), and
// the map is read once and written once.
__global__ void __launch_bounds__(MLP_THREADS, 1)
conv1x1_log_softmax_kernel(const float *__restrict__ x, int Ci, const unsigned char *__restrict__ wpack,
                           const float *__restrict__ bias, float *__restrict__ out, int Co, int P)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int b = blockIdx.z, n0 = blockIdx.x * TN;
    const float *xb = x + (size_t)b * Ci * P;
    const bool vec = ((P & 3) == 0) && ((reinterpret_cast<uintptr_t>(xb) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    float sum[64];
    packed_mainloop(smem, xb, Ci, nullptr, 0, wpack, P, n0, vec, sum);
    __syncthreads();   // the stages are free

    float *red = reinterpret_cast<float *>(smem);   // [8 warps][128 columns]
    float *colv = red + 8 * TN;                      // [128]: the column's max, then its max + log(sum)
    const int row0 = 64 * wg + 16 * (wid & 3) + (lane >> 2), c0 = 2 * (lane & 3);
    float bs[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) bs[h] = (row0 + 8 * h < Co) ? __ldg(bias + row0 + 8 * h) : 0.f;
#pragma unroll
    for (int i = 0; i < TN / 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int u = 0; u < 2; ++u) sum[4 * i + 2 * h + u] = __fadd_rn(sum[4 * i + 2 * h + u], bs[h]);

    // max over the channels (NaN if any is NaN, torch's max)
#pragma unroll
    for (int i = 0; i < TN / 8; ++i)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            float m = -INFINITY;
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (row0 + 8 * h < Co) m = max_nan(m, sum[4 * i + 2 * h + u]);
            m = max_nan(m, __shfl_xor_sync(0xffffffffu, m, 4));
            m = max_nan(m, __shfl_xor_sync(0xffffffffu, m, 8));
            m = max_nan(m, __shfl_xor_sync(0xffffffffu, m, 16));
            if (lane < 4) red[wid * TN + 8 * i + c0 + u] = m;
        }
    __syncthreads();
    if (tid < TN) {
        float m = red[tid];
        for (int w = 1; w < 8; ++w) m = max_nan(m, red[w * TN + tid]);
        colv[tid] = m;
    }
    __syncthreads();
    // sum of exp(y - max) over the channels
#pragma unroll
    for (int i = 0; i < TN / 8; ++i)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const float m = colv[8 * i + c0 + u];
            float s = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (row0 + 8 * h < Co) s = __fadd_rn(s, expf(__fsub_rn(sum[4 * i + 2 * h + u], m)));
            s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 4));
            s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 8));
            s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, 16));
            if (lane < 4) red[wid * TN + 8 * i + c0 + u] = s;
        }
    __syncthreads();
    if (tid < TN) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s = __fadd_rn(s, red[w * TN + tid]);
        red[tid] = logf(s);   // row 0 of red is read by no one else any more
    }
    __syncthreads();
    // out = y - max - log(sum), as torch's log_softmax
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int gm = row0 + 8 * h;
        if (gm >= Co) continue;
        float *orow = out + ((size_t)b * Co + gm) * P;
#pragma unroll
        for (int i = 0; i < TN / 8; ++i) {
            const int c = 8 * i + c0, gn = n0 + c;
            float y[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) y[u] = __fsub_rn(__fsub_rn(sum[4 * i + 2 * h + u], colv[c + u]), red[c + u]);
            if (vec && gn + 1 < P) {
                *reinterpret_cast<float2 *>(orow + gn) = make_float2(y[0], y[1]);
            } else {
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (gn + u < P) orow[gn + u] = y[u];
            }
        }
    }
}

// ===================================================================== weight gradient (training)
// dW[co, ci] = sum_b sum_p dZ[b, co, p] * X[b, ci, p],  X = [X1; X2]  (backward of the 1x1 conv w.r.t. its
// weight: a GEMM with M = Co, N = Ci and the long axis K = B * P).  Both operands are K-contiguous in memory
// (dZ and X are NCHW: the point axis is the fast one), so every thread loads 16 bytes along K and writes one
// whole (row; k..k+3) slot of the K-major layout -- no transposition.  Same numerics and pipeline as the
// forward layer: 3xTF32 split of both operands while they are staged, K accumulated in chunks of one k-tile that are
// added into round-to-nearest fp32 register sums.  Split-K over the grid's z axis: every CTA owns a run of
// (frame, 32-point) k-tiles and adds its 128x128 partial to dW with fp32 atomics (dW is zero-filled by the
// entry point), like cuDNN's own wgrad: summation order is not deterministic, values agree to fp32 round-off.
// DET (fusion_wgrad_det_kernel, ffb6d_fusion_mlp_wgrad_det): the same CTA stores its partial into its own slice
// dw + blockIdx.z * Co * Ci instead; wgrad_split_reduce_kernel adds the slices in split order.
template <bool DET>
__device__ __forceinline__ void
fusion_wgrad_body(const float *__restrict__ dz, const float *__restrict__ x1, int C1, const float *__restrict__ x2, int C2,
                  float *__restrict__ dw, int Co, int P, int tiles_per_frame, int total_tiles, int tiles_per_split)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
    const int Ci = C1 + C2;
    const int kt_begin = blockIdx.z * tiles_per_split, kt_end = min(total_tiles, kt_begin + tiles_per_split);
    const int nk = kt_end - kt_begin;
    if (nk <= 0) return;   // CTA-uniform

    const bool vec = ((P & 3) == 0) && ((reinterpret_cast<uintptr_t>(dz) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(x1) & 15) == 0) && (!x2 || (reinterpret_cast<uintptr_t>(x2) & 15) == 0);
    // global -> registers: warp w stages K chunk w (4 points) of both operands; lanes take rows lane + 32*i
    auto load4 = [&](const float *src, int gp) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (vec && gp + 3 < P) {
            v = __ldg(reinterpret_cast<const float4 *>(src));
        } else {
            v.x = __ldg(src);
            if (gp + 1 < P) v.y = __ldg(src + 1);
            if (gp + 2 < P) v.z = __ldg(src + 2);
            if (gp + 3 < P) v.w = __ldg(src + 3);
        }
        return v;
    };
    auto load_tile = [&](int kt, float4 (&ra)[4], float4 (&rb)[4]) {
        const int b = kt / tiles_per_frame, gp = (kt % tiles_per_frame) * TK + 4 * wid;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int gm = m0 + lane + 32 * i, gn = n0 + lane + 32 * i;
            ra[i] = (gm < Co && gp < P) ? load4(dz + ((size_t)b * Co + gm) * P + gp, gp) : make_float4(0.f, 0.f, 0.f, 0.f);
            // B rows = input channels n0 .. n0+127 of cat(x1, x2); a 128-row tile may straddle the concat
            rb[i] = (gn < Ci && gp < P)
                        ? load4((gn < C1) ? x1 + ((size_t)b * C1 + gn) * P + gp : x2 + ((size_t)b * C2 + (gn - C1)) * P + gp, gp)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto store_tile = [&](int st, const float4 (&ra)[4], const float4 (&rb)[4]) {
        unsigned char *sA_hi = smem + st * STAGE_BYTES, *sA_lo = sA_hi + TILE_BYTES;
        unsigned char *sB_hi = sA_lo + TILE_BYTES, *sB_lo = sB_hi + TILE_BYTES;
        float4 hi, lo;
#pragma unroll
        for (int i = 0; i < 4; ++i) {   // a warp's 16-byte stores are contiguous: bank-conflict free
            const int m = lane + 32 * i;
            split4(ra[i], hi, lo);
            *reinterpret_cast<float4 *>(sA_hi + wid * CHUNK_BYTES + m * 16) = hi;
            *reinterpret_cast<float4 *>(sA_lo + wid * CHUNK_BYTES + m * 16) = lo;
            split4(rb[i], hi, lo);
            *reinterpret_cast<float4 *>(sB_hi + wid * CHUNK_BYTES + m * 16) = hi;
            *reinterpret_cast<float4 *>(sB_lo + wid * CHUNK_BYTES + m * 16) = lo;
        }
    };

    float acc[64], sum[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = sum[i] = 0.f;
    float4 ra[4], rb[4];
    load_tile(kt_begin, ra, rb);
    for (int kt = 0; kt < nk; ++kt) {
        const int st = kt % NST;
        store_tile(st, ra, rb);   // stage st was last read by the MMAs of k-tile kt - 3: complete
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        if (kt + 1 < nk) load_tile(kt_begin + kt + 1, ra, rb);
        if (kt % CH == 0 && kt > 0) drain(acc, sum);
        mma_ktile(acc, smem_u32(smem + st * STAGE_BYTES), wg, kt % CH == 0);
        wgmma_wait<1>();
    }
    drain(acc, sum);
    const int row0 = m0 + 64 * wg + 16 * (wid & 3) + (lane >> 2), col0 = n0 + 2 * (lane & 3);
    if (DET) dw += (size_t)blockIdx.z * Co * Ci;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int gm = row0 + 8 * h;
        if (gm >= Co) continue;
        float *row = dw + (size_t)gm * Ci;
#pragma unroll
        for (int i = 0; i < TN / 8; ++i)
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int gn = col0 + 8 * i + u;
                if (gn < Ci) {
                    if (DET)
                        row[gn] = sum[4 * i + 2 * h + u];
                    else
                        atomicAdd(row + gn, sum[4 * i + 2 * h + u]);
                }
            }
    }
}

__global__ void __launch_bounds__(MLP_THREADS, 1)
fusion_wgrad_kernel(const float *__restrict__ dz, const float *__restrict__ x1, int C1, const float *__restrict__ x2, int C2,
                    float *__restrict__ dw, int Co, int P, int tiles_per_frame, int total_tiles, int tiles_per_split)
{
    fusion_wgrad_body<false>(dz, x1, C1, x2, C2, dw, Co, P, tiles_per_frame, total_tiles, tiles_per_split);
}

// dw = the workspace of ffb6d_fusion_mlp_wgrad_det: one [Co, Ci] slice per split
__global__ void __launch_bounds__(MLP_THREADS, 1)
fusion_wgrad_det_kernel(const float *__restrict__ dz, const float *__restrict__ x1, int C1, const float *__restrict__ x2,
                        int C2, float *__restrict__ dw, int Co, int P, int tiles_per_frame, int total_tiles, int tiles_per_split)
{
    fusion_wgrad_body<true>(dz, x1, C1, x2, C2, dw, Co, P, tiles_per_frame, total_tiles, tiles_per_split);
}

// dw[i] = the fp64 sum of part[s * n + i] over s = 0 .. nsplit-1 in that order, rounded once
__global__ void __launch_bounds__(256)
wgrad_split_reduce_kernel(const float *__restrict__ part, int nsplit, long long n, float *__restrict__ dw)
{
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    double acc = 0.0;
    for (int s = 0; s < nsplit; ++s) acc += (double)__ldg(part + (size_t)s * n + i);
    dw[i] = (float)acc;
}

// split count of fusion_wgrad_kernel (a function of the shape and the SM count only)
static int64_t wgrad_splits(int64_t B, int64_t Co, int64_t Ci, int64_t P, int64_t &per)
{
    const int64_t tpf = ceil_div(P, TK), total = B * tpf;
    const int64_t tiles = ceil_div(Ci, TN) * ceil_div(Co, TM);
    // split K so that the grid fills the SMs about twice, but keep at least 8 k-tiles (one chunk pair) per CTA
    int64_t splits = std::max<int64_t>(1, std::min<int64_t>(ceil_div(2 * (int64_t)num_sms(), tiles), ceil_div(total, 8)));
    if (splits > 65535) splits = 65535;
    per = ceil_div(total, splits);
    return ceil_div(total, per);
}

}  // namespace ffb6d

using namespace ffb6d;

static int mlp_check(const void *x1, int64_t C1, const void *x2, int64_t C2, const void *weight, const void *scale,
                     const void *shift, int64_t B, int64_t Co, int64_t P, int act, const void *out)
{
    FFB6D_CHECK_ARG(B >= 0 && C1 >= 1 && C2 >= 0 && Co >= 1 && P >= 0, "fusion_mlp_fwd: bad size");
    FFB6D_CHECK_ARG(act >= 0 && act <= 2, "fusion_mlp_fwd: act=%d (0 none, 1 ReLU, 2 LeakyReLU)", act);
    FFB6D_CHECK_ARG(B < 65536 && Co <= 65535ll * TM && P < (1ll << 31) && C1 + C2 < (1ll << 31),
                    "fusion_mlp_fwd: size too large");
    if (B == 0 || P == 0) return 1;   // nothing to do
    FFB6D_CHECK_ARG(x1 && weight && scale && shift && out && (C2 == 0 || x2), "fusion_mlp_fwd: null pointer");
    return FFB6D_OK;
}

extern "C" size_t ffb6d_fusion_mlp_pack_bytes(int64_t Co, int64_t Ci)
{
    if (Co < 1 || Ci < 1) return 0;
    return (size_t)ceil_div(Co, TM) * (size_t)ceil_div(Ci, TK) * PACK_BLOCK_BYTES;
}

extern "C" int ffb6d_fusion_mlp_pack(const float *weight, int64_t Co, int64_t Ci, void *packed, size_t packed_bytes,
                                     ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(weight && packed && Co >= 1 && Ci >= 1 && Ci < (1ll << 31) && Co <= 65535ll * TM,
                    "fusion_mlp_pack: bad argument");
    const size_t need = ffb6d_fusion_mlp_pack_bytes(Co, Ci);
    if (packed_bytes < need) {
        set_error("fusion_mlp_pack: %zu bytes required, %zu given", need, packed_bytes);
        return FFB6D_ERR_WORKSPACE;
    }
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "fusion_mlp_pack: packed must be 16-byte aligned");
    const int nk = (int)ceil_div(Ci, TK), nblocks = (int)(ceil_div(Co, TM) * nk);
    fusion_mlp_pack_kernel<<<(unsigned)ceil_div((int64_t)nblocks * 1024, 256), 256, 0, (cudaStream_t)stream>>>(
        weight, (int)Co, (int)Ci, nk, nblocks, (float4 *)packed);
    FFB6D_LAUNCH_OK("fusion_mlp_pack_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_fusion_mlp_fwd_ex(const float *x1, int64_t C1, const float *x2, int64_t C2, const void *packed,
                                       const float *scale, const float *shift, int64_t B, int64_t Co, int64_t P,
                                       int act, float negative_slope, const float *addend, const void *add_idx,
                                       int add_idx_is_i64, int64_t NA, int out_layout, float *out, ffb6d_stream_t stream)
{
    const int rc = mlp_check(x1, C1, x2, C2, packed, scale, shift, B, Co, P, act, out);
    if (rc != FFB6D_OK) return rc > 0 ? FFB6D_OK : rc;
    FFB6D_CHECK_ARG(out_layout == FFB6D_LAYOUT_NCS || out_layout == FFB6D_LAYOUT_NSC, "fusion_mlp_fwd: unknown out_layout %d",
                    out_layout);
    FFB6D_CHECK_ARG((addend == nullptr) == (add_idx == nullptr), "fusion_mlp_fwd: addend and add_idx come together");
    FFB6D_CHECK_ARG(!addend || (NA >= 1 && NA < (1ll << 31)), "fusion_mlp_fwd: bad addend length");
    FFB6D_OPTIN_SMEM(fusion_mlp_packed_kernel, MLP_SMEM);
    MlpEpilogue ep;
    ep.addend = addend;
    ep.idx = add_idx;
    ep.NA = (int)NA;
    ep.idx_is_i64 = add_idx_is_i64;
    ep.out_nsc = out_layout == FFB6D_LAYOUT_NSC;
    dim3 grid((unsigned)ceil_div(P, TN), (unsigned)ceil_div(Co, TM), (unsigned)B);
    fusion_mlp_packed_kernel<<<grid, MLP_THREADS, MLP_SMEM, (cudaStream_t)stream>>>(
        x1, (int)C1, C2 ? x2 : nullptr, (int)C2, (const unsigned char *)packed, scale, shift, out, (int)Co, (int)P,
        act, negative_slope, ep);
    FFB6D_LAUNCH_OK("fusion_mlp_packed_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_fusion_mlp_fwd_packed(const float *x1, int64_t C1, const float *x2, int64_t C2, const void *packed,
                                           const float *scale, const float *shift, int64_t B, int64_t Co, int64_t P,
                                           int act, float negative_slope, float *out, ffb6d_stream_t stream)
{
    return ffb6d_fusion_mlp_fwd_ex(x1, C1, x2, C2, packed, scale, shift, B, Co, P, act, negative_slope, nullptr, nullptr, 0,
                                   0, FFB6D_LAYOUT_NCS, out, stream);
}

extern "C" int ffb6d_fusion_mlp_wgrad(const float *grad_z, const float *x1, int64_t C1, const float *x2, int64_t C2,
                                      int64_t B, int64_t Co, int64_t P, float *grad_w, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && C1 >= 1 && C2 >= 0 && Co >= 1 && P >= 0, "fusion_mlp_wgrad: bad size");
    FFB6D_CHECK_ARG(B < 65536 && Co <= 65535ll * TM && C1 + C2 <= 65535ll * TN && P < (1ll << 31),
                    "fusion_mlp_wgrad: size too large");
    FFB6D_CHECK_ARG(grad_w, "fusion_mlp_wgrad: null grad_w");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t Ci = C1 + C2;
    FFB6D_CUDA(cudaMemsetAsync(grad_w, 0, (size_t)Co * Ci * sizeof(float), st));
    if (B == 0 || P == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(grad_z && x1 && (C2 == 0 || x2), "fusion_mlp_wgrad: null pointer");
    if (Co <= 64 && Ci <= 64)   // narrow layer: a 128x128 tensor-core tile would be mostly padding (train.cu)
        return wgrad_small_launch(grad_z, x1, C1, x2, C2, B, Co, P, grad_w, st);
    FFB6D_OPTIN_SMEM(fusion_wgrad_kernel, MLP_SMEM);
    const int64_t tpf = ceil_div(P, TK), total = B * tpf;
    FFB6D_CHECK_ARG(total < (1ll << 31), "fusion_mlp_wgrad: B * P too large");
    int64_t per = 0;
    const int64_t splits = wgrad_splits(B, Co, Ci, P, per);
    dim3 grid((unsigned)ceil_div(Ci, TN), (unsigned)ceil_div(Co, TM), (unsigned)splits);
    fusion_wgrad_kernel<<<grid, MLP_THREADS, MLP_SMEM, st>>>(grad_z, x1, (int)C1, C2 ? x2 : nullptr, (int)C2, grad_w, (int)Co, (int)P,
                                                    (int)tpf, (int)total, (int)per);
    FFB6D_LAUNCH_OK("fusion_wgrad_kernel");
    return FFB6D_OK;
}

static bool wgrad_det_sizes_ok(int64_t C1, int64_t C2, int64_t B, int64_t Co, int64_t P)
{
    return B >= 1 && C1 >= 1 && C2 >= 0 && Co >= 1 && P >= 1 && B < 65536 && Co <= 65535ll * TM && C1 + C2 <= 65535ll * TN &&
           P < (1ll << 31) && B * ceil_div(P, TK) < (1ll << 31);
}

extern "C" size_t ffb6d_fusion_mlp_wgrad_det_workspace_bytes(int64_t C1, int64_t C2, int64_t B, int64_t Co, int64_t P)
{
    if (!wgrad_det_sizes_ok(C1, C2, B, Co, P)) return 0;
    const int64_t Ci = C1 + C2;
    int64_t per = 0;
    const int64_t splits = (Co <= 64 && Ci <= 64) ? wgrad_small_splits(B, P) : wgrad_splits(B, Co, Ci, P, per);
    return align_up((size_t)splits * Co * Ci * sizeof(float), 16);
}

extern "C" int ffb6d_fusion_mlp_wgrad_det(const float *grad_z, const float *x1, int64_t C1, const float *x2, int64_t C2,
                                          int64_t B, int64_t Co, int64_t P, void *workspace, size_t workspace_bytes,
                                          float *grad_w, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && C1 >= 1 && C2 >= 0 && Co >= 1 && P >= 0, "fusion_mlp_wgrad_det: bad size");
    FFB6D_CHECK_ARG(B < 65536 && Co <= 65535ll * TM && C1 + C2 <= 65535ll * TN && P < (1ll << 31),
                    "fusion_mlp_wgrad_det: size too large");
    FFB6D_CHECK_ARG(grad_w, "fusion_mlp_wgrad_det: null grad_w");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t Ci = C1 + C2;
    if (B == 0 || P == 0) {
        FFB6D_CUDA(cudaMemsetAsync(grad_w, 0, (size_t)Co * Ci * sizeof(float), st));
        return FFB6D_OK;
    }
    FFB6D_CHECK_ARG(wgrad_det_sizes_ok(C1, C2, B, Co, P), "fusion_mlp_wgrad_det: B * P too large");
    FFB6D_CHECK_ARG(grad_z && x1 && (C2 == 0 || x2) && workspace, "fusion_mlp_wgrad_det: null pointer");
    FFB6D_CHECK_ARG(((reinterpret_cast<uintptr_t>(grad_z) | reinterpret_cast<uintptr_t>(x1) | reinterpret_cast<uintptr_t>(x2) |
                      reinterpret_cast<uintptr_t>(grad_w)) & 3) == 0,
                    "fusion_mlp_wgrad_det: grad_z, x1, x2 and grad_w must be 4-byte aligned");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "fusion_mlp_wgrad_det: workspace must be 16-byte aligned");
    const size_t need = ffb6d_fusion_mlp_wgrad_det_workspace_bytes(C1, C2, B, Co, P);
    FFB6D_CHECK_ARG(workspace_bytes >= need, "fusion_mlp_wgrad_det: workspace too small (%zu bytes required, %zu given)", need,
                    workspace_bytes);
    float *part = (float *)workspace;
    int64_t splits;
    if (Co <= 64 && Ci <= 64) {
        splits = wgrad_small_splits(B, P);
        const int rc = wgrad_small_det_launch(grad_z, x1, C1, x2, C2, B, Co, P, part, st);
        if (rc != FFB6D_OK) return rc;
    } else {
        FFB6D_OPTIN_SMEM(fusion_wgrad_det_kernel, MLP_SMEM);
        int64_t per = 0;
        splits = wgrad_splits(B, Co, Ci, P, per);
        dim3 grid((unsigned)ceil_div(Ci, TN), (unsigned)ceil_div(Co, TM), (unsigned)splits);
        fusion_wgrad_det_kernel<<<grid, MLP_THREADS, MLP_SMEM, st>>>(grad_z, x1, (int)C1, C2 ? x2 : nullptr, (int)C2, part,
                                                                     (int)Co, (int)P, (int)ceil_div(P, TK),
                                                                     (int)(B * ceil_div(P, TK)), (int)per);
        FFB6D_LAUNCH_OK("fusion_wgrad_det_kernel");
    }
    const long long n = (long long)Co * Ci;
    wgrad_split_reduce_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(part, (int)splits, n, grad_w);
    FFB6D_LAUNCH_OK("wgrad_split_reduce_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_psp_bottleneck_fwd(const float *x, int64_t B, int64_t C, int64_t H, int64_t W, const void *packed,
                                        const float *bias, int64_t Co, const float *table, float *out,
                                        ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && C >= 1 && H >= 1 && W >= 1 && Co >= 1, "psp_bottleneck_fwd: bad size");
    FFB6D_CHECK_ARG(B < 65536 && Co <= 65535ll * TM && C < (1ll << 31) && H + W <= 3072 && H * W < (1ll << 31) &&
                        B * 50 * Co < (1ll << 31),
                    "psp_bottleneck_fwd: size too large");
    FFB6D_CHECK_ARG(x && packed && bias && table && out, "psp_bottleneck_fwd: null pointer");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "psp_bottleneck_fwd: packed must be 16-byte aligned");
    FFB6D_OPTIN_SMEM(psp_bottleneck_kernel, MLP_SMEM);
    dim3 grid((unsigned)ceil_div(H * W, TN), (unsigned)ceil_div(Co, TM), (unsigned)B);
    psp_bottleneck_kernel<<<grid, MLP_THREADS, MLP_SMEM, (cudaStream_t)stream>>>(
        x, (int)C, (const unsigned char *)packed, bias, table, out, (int)Co, (int)H, (int)W, (int)B);
    FFB6D_LAUNCH_OK("psp_bottleneck_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_conv1x1_log_softmax_fwd(const float *x, int64_t B, int64_t Ci, int64_t P, const void *packed,
                                             const float *bias, int64_t Co, float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && Ci >= 1 && P >= 1 && Co >= 1, "conv1x1_log_softmax_fwd: bad size");
    FFB6D_CHECK_ARG(Co <= TM, "conv1x1_log_softmax_fwd: Co = %lld, at most %d channels", (long long)Co, TM);
    FFB6D_CHECK_ARG(B < 65536 && Ci < (1ll << 31) && P < (1ll << 31), "conv1x1_log_softmax_fwd: size too large");
    FFB6D_CHECK_ARG(x && packed && bias && out, "conv1x1_log_softmax_fwd: null pointer");
    FFB6D_CHECK_ARG((reinterpret_cast<uintptr_t>(packed) & 15) == 0,
                    "conv1x1_log_softmax_fwd: packed must be 16-byte aligned");
    FFB6D_OPTIN_SMEM(conv1x1_log_softmax_kernel, MLP_SMEM);
    dim3 grid((unsigned)ceil_div(P, TN), 1u, (unsigned)B);
    conv1x1_log_softmax_kernel<<<grid, MLP_THREADS, MLP_SMEM, (cudaStream_t)stream>>>(
        x, (int)Ci, (const unsigned char *)packed, bias, out, (int)Co, (int)P);
    FFB6D_LAUNCH_OK("conv1x1_log_softmax_kernel");
    return FFB6D_OK;
}
