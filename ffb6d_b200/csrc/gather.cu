// gather.cu -- gather + max-pool over neighbours, nearest-feature gather, neighbour
// gather and relative position encoding (sm_90a).
//
// Reference ops (ffb6d/models/ffb6d.py:159-194, 309-312; models/RandLA/RandLANet.py:
// 87-117, 216-234) are chains of reshape / repeat / torch.gather / max that
// materialise an int64 [B,C,Q*K] index tensor and a [B,C,Q*K] feature tensor.  Here
// every op is one kernel that reads each touched source row once and writes the
// result once.
//
// NCS layout ([B,C,S], point axis contiguous -- the reference's NCHW):
//   * "staged" kernel: a CTA copies CC whole channel rows (CC*S floats, coalesced
//     128-bit loads) into shared memory, then its threads walk the queries: the K
//     indices of a query are loaded once into registers and reused for all CC
//     rows, neighbour values come from shared memory, the result row is written
//     coalesced along q.  HBM traffic = rows once + idx (C/CC times, L2 hits) + out.
//   * "direct" kernel for rows that do not fit shared memory (S > ~50k): same
//     thread mapping, neighbour values through the read-only L1/L2 path.
// NSC layout ([B,S,C], channel axis contiguous -- torch channels_last): a warp owns
//   a query, lanes span channels with 128-bit loads: every neighbour is one
//   contiguous row read (embedding-lookup pattern).
#include "common.cuh"

#include <algorithm>
#include <stdlib.h>

namespace ffb6d {

// torch.max(dim) semantics: the value of the first NaN, else of the first maximal element, bit for bit.  `a` holds the
// earlier neighbours, `b` later ones.  The backward's arg-max (gather_max_bwd_kernel, gather_argmax_kernel) follows
// the same rule, so the forward's output is the feature the gradient goes to.  max.NaN.f32 (max_nan, common.cuh) would
// not do: of -0.0 then +0.0 it returns +0.0, and of a NaN the canonical NaN, not the feature's payload.
__device__ __forceinline__ float max_first(float a, float b) { return (b > a || (b != b && a == a)) ? b : a; }

template <typename IdxT, int KT>
__device__ __forceinline__ void load_ids(const IdxT *__restrict__ ip, int K, int (&id)[KT > 0 ? KT : 1])
{
    // K indices of one query are contiguous: 16 int32 = 64 B, 16 int64 = 128 B
    if constexpr (KT > 0) {
        if constexpr (sizeof(IdxT) == 4 && (KT % 4 == 0)) {
            const int4 *p4 = reinterpret_cast<const int4 *>(ip);
#pragma unroll
            for (int k = 0; k < KT / 4; ++k) {
                const int4 v = __ldg(p4 + k);
                id[4 * k + 0] = v.x;
                id[4 * k + 1] = v.y;
                id[4 * k + 2] = v.z;
                id[4 * k + 3] = v.w;
            }
        } else if constexpr (sizeof(IdxT) == 8 && (KT % 2 == 0)) {
            const longlong2 *p2 = reinterpret_cast<const longlong2 *>(ip);
#pragma unroll
            for (int k = 0; k < KT / 2; ++k) {
                const longlong2 v = __ldg(p2 + k);
                id[2 * k + 0] = (int)v.x;
                id[2 * k + 1] = (int)v.y;
            }
        } else {
#pragma unroll
            for (int k = 0; k < KT; ++k) id[k] = (int)__ldg(ip + k);
        }
    }
}

// ------------------------------------------------------------------ row staging with the bulk-copy engine
// Copies `bytes` (multiple of 16, both sides 16-byte aligned) from global to shared memory with
// cp.async.bulk (the 1-D TMA path, SASS UBLKCP): one thread programs the copies, the data never passes
// through registers, and completion is signalled on an mbarrier every thread then waits on.  Deep
// memory-level parallelism for free: a CTA has its whole 100 KB of rows in flight at once.
__device__ __forceinline__ void stage_rows_bulk(float *smem_dst, const float *gmem_src, unsigned bytes,
                                                unsigned long long *bar)
{
    const unsigned bar_a = (unsigned)__cvta_generic_to_shared(bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        const unsigned dst = (unsigned)__cvta_generic_to_shared(smem_dst);
        for (unsigned off = 0; off < bytes; off += 32768u) {
            const unsigned n = min(32768u, bytes - off);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst + off), "l"(reinterpret_cast<const char *>(gmem_src) + off), "r"(n), "r"(bar_a)
                         : "memory");
        }
    }
    unsigned done = 0;
    for (int spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, P1;\n\t}\n"
            : "=r"(done) : "r"(bar_a), "r"(0u) : "memory");
        if (spin > (1 << 26)) __trap();   // never hang the GPU on a protocol bug
    }
}

// ------------------------------------------------------------------ NCS staged
template <typename IdxT, int KT>
__global__ void __launch_bounds__(256)
gather_max_ncs_staged_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                             float *__restrict__ out, int C, int S, int Q, int K, int CC,
                             int q_per_cta)
{
    extern __shared__ __align__(16) float rows[];  // [cc][S]
    __shared__ __align__(8) unsigned long long bar[1];
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * CC;
    const int cc = min(CC, C - c0);
    const float *src = feat + ((size_t)b * C + c0) * S;
    const int n = cc * S;
    if ((n & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
        stage_rows_bulk(rows, src, (unsigned)n * 4u, bar);   // whole rows in flight, no register pass
    } else {
        for (int t = threadIdx.x; t < n; t += blockDim.x) rows[t] = __ldg(src + t);
        __syncthreads();
    }

    const int q0 = blockIdx.x * q_per_cta;
    const int q1 = min(Q, q0 + q_per_cta);
    float *dst = out + ((size_t)b * C + c0) * Q;
    for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
        const IdxT *ip = idx + ((size_t)b * Q + q) * K;
        if constexpr (KT > 0) {
            int id[KT];
            load_ids<IdxT, KT>(ip, K, id);
            for (int c = 0; c < cc; ++c) {
                const float *r = rows + c * S;
                float m = r[id[0]];
#pragma unroll
                for (int k = 1; k < KT; ++k) m = max_first(m, r[id[k]]);
                dst[(size_t)c * Q + q] = m;
            }
        } else {
            for (int c = 0; c < cc; ++c) {
                const float *r = rows + c * S;
                float m = r[(int)__ldg(ip)];
                for (int k = 1; k < K; ++k) m = max_first(m, r[(int)__ldg(ip + k)]);
                dst[(size_t)c * Q + q] = m;
            }
        }
    }
}

// ------------------------------------------------------------------ NCS staged, K == 1, four queries per thread
// nearest_interpolation / p2r gathers: small source rows, long query lists.  A thread takes four
// consecutive queries (one 128-bit index load), reads the four values of each staged row from
// shared memory and writes them with one 128-bit store: the output stream is the only HBM
// traffic that matters here and it is written in 512-byte warp bursts.
template <typename IdxT>
__global__ void __launch_bounds__(256)
gather1_ncs_staged_v4_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                             float *__restrict__ out, int C, int S, int Q, int CC, int q_per_cta)
{
    extern __shared__ __align__(16) float rows[];  // [cc][S]
    __shared__ __align__(8) unsigned long long bar[1];
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * CC;
    const int cc = min(CC, C - c0);
    const float *src = feat + ((size_t)b * C + c0) * S;
    const int n = cc * S;
    if ((n & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
        stage_rows_bulk(rows, src, (unsigned)n * 4u, bar);   // whole rows in flight, no register pass
    } else {
        for (int t = threadIdx.x; t < n; t += blockDim.x) rows[t] = __ldg(src + t);
        __syncthreads();
    }
    const int q0 = blockIdx.x * q_per_cta;          // multiple of 4
    const int q1 = min(Q, q0 + q_per_cta);          // Q is a multiple of 4
    float *dst = out + ((size_t)b * C + c0) * Q;
    const IdxT *ib = idx + (size_t)b * Q;
    auto load4 = [&](int q, int (&id)[4]) {
        if constexpr (sizeof(IdxT) == 4) {
            const int4 v = __ldg(reinterpret_cast<const int4 *>(ib + q));
            id[0] = v.x; id[1] = v.y; id[2] = v.z; id[3] = v.w;
        } else {
            const longlong2 u = __ldg(reinterpret_cast<const longlong2 *>(ib + q));
            const longlong2 w = __ldg(reinterpret_cast<const longlong2 *>(ib + q) + 1);
            id[0] = (int)u.x; id[1] = (int)u.y; id[2] = (int)w.x; id[3] = (int)w.y;
        }
    };
    // two index loads in flight per thread; the loop is otherwise bound by the latency of that load
    const int step = blockDim.x * 4;
    for (int q = q0 + threadIdx.x * 4; q < q1; q += 2 * step) {
        int ia[4], ibb[4] = {0, 0, 0, 0};
        const bool two = q + step < q1;
        load4(q, ia);
        if (two) load4(q + step, ibb);
#pragma unroll 4
        for (int c = 0; c < cc; ++c) {
            const float *r = rows + c * S;
            __stcs(reinterpret_cast<float4 *>(dst + (size_t)c * Q + q),
                   make_float4(r[ia[0]], r[ia[1]], r[ia[2]], r[ia[3]]));
            if (two)
                __stcs(reinterpret_cast<float4 *>(dst + (size_t)c * Q + q + step),
                       make_float4(r[ibb[0]], r[ibb[1]], r[ibb[2]], r[ibb[3]]));
        }
    }
}

// ------------------------------------------------------------------ NCS direct
template <typename IdxT, int KT>
__global__ void __launch_bounds__(256)
gather_max_ncs_direct_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                             float *__restrict__ out, int C, int S, int Q, int K, int CC)
{
    // rows too long for shared memory: neighbour values come through L1/L2.  All loads of a
    // channel pair are issued before the first use so 2*K requests per thread are in flight.
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * CC;
    const int cc = min(CC, C - c0);
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    const float *src = feat + ((size_t)b * C + c0) * S;
    float *dst = out + ((size_t)b * C + c0) * Q;
    const IdxT *ip = idx + ((size_t)b * Q + q) * K;
    if constexpr (KT > 0) {
        int id[KT];
        load_ids<IdxT, KT>(ip, K, id);
        int c = 0;
        for (; c + 1 < cc; c += 2) {
            const float *r0 = src + (size_t)c * S;
            const float *r1 = r0 + S;
            float v0[KT], v1[KT];
#pragma unroll
            for (int k = 0; k < KT; ++k) {
                v0[k] = __ldg(r0 + id[k]);
                v1[k] = __ldg(r1 + id[k]);
            }
            float m0 = v0[0], m1 = v1[0];
#pragma unroll
            for (int k = 1; k < KT; ++k) {
                m0 = max_first(m0, v0[k]);
                m1 = max_first(m1, v1[k]);
            }
            dst[(size_t)c * Q + q] = m0;
            dst[(size_t)(c + 1) * Q + q] = m1;
        }
        if (c < cc) {
            const float *r = src + (size_t)c * S;
            float m = __ldg(r + id[0]);
#pragma unroll
            for (int k = 1; k < KT; ++k) m = max_first(m, __ldg(r + id[k]));
            dst[(size_t)c * Q + q] = m;
        }
    } else {
        for (int c = 0; c < cc; ++c) {
            const float *r = src + (size_t)c * S;
            float m = __ldg(r + (int)__ldg(ip));
            for (int k = 1; k < K; ++k) m = max_first(m, __ldg(r + (int)__ldg(ip + k)));
            dst[(size_t)c * Q + q] = m;
        }
    }
}

// Long rows with K = 8/16/32 (r2p gathers from the 240x320 map): the K lanes of a group hold the K
// neighbours of ONE query.  Neighbours of a query are adjacent pixels, so a warp-wide load touches
// a handful of 32-byte sectors instead of 32 (lanes along the query axis would scatter every
// lane into its own sector); the max over the group is a log2(K)-step shuffle reduction.  Results
// are collected in a [channel][query] shared-memory tile and written out coalesced.  The shuffle steps go up from
// distance 1, so each combines two adjacent ranges of neighbours in their order and lane 0 ends with the first NaN or
// first maximum of all K (from distance K/2 down, lane 0 would compare {0, 8} with {4, 12}).
// A CTA takes one query per lane group (256 / K queries) and issues the loads of all its channels
// before the first shuffle: eight loads in flight per thread, and short CTAs.  (H100: 10-20 % less
// time on the sparse r2p gathers than 32 queries per CTA in rounds of four channels.)
constexpr int KLANE_CH = 8;           // channels per CTA: many CTAs per frame keep ONE frame's rows in L2
                                      // (ncu: with 64 channels per CTA twelve frames were in flight,
                                      // 235 MB of rows thrashed the L2 and DRAM read them twice)

template <typename IdxT, int KT>
__global__ void __launch_bounds__(256)
gather_max_ncs_klane_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                            float *__restrict__ out, int C, int S, int Q)
{
    constexpr int TQ = 256 / KT;      // queries per CTA: one per lane group
    __shared__ float tile[KLANE_CH][TQ + 1];
    const int b = blockIdx.z;
    const int q_tile = blockIdx.x * TQ;
    const int ql = threadIdx.x / KT, kl = threadIdx.x % KT;
    const int q = q_tile + ql;
    const bool on = q < Q;
    const int c0 = blockIdx.y * KLANE_CH;
    const int cc = min(KLANE_CH, C - c0);
    const int id = on ? (int)__ldg(idx + ((size_t)b * Q + q) * KT + kl) : 0;
    const float *src = feat + ((size_t)b * C + c0) * S + id;
    float v[KLANE_CH];
#pragma unroll
    for (int c = 0; c < KLANE_CH; ++c) v[c] = (c < cc) ? __ldg(src + (size_t)c * S) : 0.f;
#pragma unroll
    for (int c = 0; c < KLANE_CH; ++c) {
#pragma unroll
        for (int o = 1; o < KT; o <<= 1) {   // blocks of o lanes; the one with bit o clear holds the earlier neighbours
            const float u = __shfl_xor_sync(0xffffffffu, v[c], o);
            v[c] = (kl & o) ? max_first(u, v[c]) : max_first(v[c], u);
        }
        if (kl == 0 && c < cc) tile[c][ql] = v[c];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < cc * TQ; t += blockDim.x) {
        const int c = t / TQ, qt = t % TQ;
        if (q_tile + qt < Q) out[((size_t)b * C + c0 + c) * Q + q_tile + qt] = tile[c][qt];
    }
}

// K == 1 with long rows (the `choose` gather): two channels per thread, loads first.  The picks are
// scattered, so nearly every load misses to its own HBM line; two channels per thread make many short
// CTAs, which keep more lines in flight than fewer CTAs with more loads each (H100, B = 32: 0.55 ms
// against 0.60 ms with four channels and 0.64 ms with eight).
constexpr int G1_CH = 2;

template <typename IdxT>
__global__ void __launch_bounds__(256)
gather1_ncs_direct_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                          float *__restrict__ out, int C, int S, int Q)
{
    const int b = blockIdx.z;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    const int id = (int)__ldg(idx + (size_t)b * Q + q);
    for (int c0 = blockIdx.y * G1_CH; c0 < C; c0 += gridDim.y * G1_CH) {   // grid.y is capped at 65535
        const float *src = feat + ((size_t)b * C + c0) * S + id;
        float *dst = out + ((size_t)b * C + c0) * Q + q;
        float v[G1_CH];
#pragma unroll
        for (int c = 0; c < G1_CH; ++c) v[c] = (c0 + c < C) ? __ldg(src + (size_t)c * S) : 0.f;
#pragma unroll
        for (int c = 0; c < G1_CH; ++c)
            if (c0 + c < C) __stcs(dst + (size_t)c * Q, v[c]);
    }
}

// ------------------------------------------------------------------ NSC (channels last)
// one warp per query; lane l handles channels 4l..4l+3 (+128 per pass)
template <typename IdxT>
__global__ void __launch_bounds__(256)
gather_max_nsc_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                      float *__restrict__ out, int C, int S, int Q, int K, long long total_q)
{
    const int lane = threadIdx.x & 31;
    const long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (w >= total_q) return;
    const int b = (int)(w / Q);
    const IdxT *ip = idx + (size_t)w * K;
    const float *base = feat + (size_t)b * S * C;
    float *o = out + (size_t)w * C;
    // lanes fetch the indices once (K <= 64)
    int my0 = (lane < K) ? (int)__ldg(ip + lane) : 0;
    int my1 = (lane + 32 < K) ? (int)__ldg(ip + lane + 32) : 0;
    // trip counts are warp-uniform: every lane takes part in the index shuffles
    if ((C & 3) == 0) {
        for (int c0 = 0; c0 < C; c0 += 128) {
            const int c = c0 + lane * 4;
            const bool on = c < C;
            const int s0 = __shfl_sync(0xffffffffu, my0, 0);
            float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
            if (on) m = __ldg(reinterpret_cast<const float4 *>(base + (size_t)s0 * C + c));
            for (int k = 1; k < K; ++k) {
                const int s = __shfl_sync(0xffffffffu, (k < 32) ? my0 : my1, k & 31);
                if (on) {
                    const float4 v = __ldg(reinterpret_cast<const float4 *>(base + (size_t)s * C + c));
                    m.x = max_first(m.x, v.x);
                    m.y = max_first(m.y, v.y);
                    m.z = max_first(m.z, v.z);
                    m.w = max_first(m.w, v.w);
                }
            }
            if (on) *reinterpret_cast<float4 *>(o + c) = m;
        }
    } else {
        for (int c0 = 0; c0 < C; c0 += 32) {
            const int c = c0 + lane;
            const bool on = c < C;
            const int s0 = __shfl_sync(0xffffffffu, my0, 0);
            float m = on ? __ldg(base + (size_t)s0 * C + c) : 0.f;
            for (int k = 1; k < K; ++k) {
                const int s = __shfl_sync(0xffffffffu, (k < 32) ? my0 : my1, k & 31);
                if (on) m = max_first(m, __ldg(base + (size_t)s * C + c));
            }
            if (on) o[c] = m;
        }
    }
}

// ------------------------------------------------------------------ backward
// grad_feat[b,c,argmax] += grad_out[b,c,q]; the arg-max is recomputed from feat
// (first maximal k, NaN wins) so the forward stores nothing extra.
template <typename IdxT>
__global__ void __launch_bounds__(256)
gather_max_bwd_kernel(const float *__restrict__ feat, const IdxT *__restrict__ idx,
                      const float *__restrict__ gout, float *__restrict__ gfeat, int C, int S,
                      int Q, int K, int layout, long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    int b, c, q;
    size_t fs_c, fs_s;
    if (layout == FFB6D_LAYOUT_NCS) {  // t = (b*C + c)*Q + q
        q = (int)(t % Q);
        c = (int)((t / Q) % C);
        b = (int)(t / ((long long)Q * C));
        fs_c = (size_t)S;
        fs_s = 1;
    } else {  // t = (b*Q + q)*C + c
        c = (int)(t % C);
        q = (int)((t / C) % Q);
        b = (int)(t / ((long long)Q * C));
        fs_c = 1;
        fs_s = (size_t)C;
    }
    const float g = gout[t];
    const IdxT *ip = idx + ((size_t)b * Q + q) * K;
    const float *f = feat + (size_t)b * C * S + (size_t)c * fs_c;
    const unsigned Su = (unsigned)S;
    int best = (int)__ldg(ip);
    float m = __ldg(f + (size_t)min((unsigned)best, Su - 1) * fs_s);
    for (int k = 1; k < K; ++k) {
        const int s = (int)__ldg(ip + k);
        const float v = __ldg(f + (size_t)min((unsigned)s, Su - 1) * fs_s);
        if ((v > m || v != v) && !(m != m)) {
            m = v;
            best = s;
        }
    }
    // an out-of-range neighbour never writes outside grad_feat (torch.gather raises a device assert;
    // FFB6D_CHECK_INDICES=1 / ffb6d_check_indices report it)
    if ((unsigned)best < (unsigned)S) atomicAdd(gfeat + (size_t)b * C * S + (size_t)c * fs_c + (size_t)best * fs_s, g);
}

// K == 1, NCS layout: grad_feat[b,c,idx[b,q]] += grad_out[b,c,q].  Consecutive queries often share their source
// (nearest_interpolation of an image level: ~5-10 neighbouring pixels per cloud point), so a warp first sums each run
// of equal indices with a segmented shuffle scan and only the last lane of a run issues the atomic: 5-10x fewer
// atomics on the hottest addresses.
template <typename IdxT>
__global__ void __launch_bounds__(256)
gather1_bwd_runs_kernel(const IdxT *__restrict__ idx, const float *__restrict__ gout, float *__restrict__ gfeat, int C, int S,
                        int Q)
{
    const int b = blockIdx.z, c = blockIdx.y;
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool on = q < Q;
    const int key = on ? (int)__ldg(idx + (size_t)b * Q + q) : -1 - lane;          // off lanes: unique keys
    float v = on ? __ldg(gout + ((size_t)b * C + c) * Q + q) : 0.f;
    const int prev = __shfl_up_sync(0xffffffffu, key, 1);
    const bool head = lane == 0 || prev != key;
    // distance to the head of my run, then a segmented inclusive scan
    unsigned heads = __ballot_sync(0xffffffffu, head);
    const int start = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));           // lane of my run's head
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane - o >= start) v += u;
    }
    const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
    if (on && tail && (unsigned)key < (unsigned)S) atomicAdd(gfeat + ((size_t)b * C + c) * S + key, v);
}

// ------------------------------------------------------------------ neighbour gather
// out[b,n,k,:] = pc[b,idx[b,n,k],:]; one thread per output float (4 when D%4==0)
template <typename IdxT, int VEC>
__global__ void __launch_bounds__(256)
gather_neighbour_kernel(const float *__restrict__ pc, const IdxT *__restrict__ idx,
                        float *__restrict__ out, int S, int D, long long rows_per_b,
                        long long total_vec)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total_vec) return;
    const int dv = D / VEC;
    const long long row = t / dv;  // (b*N + n)*K + k
    const int j = (int)(t % dv) * VEC;
    const int b = (int)(row / rows_per_b);
    const int s = (int)__ldg(idx + row);
    const float *src = pc + ((size_t)b * S + s) * D + j;
    float *dst = out + (size_t)row * D + j;
    if constexpr (VEC == 4) {
        *reinterpret_cast<float4 *>(dst) = __ldg(reinterpret_cast<const float4 *>(src));
    } else {
        *dst = __ldg(src);
    }
}

// The scatter-add runs in float64: every source element receives up to N * K terms in whatever order the
// atomics land, and in fp32 a sum that nearly cancels would depend on that order.  The float64 sum carries
// 29 more bits than the fp32 result, so its order-dependent round-off stays far below the final rounding.
template <typename IdxT>
__global__ void __launch_bounds__(256)
gather_neighbour_bwd_kernel(const float *__restrict__ gout, const IdxT *__restrict__ idx,
                            double *__restrict__ acc, int S, int D, long long rows_per_b,
                            long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const long long row = t / D;
    const int j = (int)(t % D);
    const int b = (int)(row / rows_per_b);
    const int s = (int)__ldg(idx + row);
    if ((unsigned)s < (unsigned)S) atomicAdd(acc + ((size_t)b * S + s) * D + j, (double)gout[t]);
}

__global__ void __launch_bounds__(256)
round_to_f32_kernel(const double *__restrict__ acc, float *__restrict__ out, long long n)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) out[t] = __double2float_rn(acc[t]);
}

// ------------------------------------------------------------------ relative position encoding
// out[b,n,k,0..9] = [dist, dx,dy,dz, x_n,y_n,z_n, x_j,y_j,z_j]   (RandLANet.py:216-223)
template <typename IdxT>
__global__ void __launch_bounds__(256)
rel_pos_enc_kernel(const float *__restrict__ xyz, const IdxT *__restrict__ idx,
                   float *__restrict__ out, int N, int K, long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // (b*N+n)*K+k
    if (t >= total) return;
    const long long bn = t / K;
    const int b = (int)(bn / N);
    const int j = (int)__ldg(idx + t);
    const float *pc = xyz + (size_t)bn * 3;
    const float *pn = xyz + ((size_t)b * N + j) * 3;
    const float cx = __ldg(pc), cy = __ldg(pc + 1), cz = __ldg(pc + 2);
    const float nx = __ldg(pn), ny = __ldg(pn + 1), nz = __ldg(pn + 2);
    const float dx = __fsub_rn(cx, nx), dy = __fsub_rn(cy, ny), dz = __fsub_rn(cz, nz);
    const float ss = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    float *o = out + (size_t)t * 10;
    o[0] = __fsqrt_rn(ss);
    o[1] = dx;
    o[2] = dy;
    o[3] = dz;
    o[4] = cx;
    o[5] = cy;
    o[6] = cz;
    o[7] = nx;
    o[8] = ny;
    o[9] = nz;
}

// channel-major variant: out[b, j, n, k], j = 0..9 (coalesced along k/n per channel plane)
template <typename IdxT>
__global__ void __launch_bounds__(256)
rel_pos_enc_cm_kernel(const float *__restrict__ xyz, const IdxT *__restrict__ idx,
                      float *__restrict__ out, int N, int K, long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // (b*N+n)*K+k
    if (t >= total) return;
    const long long bn = t / K;
    const int b = (int)(bn / N);
    const long long plane = (long long)N * K;
    const long long within = t - (long long)b * plane;   // n*K + k
    const int j = (int)__ldg(idx + t);
    const float *pc = xyz + (size_t)bn * 3;
    const float *pn = xyz + ((size_t)b * N + j) * 3;
    const float cx = __ldg(pc), cy = __ldg(pc + 1), cz = __ldg(pc + 2);
    const float nx = __ldg(pn), ny = __ldg(pn + 1), nz = __ldg(pn + 2);
    const float dx = __fsub_rn(cx, nx), dy = __fsub_rn(cy, ny), dz = __fsub_rn(cz, nz);
    const float ss = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    float *o = out + (size_t)b * 10 * plane + within;
    o[0 * plane] = __fsqrt_rn(ss);
    o[1 * plane] = dx;
    o[2 * plane] = dy;
    o[3 * plane] = dz;
    o[4 * plane] = cx;
    o[5 * plane] = cy;
    o[6 * plane] = cz;
    o[7 * plane] = nx;
    o[8 * plane] = ny;
    o[9 * plane] = nz;
}

// ------------------------------------------------------------------ attentive pooling core
// out[b,c,n] = sum_k f[b,c,n,k] * softmax_k(att[b,c,n,:])[k]   (models/RandLA/RandLANet.py:245-248:
// softmax(dim=3) -> mul -> sum(dim=3)); one thread per (b,c,n), the K values of f and att are
// contiguous (two coalesced 4K-byte reads).  softmax as torch computes it: exp(x - max) / sum.
template <int KT>
__global__ void __launch_bounds__(256)
att_pool_kernel(const float *__restrict__ f1, int C1, const float *__restrict__ f2, int C2,
                const float *__restrict__ att, int N, int K, float *__restrict__ out, long long total)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // (b*C + c)*N + n
    if (t >= total) return;
    const int C = C1 + C2;
    const int n = (int)(t % N);
    const int c = (int)((t / N) % C);
    const int b = (int)(t / ((long long)N * C));
    const float *fp = (c < C1) ? f1 + (((size_t)b * C1 + c) * N + n) * K
                               : f2 + (((size_t)b * C2 + (c - C1)) * N + n) * K;
    const float *ap = att + (size_t)t * K;
    float fv[KT > 0 ? KT : 1], av[KT > 0 ? KT : 1];
    if constexpr (KT > 0) {
        if ((KT % 4 == 0) && ((reinterpret_cast<uintptr_t>(fp) & 15) == 0) && ((reinterpret_cast<uintptr_t>(ap) & 15) == 0)) {
#pragma unroll
            for (int k = 0; k < KT / 4; ++k) {
                const float4 u = __ldg(reinterpret_cast<const float4 *>(fp) + k);
                const float4 v = __ldg(reinterpret_cast<const float4 *>(ap) + k);
                fv[4 * k] = u.x; fv[4 * k + 1] = u.y; fv[4 * k + 2] = u.z; fv[4 * k + 3] = u.w;
                av[4 * k] = v.x; av[4 * k + 1] = v.y; av[4 * k + 2] = v.z; av[4 * k + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int k = 0; k < KT; ++k) {
                fv[k] = __ldg(fp + k);
                av[k] = __ldg(ap + k);
            }
        }
        float m = av[0];
#pragma unroll
        for (int k = 1; k < KT; ++k) m = fmaxf(m, av[k]);
        float den = 0.f, num = 0.f;
        // torch: scores = exp(a - m) / sum; f_agg = sum_k f * scores  -> same operation order
        float e[KT];
#pragma unroll
        for (int k = 0; k < KT; ++k) {
            e[k] = expf(av[k] - m);
            den += e[k];
        }
#pragma unroll
        for (int k = 0; k < KT; ++k) num += fv[k] * (e[k] / den);
        out[t] = num;
    } else {
        float m = __ldg(ap);
        for (int k = 1; k < K; ++k) m = fmaxf(m, __ldg(ap + k));
        float den = 0.f;
        for (int k = 0; k < K; ++k) den += expf(__ldg(ap + k) - m);
        float num = 0.f;
        for (int k = 0; k < K; ++k) num += __ldg(fp + k) * (expf(__ldg(ap + k) - m) / den);
        out[t] = num;
    }
}

// ------------------------------------------------------------------ index validation (debugging aid)
// The gather kernels trust their indices (an out-of-range neighbour reads stale shared memory or a
// foreign row where torch.gather raises a device assert).  This pass counts the offenders; it is run
// by ffb6d_check_indices and, with FFB6D_CHECK_INDICES=1, in front of every gather entry point.
template <typename IdxT>
__global__ void __launch_bounds__(256)
check_indices_kernel(const IdxT *__restrict__ idx, long long n, long long S, unsigned long long *__restrict__ bad)
{
    unsigned long long mine = 0;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const long long v = (long long)idx[t];
        mine += (v < 0 || v >= S) ? 1ull : 0ull;
    }
    if (mine) atomicAdd(bad, mine);
}

static int check_indices_sync(const void *idx, int idx_is_i64, long long n, long long S, cudaStream_t st, const char *who)
{
    if (n <= 0) return FFB6D_OK;
    static unsigned long long *flag[kMaxDevices] = {nullptr};
    const int dev = current_device() & (kMaxDevices - 1);
    if (!flag[dev]) FFB6D_CUDA(cudaMalloc(&flag[dev], sizeof(unsigned long long)));
    FFB6D_CUDA(cudaMemsetAsync(flag[dev], 0, sizeof(unsigned long long), st));
    const unsigned blocks = (unsigned)std::min<long long>(ceil_div(n, 256), 4 * num_sms());
    if (idx_is_i64)
        check_indices_kernel<long long><<<blocks, 256, 0, st>>>((const long long *)idx, n, S, flag[dev]);
    else
        check_indices_kernel<int><<<blocks, 256, 0, st>>>((const int *)idx, n, S, flag[dev]);
    FFB6D_LAUNCH_OK("check_indices_kernel");
    unsigned long long bad = 0;
    FFB6D_CUDA(cudaMemcpyAsync(&bad, flag[dev], sizeof(bad), cudaMemcpyDeviceToHost, st));
    FFB6D_CUDA(cudaStreamSynchronize(st));
    if (bad) {
        set_error("%s: %llu of %lld indices outside [0, %lld)", who, bad, n, S);
        return FFB6D_ERR_INVALID;
    }
    return FFB6D_OK;
}

// ------------------------------------------------------------------ host-side launch logic
static int max_smem_optin() { return device_info().max_smem_optin; }

// Channels per CTA of the staged kernels for a gather with KT neighbours (0: any K without a K-lane kernel), or 0
// when the rows are not staged: rows longer than half the shared memory (two CTAs per SM hide the staging latency),
// few queries against long rows (Q*K gathered elements << S: staging whole rows would read far more than the ~5
// sectors a query's K adjacent neighbours touch per row -> K-lane gather instead), or more channel chunks than
// grid.y holds (65535; the direct and K-lane kernels take every C the entry point admits).
static int staged_channels(int64_t B, int64_t C, int64_t S, int64_t Q, int KT)
{
    const size_t budget = (size_t)(max_smem_optin() - 1024) / 2;
    const size_t row_bytes = (size_t)S * sizeof(float);
    const bool sparse_queries = (KT == 8 || KT == 16 || KT == 32) && Q * 40 < S;
    if (C < 1 || row_bytes > budget || sparse_queries) return 0;
    const int64_t want = 4 * num_sms();   // CTAs to aim for
    int CC = (int)(budget / row_bytes);
    if (CC > C) CC = (int)C;
    // the K indices of a query are re-read once per channel chunk: keep chunks wide when K
    // is large (index bytes ~ K/CC of the output bytes), narrow when K == 1
    const int cc_cap = (KT == 1) ? 8 : 32;
    if (CC > cc_cap) CC = cc_cap;
    if (KT != 1)
        while (CC > 4 && B * ceil_div(C, CC) < want) CC = (CC + 1) / 2;
    return ceil_div(C, CC) <= 65535 ? CC : 0;
}

template <typename IdxT, int KT>
static int launch_ncs(const float *feat, const IdxT *idx, float *out, int64_t B, int64_t C,
                      int64_t S, int64_t Q, int K, cudaStream_t st)
{
    const size_t row_bytes = (size_t)S * sizeof(float);
    const int64_t want = 4 * num_sms();   // CTAs to aim for
    const int CC = staged_channels(B, C, S, Q, KT);
    if (CC) {
        const int64_t ctas = B * ceil_div(C, CC);
        int64_t nq = ctas < want ? ceil_div(want, ctas) : 1;
        // every query chunk stages the rows again: keep a chunk at least 4 rows long
        int64_t q_per_cta = ceil_div(Q, nq);
        const int64_t q_min = std::max<int64_t>(1024, 4 * S);
        if (q_per_cta < q_min) q_per_cta = q_min;
        q_per_cta = ceil_div(q_per_cta, 1024) * 1024;
        nq = ceil_div(Q, q_per_cta);
        const size_t smem = (size_t)CC * row_bytes;
        dim3 grid((unsigned)nq, (unsigned)ceil_div(C, CC), (unsigned)B);
        if constexpr (KT == 1) {
            const bool v4 = (Q % 4 == 0) && ((reinterpret_cast<uintptr_t>(idx) & 15) == 0) &&
                            ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
            if (v4) {
                auto kern = gather1_ncs_staged_v4_kernel<IdxT>;
                FFB6D_OPTIN_SMEM(kern, max_smem_optin() - 1024);
                kern<<<grid, 256, smem, st>>>(feat, idx, out, (int)C, (int)S, (int)Q, CC, (int)q_per_cta);
                FFB6D_LAUNCH_OK("gather1_ncs_staged_v4_kernel");
                return FFB6D_OK;
            }
        }
        auto kern = gather_max_ncs_staged_kernel<IdxT, KT>;
        FFB6D_OPTIN_SMEM(kern, max_smem_optin() - 1024);   // per instantiation and device; not a stream op
        kern<<<grid, 256, smem, st>>>(feat, idx, out, (int)C, (int)S, (int)Q, K, CC,
                                      (int)q_per_cta);
        FFB6D_LAUNCH_OK("gather_max_ncs_staged_kernel");
    } else if (KT == 1) {
        dim3 grid((unsigned)ceil_div(Q, 256), (unsigned)std::min<int64_t>(ceil_div(C, G1_CH), 65535), (unsigned)B);
        gather1_ncs_direct_kernel<IdxT><<<grid, 256, 0, st>>>(feat, idx, out, (int)C, (int)S, (int)Q);
        FFB6D_LAUNCH_OK("gather1_ncs_direct_kernel");
    } else if constexpr (KT == 8 || KT == 16 || KT == 32) {
        dim3 grid((unsigned)ceil_div(Q, 256 / KT), (unsigned)ceil_div(C, KLANE_CH), (unsigned)B);
        gather_max_ncs_klane_kernel<IdxT, KT><<<grid, 256, 0, st>>>(feat, idx, out, (int)C, (int)S, (int)Q);
        FFB6D_LAUNCH_OK("gather_max_ncs_klane_kernel");
    } else {
        const int CC = 8;
        dim3 grid((unsigned)ceil_div(Q, 256), (unsigned)ceil_div(C, CC), (unsigned)B);
        gather_max_ncs_direct_kernel<IdxT, KT>
            <<<grid, 256, 0, st>>>(feat, idx, out, (int)C, (int)S, (int)Q, K, CC);
        FFB6D_LAUNCH_OK("gather_max_ncs_direct_kernel");
    }
    return FFB6D_OK;
}

template <typename IdxT>
static int gather_max_fwd_t(const float *feat, const IdxT *idx, int64_t B, int64_t C, int64_t S,
                            int64_t Q, int K, int layout, float *out, cudaStream_t st)
{
    if (layout == FFB6D_LAYOUT_NSC) {
        const long long total_q = (long long)B * Q;
        const int warps = 8;
        gather_max_nsc_kernel<IdxT><<<(unsigned)ceil_div(total_q, warps), warps * 32, 0, st>>>(
            feat, idx, out, (int)C, (int)S, (int)Q, K, total_q);
        FFB6D_LAUNCH_OK("gather_max_nsc_kernel");
        return FFB6D_OK;
    }
    const bool aligned = (reinterpret_cast<uintptr_t>(idx) & 15) == 0;
    if (K == 1) return launch_ncs<IdxT, 1>(feat, idx, out, B, C, S, Q, K, st);
    if (K == 8 && aligned) return launch_ncs<IdxT, 8>(feat, idx, out, B, C, S, Q, K, st);
    if (K == 16 && aligned) return launch_ncs<IdxT, 16>(feat, idx, out, B, C, S, Q, K, st);
    if (K == 32 && aligned) return launch_ncs<IdxT, 32>(feat, idx, out, B, C, S, Q, K, st);
    return launch_ncs<IdxT, 0>(feat, idx, out, B, C, S, Q, K, st);
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" {

const char *ffb6d_gather_kernel_name(int64_t B, int64_t C, int64_t S, int64_t Q, int K, int layout)
{
    // mirrors gather_max_fwd_t / launch_ncs (aligned pointers assumed)
    if (layout == FFB6D_LAYOUT_NSC) return "gather_max_nsc_kernel";
    const bool klane = K == 8 || K == 16 || K == 32;
    const bool staged = staged_channels(B, C, S, Q, (K == 1 || klane) ? K : 0) != 0;
    if (K == 1) return staged ? ((Q % 4 == 0) ? "gather1_ncs_staged_v4_kernel" : "gather_max_ncs_staged_kernel")
                              : "gather1_ncs_direct_kernel";
    if (staged) return "gather_max_ncs_staged_kernel";
    if (klane) return "gather_max_ncs_klane_kernel";
    return "gather_max_ncs_direct_kernel";
}

int ffb6d_gather_max_fwd(const float *feat, const void *idx, int idx_is_i64, int64_t B, int64_t C,
                         int64_t S, int64_t Q, int K, int layout, float *out,
                         ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && C >= 0 && S >= 0 && Q >= 0, "gather_max_fwd: negative size");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "gather_max_fwd: K=%d outside [1,%d]", K,
                    FFB6D_MAX_K);
    FFB6D_CHECK_ARG(layout == FFB6D_LAYOUT_NCS || layout == FFB6D_LAYOUT_NSC,
                    "gather_max_fwd: unknown layout %d", layout);
    FFB6D_CHECK_ARG(S < (1ll << 31) && Q < (1ll << 31) && C < (1ll << 31) && B < 65536 &&
                        C <= 65535ll * 8,
                    "gather_max_fwd: size too large");
    // the channels-last kernel takes 8 queries per block in grid.x (at most 2^31 - 1 blocks)
    FFB6D_CHECK_ARG(layout != FFB6D_LAYOUT_NSC || B * Q <= 8ll * 0x7fffffff,
                    "gather_max_fwd: B*Q=%lld too large for the channels-last layout", (long long)(B * Q));
    if (B == 0 || C == 0 || Q == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(S > 0, "gather_max_fwd: empty source with non-empty index");
    FFB6D_CHECK_ARG(feat && idx && out, "gather_max_fwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (env().check_indices) {
        const int rc = check_indices_sync(idx, idx_is_i64, (long long)B * Q * K, S, st, "gather_max_fwd");
        if (rc) return rc;
    }
    if (idx_is_i64)
        return gather_max_fwd_t<long long>(feat, (const long long *)idx, B, C, S, Q, K, layout, out, st);
    return gather_max_fwd_t<int>(feat, (const int *)idx, B, C, S, Q, K, layout, out, st);
}

int ffb6d_check_indices(const void *idx, int idx_is_i64, int64_t count, int64_t S, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(count >= 0 && S >= 0, "check_indices: negative size");
    if (count == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(idx, "check_indices: null pointer");
    return check_indices_sync(idx, idx_is_i64, (long long)count, (long long)S, (cudaStream_t)stream, "check_indices");
}

int ffb6d_gather_max_bwd(const float *feat, const void *idx, int idx_is_i64, const float *grad_out,
                         int64_t B, int64_t C, int64_t S, int64_t Q, int K, int layout,
                         float *grad_feat, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && C >= 0 && S >= 0 && Q >= 0, "gather_max_bwd: negative size");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "gather_max_bwd: K=%d outside [1,%d]", K,
                    FFB6D_MAX_K);
    FFB6D_CHECK_ARG(layout == FFB6D_LAYOUT_NCS || layout == FFB6D_LAYOUT_NSC,
                    "gather_max_bwd: unknown layout %d", layout);
    cudaStream_t st = (cudaStream_t)stream;
    if (B * C * S > 0) {
        FFB6D_CHECK_ARG(grad_feat, "gather_max_bwd: null grad_feat");
        FFB6D_CUDA(cudaMemsetAsync(grad_feat, 0, (size_t)B * C * S * sizeof(float), st));
    }
    if (B == 0 || C == 0 || Q == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(S > 0, "gather_max_bwd: empty source with non-empty index");
    FFB6D_CHECK_ARG(feat && idx && grad_out, "gather_max_bwd: null pointer");
    if (env().check_indices) {
        const int rc = check_indices_sync(idx, idx_is_i64, (long long)B * Q * K, S, st, "gather_max_bwd");
        if (rc) return rc;
    }
    if (K == 1 && layout == FFB6D_LAYOUT_NCS && C <= 65535) {   // max over one element: a pure scatter-add, run-aggregated
        dim3 grid((unsigned)ceil_div(Q, 256), (unsigned)C, (unsigned)B);
        if (idx_is_i64)
            gather1_bwd_runs_kernel<long long><<<grid, 256, 0, st>>>((const long long *)idx, grad_out, grad_feat, (int)C, (int)S, (int)Q);
        else
            gather1_bwd_runs_kernel<int><<<grid, 256, 0, st>>>((const int *)idx, grad_out, grad_feat, (int)C, (int)S, (int)Q);
        FFB6D_LAUNCH_OK("gather1_bwd_runs_kernel");
        return FFB6D_OK;
    }
    const long long total = (long long)B * C * Q;
    const unsigned blocks = (unsigned)ceil_div(total, 256);
    if (idx_is_i64)
        gather_max_bwd_kernel<long long><<<blocks, 256, 0, st>>>(
            feat, (const long long *)idx, grad_out, grad_feat, (int)C, (int)S, (int)Q, K, layout, total);
    else
        gather_max_bwd_kernel<int><<<blocks, 256, 0, st>>>(feat, (const int *)idx, grad_out, grad_feat,
                                                          (int)C, (int)S, (int)Q, K, layout, total);
    FFB6D_LAUNCH_OK("gather_max_bwd_kernel");
    return FFB6D_OK;
}

int ffb6d_gather_neighbour_fwd(const float *pc, const void *idx, int idx_is_i64, int64_t B,
                               int64_t S, int64_t D, int64_t N, int K, float *out,
                               ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && S >= 0 && D >= 0 && N >= 0 && K >= 0,
                    "gather_neighbour_fwd: negative size");
    if (B == 0 || D == 0 || N == 0 || K == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(S > 0, "gather_neighbour_fwd: empty source with non-empty index");
    FFB6D_CHECK_ARG(pc && idx && out, "gather_neighbour_fwd: null pointer");
    FFB6D_CHECK_ARG(S < (1ll << 31) && D < (1ll << 31), "gather_neighbour_fwd: size too large");
    cudaStream_t st = (cudaStream_t)stream;
    if (env().check_indices) {
        const int rc = check_indices_sync(idx, idx_is_i64, (long long)B * N * K, S, st, "gather_neighbour_fwd");
        if (rc) return rc;
    }
    const long long rows_per_b = (long long)N * K;
    const bool v4 = (D % 4 == 0) && ((reinterpret_cast<uintptr_t>(pc) & 15) == 0) &&
                    ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    const long long total = (long long)B * rows_per_b * (v4 ? D / 4 : D);
    const unsigned blocks = (unsigned)ceil_div(total, 256);
    if (idx_is_i64) {
        if (v4)
            gather_neighbour_kernel<long long, 4><<<blocks, 256, 0, st>>>(
                pc, (const long long *)idx, out, (int)S, (int)D, rows_per_b, total);
        else
            gather_neighbour_kernel<long long, 1><<<blocks, 256, 0, st>>>(
                pc, (const long long *)idx, out, (int)S, (int)D, rows_per_b, total);
    } else {
        if (v4)
            gather_neighbour_kernel<int, 4><<<blocks, 256, 0, st>>>(pc, (const int *)idx, out, (int)S,
                                                                   (int)D, rows_per_b, total);
        else
            gather_neighbour_kernel<int, 1><<<blocks, 256, 0, st>>>(pc, (const int *)idx, out, (int)S,
                                                                   (int)D, rows_per_b, total);
    }
    FFB6D_LAUNCH_OK("gather_neighbour_kernel");
    return FFB6D_OK;
}

int ffb6d_gather_neighbour_bwd(const float *grad_out, const void *idx, int idx_is_i64, int64_t B,
                               int64_t S, int64_t D, int64_t N, int K, float *grad_pc,
                               ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && S >= 0 && D >= 0 && N >= 0 && K >= 0,
                    "gather_neighbour_bwd: negative size");
    cudaStream_t st = (cudaStream_t)stream;
    if (B * S * D > 0) {
        FFB6D_CHECK_ARG(grad_pc, "gather_neighbour_bwd: null grad_pc");
        FFB6D_CUDA(cudaMemsetAsync(grad_pc, 0, (size_t)B * S * D * sizeof(float), st));
    }
    if (B == 0 || D == 0 || N == 0 || K == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(S > 0, "gather_neighbour_bwd: empty source with non-empty index");
    FFB6D_CHECK_ARG(grad_out && idx, "gather_neighbour_bwd: null pointer");
    const long long rows_per_b = (long long)N * K;
    const long long total = (long long)B * rows_per_b * D;
    const long long n_out = (long long)B * S * D;
    double *acc = nullptr;
    FFB6D_CUDA(cudaMallocAsync((void **)&acc, (size_t)n_out * sizeof(double), st));
    cudaError_t e = cudaMemsetAsync(acc, 0, (size_t)n_out * sizeof(double), st);
    if (e == cudaSuccess) {
        const unsigned blocks = (unsigned)ceil_div(total, 256);
        if (idx_is_i64)
            gather_neighbour_bwd_kernel<long long><<<blocks, 256, 0, st>>>(
                grad_out, (const long long *)idx, acc, (int)S, (int)D, rows_per_b, total);
        else
            gather_neighbour_bwd_kernel<int><<<blocks, 256, 0, st>>>(grad_out, (const int *)idx, acc,
                                                                    (int)S, (int)D, rows_per_b, total);
        e = cudaGetLastError();
        if (e == cudaSuccess) {
            count_launch();
            round_to_f32_kernel<<<(unsigned)ceil_div(n_out, 256), 256, 0, st>>>(acc, grad_pc, n_out);
        }
    }
    cudaFreeAsync(acc, st);
    if (e != cudaSuccess) {
        set_error("gather_neighbour_bwd: %s", cudaGetErrorString(e));
        return FFB6D_ERR_CUDA;
    }
    FFB6D_LAUNCH_OK("round_to_f32_kernel");
    return FFB6D_OK;
}

int ffb6d_relative_pos_encoding_fwd(const float *xyz, const void *idx, int idx_is_i64, int64_t B,
                                    int64_t N, int K, float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && N >= 0 && K >= 0, "relative_pos_encoding_fwd: negative size");
    if (B == 0 || N == 0 || K == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(xyz && idx && out, "relative_pos_encoding_fwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const long long total = (long long)B * N * K;
    const unsigned blocks = (unsigned)ceil_div(total, 256);
    if (idx_is_i64)
        rel_pos_enc_kernel<long long><<<blocks, 256, 0, st>>>(xyz, (const long long *)idx, out, (int)N,
                                                             K, total);
    else
        rel_pos_enc_kernel<int><<<blocks, 256, 0, st>>>(xyz, (const int *)idx, out, (int)N, K, total);
    FFB6D_LAUNCH_OK("rel_pos_enc_kernel");
    return FFB6D_OK;
}

int ffb6d_relative_pos_encoding_cm_fwd(const float *xyz, const void *idx, int idx_is_i64, int64_t B,
                                       int64_t N, int K, float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && N >= 0 && K >= 0, "relative_pos_encoding_cm_fwd: negative size");
    if (B == 0 || N == 0 || K == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(xyz && idx && out, "relative_pos_encoding_cm_fwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const long long total = (long long)B * N * K;
    const unsigned blocks = (unsigned)ceil_div(total, 256);
    if (idx_is_i64)
        rel_pos_enc_cm_kernel<long long><<<blocks, 256, 0, st>>>(xyz, (const long long *)idx, out, (int)N, K, total);
    else
        rel_pos_enc_cm_kernel<int><<<blocks, 256, 0, st>>>(xyz, (const int *)idx, out, (int)N, K, total);
    FFB6D_LAUNCH_OK("rel_pos_enc_cm_kernel");
    return FFB6D_OK;
}

int ffb6d_att_pool_fwd(const float *f1, int64_t C1, const float *f2, int64_t C2, const float *att, int64_t B,
                       int64_t N, int K, float *out, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && C1 >= 1 && C2 >= 0 && N >= 0, "att_pool_fwd: bad size");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "att_pool_fwd: K=%d outside [1,%d]", K, FFB6D_MAX_K);
    if (B == 0 || N == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(f1 && att && out && (C2 == 0 || f2), "att_pool_fwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const long long total = (long long)B * (C1 + C2) * N;
    const unsigned blocks = (unsigned)ceil_div(total, 256);
    if (K == 16)
        att_pool_kernel<16><<<blocks, 256, 0, st>>>(f1, (int)C1, f2, (int)C2, att, (int)N, K, out, total);
    else if (K == 8)
        att_pool_kernel<8><<<blocks, 256, 0, st>>>(f1, (int)C1, f2, (int)C2, att, (int)N, K, out, total);
    else if (K == 32)
        att_pool_kernel<32><<<blocks, 256, 0, st>>>(f1, (int)C1, f2, (int)C2, att, (int)N, K, out, total);
    else
        att_pool_kernel<0><<<blocks, 256, 0, st>>>(f1, (int)C1, f2, (int)C2, att, (int)N, K, out, total);
    FFB6D_LAUNCH_OK("att_pool_kernel");
    return FFB6D_OK;
}

}  // extern "C"
