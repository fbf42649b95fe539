// pose.cu -- keypoint voting (mean shift) and least-squares pose fitting on the device (sm_90a).
//
// The step right after the network (SURVEY.md §8 f-4): every point of an object votes for the
// object's keypoints and centre, the votes are clustered with a Gaussian mean shift
// (MeanShiftTorch.fit, ffb6d/utils/meanshift_pytorch.py:28-57) and the cluster centres are aligned
// with the mesh keypoints by a least-squares rigid fit (best_fit_transform,
// ffb6d/utils/pvn3d_eval_utils_kpls.py:28-59).  The reference materialises the N x N distance and
// weight matrices in HBM every iteration (3 x 600 MB at N = 12288) and synchronises with the host
// once per iteration for the stop test; one call per keypoint, 9 calls per object.
//
// Here all G vote sets of an object are ONE persistent cooperative kernel: the modes live in L2
// (16 B per point, ping-pong), a CTA owns 128 points of one set at a time and streams the whole
// set through shared memory, the N x N matrix never exists, and the stop test is a device-side
// max + grid barrier.  The arithmetic is exp-bound (one MUFU.EX2 + ~11 FP32 per pair), not
// HBM-bound.  Results are floating point: sums run in a different order than torch's, so parity is
// by tolerance (tests/test_gpu_pose.py), never bitwise.
#include <algorithm>

#include "common.cuh"

namespace ffb6d {

constexpr int MS_THREADS = 256;
constexpr int MS_IT = 128;         // points of one work item (two per thread, four j-slices)
constexpr int MS_JT = 2048;        // points of one staged tile (32 KB)
constexpr int MS_MAX_G = 64;       // vote sets per call

struct MsGroup {
    int n;                          // valid points
    int iters;                      // iterations run
    unsigned shift[3];              // max |new - old| of an iteration (float bits), rotating slots
    unsigned pad;
    unsigned long long best;        // (count << 32) | ~index of the densest mode
};

__device__ __forceinline__ void grid_sync(unsigned *counter, unsigned &target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        __threadfence();
        atomicAdd(counter, 1u);
        unsigned v;
        do {
            asm volatile("ld.acquire.gpu.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
        } while ((int)(v - target) < 0);
        __threadfence();
    }
    __syncthreads();
}

__device__ __forceinline__ float4 ldcg4(const float4 *p) { return __ldcg(p); }

// 2^x on the SFU without exp2f's denormal-range fix-up (3 extra instructions per call): weights below 2^-126 flush
// to zero, and a weight of 1e-38 against the point's own weight of 1 is below fp32 resolution anyway
__device__ __forceinline__ float ex2_ftz(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// MODE 0: one mean-shift update of the item's points; MODE 1: neighbours within the bandwidth
template <int MODE>
__device__ __forceinline__ void ms_item(const float4 *__restrict__ cur, float4 *__restrict__ nxt, int n, int tile,
                                        float neg_scale, float bw, float4 *s_tile, float (*s_part)[MS_IT][4],
                                        float &cta_max, unsigned long long &cta_best)
{
    const int t = threadIdx.x, il = t & 63, slice = t >> 6;
    const int i0 = tile * MS_IT + il, i1 = i0 + 64;
    const float4 p0 = i0 < n ? ldcg4(cur + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 p1 = i1 < n ? ldcg4(cur + i1) : make_float4(0.f, 0.f, 0.f, 0.f);
    float a0x = 0.f, a0y = 0.f, a0z = 0.f, a0w = 0.f, a1x = 0.f, a1y = 0.f, a1z = 0.f, a1w = 0.f;
    for (int j0 = 0; j0 < n; j0 += MS_JT) {
        const int jn = min(MS_JT, n - j0);
        __syncthreads();
        for (int j = t; j < jn; j += MS_THREADS) s_tile[j] = ldcg4(cur + j0 + j);
        __syncthreads();
#pragma unroll 4
        for (int j = slice; j < jn; j += 4) {
            const float4 c = s_tile[j];            // the warp reads one address: a broadcast
            float dx = p0.x - c.x, dy = p0.y - c.y, dz = p0.z - c.z;
            const float d0 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            dx = p1.x - c.x, dy = p1.y - c.y, dz = p1.z - c.z;
            const float d1 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            if (MODE == 0) {
                const float w0 = ex2_ftz(d0 * neg_scale), w1 = ex2_ftz(d1 * neg_scale);
                a0x = fmaf(w0, c.x, a0x), a0y = fmaf(w0, c.y, a0y), a0z = fmaf(w0, c.z, a0z), a0w += w0;
                a1x = fmaf(w1, c.x, a1x), a1y = fmaf(w1, c.y, a1y), a1z = fmaf(w1, c.z, a1z), a1w += w1;
            } else {
                a0w += (sqrtf(d0) < bw) ? 1.f : 0.f;   // counts stay exact in fp32 (n < 2^24)
                a1w += (sqrtf(d1) < bw) ? 1.f : 0.f;
            }
        }
    }
    s_part[slice][il][0] = a0x, s_part[slice][il][1] = a0y, s_part[slice][il][2] = a0z, s_part[slice][il][3] = a0w;
    s_part[slice][il + 64][0] = a1x, s_part[slice][il + 64][1] = a1y, s_part[slice][il + 64][2] = a1z, s_part[slice][il + 64][3] = a1w;
    __syncthreads();
    if (t < MS_IT) {
        const int i = tile * MS_IT + t;
        if (i < n) {
            float sx = 0.f, sy = 0.f, sz = 0.f, sw = 0.f;
#pragma unroll
            for (int s = 0; s < 4; ++s) sx += s_part[s][t][0], sy += s_part[s][t][1], sz += s_part[s][t][2], sw += s_part[s][t][3];
            if (MODE == 0) {
                const float4 p = ldcg4(cur + i);
                const float nx = sx / sw, ny = sy / sw, nz = sz / sw;      // sw >= 1: the point's own weight
                const float ex = nx - p.x, ey = ny - p.y, ez = nz - p.z;
                nxt[i] = make_float4(nx, ny, nz, 0.f);
                cta_max = fmaxf(cta_max, sqrtf(fmaf(ez, ez, fmaf(ey, ey, ex * ex))));
            } else {
                const unsigned long long key = ((unsigned long long)(unsigned)sw << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
                cta_best = max(cta_best, key);
            }
        }
    }
}

__global__ void __launch_bounds__(MS_THREADS, 2)
mean_shift_kernel(const float *__restrict__ votes, const unsigned char *__restrict__ valid, long long valid_stride, int G,
                  int N, float bandwidth, float stop_thresh, int max_iter, unsigned *__restrict__ barrier,
                  MsGroup *__restrict__ state, float4 *__restrict__ buf0, float4 *__restrict__ buf1, int *__restrict__ src,
                  float *__restrict__ centres, unsigned char *__restrict__ labels, int *__restrict__ iters_out,
                  float *__restrict__ modes)
{
    __shared__ float4 s_tile[MS_JT];
    __shared__ float s_part[4][MS_IT][4];
    __shared__ int s_first[MS_MAX_G + 1];     // first work item of every set this round
    __shared__ int s_n[MS_MAX_G], s_iters[MS_MAX_G];
    __shared__ unsigned char s_done[MS_MAX_G];
    __shared__ float s_red[MS_THREADS / 32];
    __shared__ unsigned long long s_red64[MS_THREADS / 32];
    __shared__ int s_scan[MS_THREADS / 32 + 1];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    unsigned target = 0;

    // ---- phase A: ordered compaction of the valid votes of every set (the reference's votes[mask]) ----
    for (int g = blockIdx.x; g < G; g += gridDim.x) {
        const unsigned char *v = valid ? valid + (size_t)g * valid_stride : nullptr;
        const float *src_pts = votes + (size_t)g * N * 3;
        float4 *dst = buf0 + (size_t)g * N;
        int base = 0;
        for (int i0 = 0; i0 < N; i0 += MS_THREADS) {
            const int i = i0 + t;
            const bool ok = i < N && (!v || v[i] != 0);
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            if (lane == 0) s_scan[wid + 1] = __popc(m);
            __syncthreads();
            if (t == 0) {
                s_scan[0] = 0;
                for (int w = 0; w < MS_THREADS / 32; ++w) s_scan[w + 1] += s_scan[w];
            }
            __syncthreads();
            if (ok) {
                const int k = base + s_scan[wid] + __popc(m & ((1u << lane) - 1u));
                dst[k] = make_float4(src_pts[3 * (size_t)i], src_pts[3 * (size_t)i + 1], src_pts[3 * (size_t)i + 2], 0.f);
                src[(size_t)g * N + k] = i;
            }
            if (i < N) {
                labels[(size_t)g * N + i] = 0;
                if (modes) modes[((size_t)g * N + i) * 3] = 0.f, modes[((size_t)g * N + i) * 3 + 1] = 0.f, modes[((size_t)g * N + i) * 3 + 2] = 0.f;
            }
            base += s_scan[MS_THREADS / 32];
            __syncthreads();
        }
        if (t == 0) state[g].n = base;
    }
    grid_sync(barrier, target);
    if (t < G) {
        int n;
        asm volatile("ld.acquire.gpu.s32 %0, [%1];" : "=r"(n) : "l"(&state[t].n) : "memory");
        s_n[t] = n, s_iters[t] = 0, s_done[t] = (n == 0);
    }
    __syncthreads();

    // ---- phase B: mean-shift rounds; every CTA derives the same work list from the same flags ----
    const float neg_scale = -0.5f * 1.4426950408889634f / (bandwidth * bandwidth);   // exp(-d^2 / 2bw^2) as exp2
    for (int it = 1; it <= max_iter + 1; ++it) {
        if (t == 0) {
            int acc = 0;
            for (int g = 0; g < G; ++g) {
                s_first[g] = acc;
                if (!s_done[g]) acc += (s_n[g] + MS_IT - 1) / MS_IT;
            }
            s_first[G] = acc;
        }
        __syncthreads();
        const int total = s_first[G];
        if (total == 0) break;
        if (blockIdx.x == 0 && t < G) state[t].shift[(it + 1) % 3] = 0u;       // the slot of the NEXT round
        for (int item = blockIdx.x; item < total; item += gridDim.x) {
            int g = 0;
            while (s_first[g + 1] <= item) ++g;
            const int par = s_iters[g] & 1;
            const float4 *cur = (par ? buf1 : buf0) + (size_t)g * N;
            float4 *nxt = (par ? buf0 : buf1) + (size_t)g * N;
            float cta_max = 0.f;
            unsigned long long unused = 0;
            ms_item<0>(cur, nxt, s_n[g], item - s_first[g], neg_scale, bandwidth, s_tile, s_part, cta_max, unused);
#pragma unroll
            for (int o = 16; o; o >>= 1) cta_max = fmaxf(cta_max, __shfl_xor_sync(0xffffffffu, cta_max, o));
            if (lane == 0) s_red[wid] = cta_max;
            __syncthreads();
            if (t == 0) {
                float m = 0.f;
                for (int w = 0; w < MS_THREADS / 32; ++w) m = fmaxf(m, s_red[w]);
                atomicMax(&state[g].shift[it % 3], __float_as_uint(m));       // non-negative floats order as unsigned
            }
        }
        grid_sync(barrier, target);
        if (t < G && !s_done[t]) {
            unsigned bits;
            asm volatile("ld.acquire.gpu.u32 %0, [%1];" : "=r"(bits) : "l"(&state[t].shift[it % 3]) : "memory");
            s_iters[t] = it;
            // the reference's `torch.max(Cdis) < stop_thresh or it > max_iter` (meanshift_pytorch.py:46)
            if (__uint_as_float(bits) < stop_thresh || it > max_iter) s_done[t] = 1;
        }
        __syncthreads();
    }

    // ---- phase C: the mode with the most modes within one bandwidth (first index on ties) ----
    __syncthreads();   // the `break` above leaves the loop right after reading s_first[G]: order that read before the rewrite
    if (t == 0) {
        int acc = 0;
        for (int g = 0; g < G; ++g) s_first[g] = acc, acc += (s_n[g] + MS_IT - 1) / MS_IT;
        s_first[G] = acc;
    }
    __syncthreads();
    for (int item = blockIdx.x; item < s_first[G]; item += gridDim.x) {
        int g = 0;
        while (s_first[g + 1] <= item) ++g;
        const float4 *cur = ((s_iters[g] & 1) ? buf1 : buf0) + (size_t)g * N;
        float unused = 0.f;
        unsigned long long best = 0;
        ms_item<1>(cur, nullptr, s_n[g], item - s_first[g], 0.f, bandwidth, s_tile, s_part, unused, best);
#pragma unroll
        for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (lane == 0) s_red64[wid] = best;
        __syncthreads();
        if (t == 0) {
            unsigned long long m = 0;
            for (int w = 0; w < MS_THREADS / 32; ++w) m = max(m, s_red64[w]);
            atomicMax(&state[g].best, m);
        }
    }
    grid_sync(barrier, target);

    // ---- phase D: centre, inlier labels (original point order), iteration counts ----
    for (int g = 0; g < G; ++g) {
        const int n = s_n[g];
        if (blockIdx.x == 0 && t == 0) {
            iters_out[g] = s_iters[g];
            if (n == 0) centres[3 * g] = 0.f, centres[3 * g + 1] = 0.f, centres[3 * g + 2] = 0.f;
        }
        if (n == 0) continue;
        const float4 *cur = ((s_iters[g] & 1) ? buf1 : buf0) + (size_t)g * N;
        unsigned long long best;
        asm volatile("ld.acquire.gpu.u64 %0, [%1];" : "=l"(best) : "l"(&state[g].best) : "memory");
        const int mi = (int)(0xFFFFFFFFu - (unsigned)(best & 0xFFFFFFFFull));
        const float4 c = ldcg4(cur + mi);
        if (blockIdx.x == 0 && t == 0) centres[3 * g] = c.x, centres[3 * g + 1] = c.y, centres[3 * g + 2] = c.z;
        for (int i = blockIdx.x * MS_THREADS + t; i < n; i += gridDim.x * MS_THREADS) {
            const float4 p = ldcg4(cur + i);
            const float dx = c.x - p.x, dy = c.y - p.y, dz = c.z - p.z;
            const int o = src[(size_t)g * N + i];
            labels[(size_t)g * N + o] = sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx))) < bandwidth;
            if (modes) modes[((size_t)g * N + o) * 3] = p.x, modes[((size_t)g * N + o) * 3 + 1] = p.y, modes[((size_t)g * N + o) * 3 + 2] = p.z;
        }
    }
}

// ---- least-squares rigid fit (Kabsch) of M point pairs, one thread per problem, fp64 like numpy ----
__global__ void best_fit_kernel(const float *__restrict__ A, const float *__restrict__ Bp, int G, int M, double *__restrict__ T)
{
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const float *a = A + (size_t)g * M * 3, *b = Bp + (size_t)g * M * 3;
    double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0};
    for (int m = 0; m < M; ++m)
        for (int d = 0; d < 3; ++d) ca[d] += (double)a[3 * m + d], cb[d] += (double)b[3 * m + d];
    for (int d = 0; d < 3; ++d) ca[d] /= (double)M, cb[d] /= (double)M;
    double H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};          // H = AA^T BB  (pvn3d_eval_utils_kpls.py:47)
    for (int m = 0; m < M; ++m)
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) H[r][c] += ((double)a[3 * m + r] - ca[r]) * ((double)b[3 * m + c] - cb[c]);
    // one-sided Jacobi: rotate column pairs of H (and of V) until orthogonal: H V = U S
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double al = 0, be = 0, ga = 0;
                for (int r = 0; r < 3; ++r) al += H[r][p] * H[r][p], be += H[r][q] * H[r][q], ga += H[r][p] * H[r][q];
                // a pair is done when its columns are orthogonal to working precision, or when one of them is
                // negligible next to the other (norm ratio <= 1e-15, below the rank cut-off `tiny` further down, so
                // its direction is never used: rotating it only spins on rounding noise).  sqrt(al) * sqrt(be),
                // not sqrt(al * be): the product underflows to 0 for spreads of float32 subnormals.
                const double nrm = sqrt(al) * sqrt(be);
                if (fabs(ga) <= 1e-17 * nrm || fmin(al, be) <= 1e-30 * fmax(al, be)) continue;
                off = fmax(off, fabs(ga) / nrm);
                const double zeta = (be - al) / (2.0 * ga);
                const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double cs = 1.0 / sqrt(1.0 + tt * tt), sn = cs * tt;
                for (int r = 0; r < 3; ++r) {
                    const double hp = H[r][p], hq = H[r][q];
                    H[r][p] = cs * hp - sn * hq, H[r][q] = sn * hp + cs * hq;
                    const double vp = V[r][p], vq = V[r][q];
                    V[r][p] = cs * vp - sn * vq, V[r][q] = sn * vp + cs * vq;
                }
            }
        if (off < 1e-15) break;
    }
    double sg[3];
    int ord[3] = {0, 1, 2};
    for (int k = 0; k < 3; ++k) sg[k] = sqrt(H[0][k] * H[0][k] + H[1][k] * H[1][k] + H[2][k] * H[2][k]);
    for (int x = 0; x < 2; ++x)                      // singular values in descending order
        for (int y = 0; y < 2 - x; ++y)
            if (sg[ord[y]] < sg[ord[y + 1]]) { const int tmp = ord[y]; ord[y] = ord[y + 1], ord[y + 1] = tmp; }
    double U[3][3], W[3][3];
    for (int k = 0; k < 3; ++k)
        for (int r = 0; r < 3; ++r) W[r][k] = V[r][ord[k]];
    // U = H V / S where a singular value is above `tiny`; the rest of the basis is completed so that U stays
    // orthonormal: rank 3 none, rank 2 (coplanar) U2 = U0 x U1, rank 1 (collinear, or M = 2) U1 = the coordinate
    // axis least aligned with U0 made orthogonal to it, then U2 = U0 x U1, rank 0 (all points identical) the
    // identity.  Below rank 3 the fit is not unique: any such completion gives a proper rotation (after the
    // reflection flip) that reaches the least-squares minimum, as every choice of numpy's SVD does.
    const double tiny = 1e-12 * fmax(sg[ord[0]], 1e-300);
    for (int k = 0; k < 2; ++k)
        for (int r = 0; r < 3; ++r) U[r][k] = sg[ord[k]] > tiny ? H[r][ord[k]] / sg[ord[k]] : (r == k ? 1.0 : 0.0);
    if (sg[ord[0]] > tiny && sg[ord[1]] <= tiny) {
        int k = 0;
        for (int r = 1; r < 3; ++r)
            if (fabs(U[r][0]) < fabs(U[k][0])) k = r;
        for (int r = 0; r < 3; ++r) U[r][1] = (r == k ? 1.0 : 0.0) - U[k][0] * U[r][0];      // Gram-Schmidt of e_k
        const double nu = sqrt(U[0][1] * U[0][1] + U[1][1] * U[1][1] + U[2][1] * U[2][1]);    // >= sqrt(2/3)
        for (int r = 0; r < 3; ++r) U[r][1] /= nu;
    }
    if (sg[ord[2]] > tiny)
        for (int r = 0; r < 3; ++r) U[r][2] = H[r][ord[2]] / sg[ord[2]];
    else {                                           // rank <= 2: complete the basis
        U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
        U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
        U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
    }
    double R[3][3];
    for (int pass = 0; pass < 2; ++pass) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) R[r][c] = W[r][0] * U[c][0] + W[r][1] * U[c][1] + W[r][2] * U[c][2];   // R = V U^T
        const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) - R[0][1] * (R[1][0] * R[2][2] - R[1][2] * R[2][0]) +
                           R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
        if (det >= 0) break;
        for (int r = 0; r < 3; ++r) W[r][2] = -W[r][2];     // the reflection case (:52-54)
    }
    double *out = T + (size_t)g * 12;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) out[4 * r + c] = R[r][c];
        out[4 * r + 3] = cb[r] - (R[r][0] * ca[0] + R[r][1] * ca[1] + R[r][2] * ca[2]);
    }
}

}  // namespace ffb6d

using namespace ffb6d;

static size_t ms_header_bytes(int64_t G) { return align_up(256 + (size_t)G * sizeof(MsGroup), 256); }

extern "C" size_t ffb6d_mean_shift_workspace_bytes(int64_t G, int64_t N)
{
    if (G <= 0 || N <= 0) return 0;
    return ms_header_bytes(G) + 2 * align_up((size_t)G * N * sizeof(float4), 256) + align_up((size_t)G * N * sizeof(int), 256);
}

extern "C" int ffb6d_mean_shift_fit(const float *votes, const unsigned char *valid, int64_t valid_stride, int64_t G, int64_t N,
                                    float bandwidth, int max_iter, float *centres, unsigned char *labels, int *iters,
                                    float *modes, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(G >= 0 && G <= MS_MAX_G && N >= 0 && N < (1ll << 24), "mean_shift_fit: G must be <= %d and N < 2^24", MS_MAX_G);
    FFB6D_CHECK_ARG(bandwidth > 0.f && max_iter >= 0, "mean_shift_fit: bandwidth must be positive, max_iter >= 0");
    if (G == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(centres && iters, "mean_shift_fit: null output");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        FFB6D_CUDA(cudaMemsetAsync(centres, 0, (size_t)G * 3 * sizeof(float), st));
        FFB6D_CUDA(cudaMemsetAsync(iters, 0, (size_t)G * sizeof(int), st));
        return FFB6D_OK;
    }
    FFB6D_CHECK_ARG(votes && labels && workspace, "mean_shift_fit: null pointer");
    FFB6D_CHECK_ARG(valid_stride == 0 || valid_stride >= N, "mean_shift_fit: valid_stride must be 0 (shared mask) or >= N");
    FFB6D_CHECK_ARG(workspace_bytes >= ffb6d_mean_shift_workspace_bytes(G, N), "mean_shift_fit: workspace too small");
    char *ws = (char *)workspace;
    unsigned *barrier = (unsigned *)ws;
    MsGroup *state = (MsGroup *)(ws + 256);
    const size_t hb = ms_header_bytes(G), cb = align_up((size_t)G * N * sizeof(float4), 256);
    float4 *buf0 = (float4 *)(ws + hb), *buf1 = (float4 *)(ws + hb + cb);
    int *src = (int *)(ws + hb + 2 * cb);
    FFB6D_CUDA(cudaMemsetAsync(ws, 0, hb, st));
    // all CTAs must be co-resident for the grid barrier: a cooperative launch sized from the occupancy
    static std::atomic<int> per_sm[kMaxDevices];
    const int dev = current_device() & (kMaxDevices - 1);
    int occ = per_sm[dev].load(std::memory_order_relaxed);
    if (occ == 0) {
        FFB6D_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mean_shift_kernel, MS_THREADS, 0));
        FFB6D_CHECK_ARG(occ >= 1, "mean_shift_fit: kernel does not fit an SM");
        per_sm[dev].store(occ, std::memory_order_relaxed);
    }
    const int64_t items = G * ceil_div(N, MS_IT);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)num_sms() * std::min(occ, 2), items));
    int Gi = (int)G, Ni = (int)N;
    long long vs = valid_stride;
    float stop = (float)((double)bandwidth * 1e-3);        // MeanShiftTorch.stop_thresh (:31)
    void *args[] = {&votes, &valid, &vs, &Gi, &Ni, &bandwidth, &stop, &max_iter, &barrier, &state, &buf0, &buf1, &src,
                    &centres, &labels, &iters, &modes};
    FFB6D_CUDA(cudaLaunchCooperativeKernel((const void *)mean_shift_kernel, dim3((unsigned)grid), dim3(MS_THREADS), args, 0, st));
    count_launch();
    return FFB6D_OK;
}

extern "C" int ffb6d_best_fit_transform(const float *A, const float *B, int64_t G, int64_t M, double *T, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(G >= 0 && M >= 1 && M <= 4096, "best_fit_transform: need 1 <= M <= 4096 point pairs");
    if (G == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(A && B && T, "best_fit_transform: null pointer");
    best_fit_kernel<<<(unsigned)ceil_div(G, 64), 64, 0, (cudaStream_t)stream>>>(A, B, (int)G, (int)M, T);
    FFB6D_LAUNCH_OK("best_fit_kernel");
    return FFB6D_OK;
}
