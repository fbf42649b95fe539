// loss.cu -- FFB6D's training loss on the GPU (sm_90a): FocalLoss and the offset L1 loss (of_l1_loss / OFLoss) of
// models/loss.py:12-90, as train_ycb.py:237-253 and train_lm.py combine them, with an optional per-frame mask.
//
// Focal loss, [B,C,N] logits (layout 0, the head's) or [B,N,C] rows (layout 1), labels [B,N]:
//   lse = max + log(sum exp(z - max)),  logpt = z_t - lse,  pt = exp(logpt) (detached, as the reference's
//   Variable(logpt.data.exp())),  term = -(1 - pt)^gamma * logpt * alpha[t]
//   forward   sum (or mean over the M counted points) of term; also the arg-max accuracy (lowest index on ties)
//   backward  dz_j = g_t * [j == t] - exp(z_j - lse) * g_t,  g_t = -(1 - pt)^gamma * alpha[t] * g / M
// Offset L1, pred [B,K,N,3] (the head's layout), targ [B,N,K,3] (the item's layout), w_n = labels[b,n] > 0:
//   forward   out[b,k] = S_bk / (float(cnt_b) + 1e-3f),  S_bk = sum_n sum_c w_n |pred - targ|,  cnt_b = sum_n w_n
//   backward  grad = (g_bk / (cnt_b + 1e-3f)) * w_n * sign(pred - targ), the reference's autograd product in fp32
// A frame with valid[b] == 0 adds nothing and gets zero gradients.  The forwards write fp64 partials per CTA into
// the workspace and a finalize kernel adds them in a fixed order, so every result is the same from run to run; no
// call allocates, synchronises the host or uses atomics.
#include <cmath>

#include "common.cuh"

namespace ffb6d {

constexpr int FT = 256;            // focal: threads per CTA, one point each
constexpr int OP = 128;            // offset L1: points per CTA
constexpr int OTH = OP * 3;        // offset L1: threads per CTA, one (point, coordinate) each
constexpr int OWARPS = OTH / 32;

struct FocalPart {
    double term;                   // sum of the CTA's focal terms
    unsigned count, correct;       // points counted, arg-max == label
};
static_assert(sizeof(FocalPart) == 16, "FocalPart is 16 bytes");

__device__ __forceinline__ long long load_label(const void *labels, int is64, size_t i)
{
    return is64 ? (long long)__ldg(static_cast<const long long *>(labels) + i)
                : (long long)__ldg(static_cast<const int *>(labels) + i);
}

// (1 - pt)^gamma; torch evaluates x ** 2 as x * x
__device__ __forceinline__ float focal_weight(float x, float gamma)
{
    if (gamma == 2.0f) return __fmul_rn(x, x);
    if (gamma == 0.0f) return 1.0f;
    if (gamma == 1.0f) return x;
    return powf(x, gamma);
}

__device__ __forceinline__ bool frame_on(const uint8_t *valid, int b) { return valid == nullptr || __ldg(valid + b); }

__global__ void __launch_bounds__(FT)
focal_fwd_kernel(const float *__restrict__ x, int layout, const void *__restrict__ labels, int is64,
                 const uint8_t *__restrict__ valid, int C, int N, float gamma, const float *__restrict__ alpha,
                 float *__restrict__ lse_out, FocalPart *__restrict__ part)
{
    const int b = blockIdx.y, n = blockIdx.x * FT + threadIdx.x;
    const bool on = frame_on(valid, b);
    double term = 0.0;
    unsigned cnt = 0, ok = 0;
    if (n < N) {
        float lse = 0.0f;
        if (on) {
            const size_t sc = layout ? 1 : (size_t)N;
            const float *xp = x + (size_t)b * C * N + (layout ? (size_t)n * C : (size_t)n);
            float m = __ldg(xp);
            int am = 0;
            for (int c = 1; c < C; ++c) {
                const float v = __ldg(xp + c * sc);
                if (v > m) { m = v; am = c; }
            }
            float s = 0.0f;
            for (int c = 0; c < C; ++c) s = __fadd_rn(s, expf(__fsub_rn(__ldg(xp + c * sc), m)));
            lse = __fadd_rn(m, logf(s));
            const long long t = load_label(labels, is64, (size_t)b * N + n);
            const bool in = t >= 0 && t < C;
            const float nan = __int_as_float(0x7fffffff);
            // a label outside [0, C) reads nothing and makes the term NaN
            const float logpt = __fsub_rn(in ? __ldg(xp + t * sc) : nan, lse);
            const float w = focal_weight(__fsub_rn(1.0f, expf(logpt)), gamma);
            const float lp = alpha ? __fmul_rn(logpt, in ? __ldg(alpha + t) : nan) : logpt;
            term = (double)__fmul_rn(-w, lp);
            cnt = 1;
            ok = am == t;
        }
        lse_out[(size_t)b * N + n] = lse;
    }
    // fixed-order reduction: warp tree, then the CTA's warps in order
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        term += __shfl_down_sync(0xffffffffu, term, off);
        cnt += __shfl_down_sync(0xffffffffu, cnt, off);
        ok += __shfl_down_sync(0xffffffffu, ok, off);
    }
    __shared__ FocalPart wp[FT / 32];
    if ((threadIdx.x & 31) == 0) wp[threadIdx.x >> 5] = FocalPart{term, cnt, ok};
    __syncthreads();
    if (threadIdx.x == 0) {
        FocalPart p = wp[0];
        for (int w = 1; w < FT / 32; ++w) {
            p.term += wp[w].term;
            p.count += wp[w].count;
            p.correct += wp[w].correct;
        }
        part[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = p;
    }
}

constexpr int FIN = 256;

// one CTA: the partials in a fixed order (strided per thread, then a tree), rounded once
__global__ void __launch_bounds__(FIN)
focal_finalize_kernel(const FocalPart *__restrict__ part, int nparts, int size_average, float *__restrict__ loss,
                      float *__restrict__ acc, long long *__restrict__ count)
{
    double s = 0.0;
    unsigned long long c = 0, k = 0;
    for (int i = threadIdx.x; i < nparts; i += FIN) {
        s += part[i].term;
        c += part[i].count;
        k += part[i].correct;
    }
    __shared__ double ss[FIN];
    __shared__ unsigned long long sc[FIN], sk[FIN];
    ss[threadIdx.x] = s;
    sc[threadIdx.x] = c;
    sk[threadIdx.x] = k;
    __syncthreads();
    for (int h = FIN / 2; h; h >>= 1) {
        if (threadIdx.x < h) {
            ss[threadIdx.x] += ss[threadIdx.x + h];
            sc[threadIdx.x] += sc[threadIdx.x + h];
            sk[threadIdx.x] += sk[threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const unsigned long long M = sc[0];
        // no counted point (every frame masked): loss and accuracy are 0, not NaN
        *loss = M == 0 ? 0.0f : __double2float_rn(size_average ? ss[0] / (double)M : ss[0]);
        *acc = M == 0 ? 0.0f : __double2float_rn((double)sk[0] / (double)M);
        *count = (long long)M;
    }
}

__global__ void __launch_bounds__(FT)
focal_bwd_kernel(const float *__restrict__ x, int layout, const void *__restrict__ labels, int is64,
                 const uint8_t *__restrict__ valid, int C, int N, float gamma, const float *__restrict__ alpha,
                 int size_average, const float *__restrict__ lse_in, const long long *__restrict__ count,
                 const float *__restrict__ grad_loss, float *__restrict__ grad)
{
    const int b = blockIdx.y, n = blockIdx.x * FT + threadIdx.x;
    if (n >= N) return;
    const size_t sc = layout ? 1 : (size_t)N, base = (size_t)b * C * N + (layout ? (size_t)n * C : (size_t)n);
    const long long M = __ldg(count);
    if (!frame_on(valid, b) || M == 0) {
        for (int c = 0; c < C; ++c) grad[base + c * sc] = 0.0f;
        return;
    }
    const float *xp = x + base;
    const float lse = __ldg(lse_in + (size_t)b * N + n);
    const long long t = load_label(labels, is64, (size_t)b * N + n);
    const bool in = t >= 0 && t < C;
    const float nan = __int_as_float(0x7fffffff);
    const float g = size_average ? __fdiv_rn(__ldg(grad_loss), (float)M) : __ldg(grad_loss);
    const float w = focal_weight(__fsub_rn(1.0f, expf(__fsub_rn(in ? __ldg(xp + t * sc) : nan, lse))), gamma);
    float gt = __fmul_rn(-w, g);
    if (alpha) gt = __fmul_rn(gt, in ? __ldg(alpha + t) : nan);
    for (int c = 0; c < C; ++c) {
        const float e = __fmul_rn(expf(__fsub_rn(__ldg(xp + c * sc), lse)), gt);
        grad[base + c * sc] = c == t ? __fsub_rn(gt, e) : -e;
    }
}

// stage a tile's targets [np, K, 3] (contiguous in the item's layout) and weights into shared memory
__device__ __forceinline__ int stage_tile(const float *targ, const void *labels, int is64, int b, int K, int N,
                                          int n0, float *tg, float *wsm)
{
    const int np = min(OP, N - n0);
    const float *src = targ + ((size_t)b * N + n0) * K * 3;
    for (int i = threadIdx.x; i < np * K * 3; i += OTH) tg[i] = __ldg(src + i);
    for (int i = threadIdx.x; i < OP; i += OTH)
        wsm[i] = i < np && load_label(labels, is64, (size_t)b * N + n0 + i) > 0 ? 1.0f : 0.0f;
    __syncthreads();
    return np;
}

__global__ void __launch_bounds__(OTH)
of_fwd_kernel(const float *__restrict__ pred, const float *__restrict__ targ, const void *__restrict__ labels,
              int is64, const uint8_t *__restrict__ valid, int K, int N, double *__restrict__ part_s,
              unsigned *__restrict__ part_n)
{
    const int b = blockIdx.y, n0 = blockIdx.x * OP, tile = (int)(blockIdx.y * gridDim.x + blockIdx.x);
    if (!frame_on(valid, b)) return;          // the finalize kernel does not read a masked frame's partials
    extern __shared__ float sm[];
    float *tg = sm, *wsm = sm + OP * K * 3;
    __shared__ double wpart[OWARPS][FFB6D_ITEM_MAX_KPS];
    const int np = stage_tile(targ, labels, is64, b, K, N, n0, tg, wsm);
    const int p = threadIdx.x / 3, c = threadIdx.x - 3 * p;
    const bool have = p < np;
    const float w = wsm[p];
    const float *pp = pred + ((size_t)b * K * N + n0) * 3 + threadIdx.x;
    for (int k = 0; k < K; ++k) {
        double v = 0.0;
        if (have) v = (double)__fmul_rn(w, fabsf(__fsub_rn(__ldg(pp + (size_t)k * N * 3), tg[(p * K + k) * 3 + c])));
#pragma unroll
        for (int off = 16; off; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
        if ((threadIdx.x & 31) == 0) wpart[threadIdx.x >> 5][k] = v;
    }
    if (threadIdx.x < 32) {
        unsigned cnt = 0;
        for (int j = 0; j < OP / 32; ++j) cnt += __popc(__ballot_sync(0xffffffffu, wsm[j * 32 + threadIdx.x] != 0.0f));
        if (threadIdx.x == 0) part_n[tile] = cnt;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        double s = wpart[0][threadIdx.x];
        for (int i = 1; i < OWARPS; ++i) s += wpart[i][threadIdx.x];
        part_s[(size_t)tile * K + threadIdx.x] = s;
    }
}

// one CTA per frame, one thread per keypoint: the frame's tiles in order
__global__ void __launch_bounds__(32)
of_finalize_kernel(const double *__restrict__ part_s, const unsigned *__restrict__ part_n,
                   const uint8_t *__restrict__ valid, int K, int tiles, float *__restrict__ out,
                   float *__restrict__ count)
{
    const int b = blockIdx.x, k = threadIdx.x;
    if (k >= K) return;
    if (!frame_on(valid, b)) {
        out[(size_t)b * K + k] = 0.0f;
        if (k == 0) count[b] = 0.0f;
        return;
    }
    double s = 0.0;
    unsigned long long cnt = 0;
    for (int t = 0; t < tiles; ++t) {
        s += part_s[((size_t)b * tiles + t) * K + k];
        cnt += part_n[(size_t)b * tiles + t];
    }
    const float den = __fadd_rn((float)cnt, 1e-3f);
    out[(size_t)b * K + k] = __double2float_rn(s / (double)den);
    if (k == 0) count[b] = (float)cnt;
}

__global__ void __launch_bounds__(OTH)
of_bwd_kernel(const float *__restrict__ pred, const float *__restrict__ targ, const void *__restrict__ labels,
              int is64, const uint8_t *__restrict__ valid, int K, int N, const float *__restrict__ count,
              const float *__restrict__ grad_out, float *__restrict__ grad)
{
    const int b = blockIdx.y, n0 = blockIdx.x * OP;
    const int np = min(OP, N - n0);
    const bool have = (int)threadIdx.x < np * 3;
    const size_t off = ((size_t)b * K * N + n0) * 3 + threadIdx.x;
    if (!frame_on(valid, b)) {
        if (have)
            for (int k = 0; k < K; ++k) grad[off + (size_t)k * N * 3] = 0.0f;
        return;
    }
    extern __shared__ float sm[];
    float *tg = sm, *wsm = sm + OP * K * 3;
    stage_tile(targ, labels, is64, b, K, N, n0, tg, wsm);
    if (!have) return;
    const int p = threadIdx.x / 3, c = threadIdx.x - 3 * p;
    const float w = wsm[p];
    const float den = __fadd_rn(__ldg(count + b), 1e-3f);
    for (int k = 0; k < K; ++k) {
        const float d = __fsub_rn(__ldg(pred + off + (size_t)k * N * 3), tg[(p * K + k) * 3 + c]);
        const float sgn = d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f);
        const float gd = __fdiv_rn(__ldg(grad_out + (size_t)b * K + k), den);
        grad[off + (size_t)k * N * 3] = __fmul_rn(__fmul_rn(gd, w), sgn);
    }
}

static size_t focal_ws_bytes(int64_t B, int64_t N) { return (size_t)(B * ceil_div(N, FT)) * sizeof(FocalPart); }
static size_t of_ws_bytes(int64_t B, int64_t N, int64_t K)
{
    const size_t parts = (size_t)(B * ceil_div(N, OP));
    return align_up(parts * K * sizeof(double), 16) + align_up(parts * sizeof(unsigned), 16);
}
static bool aligned(const void *p, size_t a) { return (uintptr_t)p % a == 0; }

}  // namespace ffb6d

using namespace ffb6d;

#define LOSS_SIZES_OK(B, N) ((B) >= 1 && (B) < 65536 && (N) >= 1 && (N) < (1ll << 31) - OP)

extern "C" size_t ffb6d_loss_workspace_bytes(int64_t B, int64_t N, int64_t n_kps)
{
    if (!LOSS_SIZES_OK(B, N) || n_kps < 1 || n_kps > FFB6D_ITEM_MAX_KPS) return 0;
    const size_t f = focal_ws_bytes(B, N), o = of_ws_bytes(B, N, n_kps);
    return align_up(f > o ? f : o, 16);
}

static int check_focal(const char *fn, const float *logits, int layout, const void *labels, int labels_is_i64,
                       int64_t B, int64_t C, int64_t N, float gamma, const float *alpha)
{
    FFB6D_CHECK_ARG(LOSS_SIZES_OK(B, N) && C >= 1 && C <= 256 && B * C * N < (1ll << 40),
                    "%s: bad size (B=%lld C=%lld N=%lld; 1 <= C <= 256)", fn, (long long)B, (long long)C,
                    (long long)N);
    FFB6D_CHECK_ARG(layout == 0 || layout == 1, "%s: layout must be 0 ([B,C,N]) or 1 ([B,N,C]), got %d", fn, layout);
    FFB6D_CHECK_ARG(labels_is_i64 == 0 || labels_is_i64 == 1, "%s: labels_is_i64 must be 0 or 1", fn);
    FFB6D_CHECK_ARG(std::isfinite(gamma) && gamma >= 0.0f, "%s: gamma must be finite and >= 0", fn);
    FFB6D_CHECK_ARG(logits && labels, "%s: null pointer", fn);
    FFB6D_CHECK_ARG(aligned(logits, 4) && aligned(labels, labels_is_i64 ? 8 : 4) && aligned(alpha, 4),
                    "%s: misaligned pointer", fn);
    return FFB6D_OK;
}

extern "C" int ffb6d_focal_loss_fwd(const float *logits, int layout, const void *labels, int labels_is_i64,
                                    const uint8_t *valid, int64_t B, int64_t C, int64_t N, float gamma,
                                    const float *alpha, int size_average, float *loss, float *acc, int64_t *count,
                                    float *lse, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    const int rc = check_focal("focal_loss_fwd", logits, layout, labels, labels_is_i64, B, C, N, gamma, alpha);
    if (rc) return rc;
    FFB6D_CHECK_ARG(loss && acc && count && lse && workspace, "focal_loss_fwd: null pointer");
    FFB6D_CHECK_ARG(aligned(loss, 4) && aligned(acc, 4) && aligned(count, 8) && aligned(lse, 4) &&
                        aligned(workspace, 16),
                    "focal_loss_fwd: misaligned pointer");
    const size_t need = focal_ws_bytes(B, N);
    if (workspace_bytes < need) {
        set_error("focal_loss_fwd: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid((unsigned)ceil_div(N, FT), (unsigned)B);
    FocalPart *part = static_cast<FocalPart *>(workspace);
    focal_fwd_kernel<<<grid, FT, 0, st>>>(logits, layout, labels, labels_is_i64, valid, (int)C, (int)N, gamma, alpha,
                                          lse, part);
    FFB6D_LAUNCH_OK("focal_fwd_kernel");
    focal_finalize_kernel<<<1, FIN, 0, st>>>(part, (int)(grid.x * grid.y), size_average != 0, loss, acc,
                                             reinterpret_cast<long long *>(count));
    FFB6D_LAUNCH_OK("focal_finalize_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_focal_loss_bwd(const float *logits, int layout, const void *labels, int labels_is_i64,
                                    const uint8_t *valid, int64_t B, int64_t C, int64_t N, float gamma,
                                    const float *alpha, int size_average, const float *lse, const int64_t *count,
                                    const float *grad_loss, float *grad_logits, ffb6d_stream_t stream)
{
    const int rc = check_focal("focal_loss_bwd", logits, layout, labels, labels_is_i64, B, C, N, gamma, alpha);
    if (rc) return rc;
    FFB6D_CHECK_ARG(lse && count && grad_loss && grad_logits, "focal_loss_bwd: null pointer");
    FFB6D_CHECK_ARG(aligned(lse, 4) && aligned(count, 8) && aligned(grad_loss, 4) && aligned(grad_logits, 4),
                    "focal_loss_bwd: misaligned pointer");
    const dim3 grid((unsigned)ceil_div(N, FT), (unsigned)B);
    focal_bwd_kernel<<<grid, FT, 0, (cudaStream_t)stream>>>(logits, layout, labels, labels_is_i64, valid, (int)C,
                                                            (int)N, gamma, alpha, size_average != 0, lse,
                                                            reinterpret_cast<const long long *>(count), grad_loss,
                                                            grad_logits);
    FFB6D_LAUNCH_OK("focal_bwd_kernel");
    return FFB6D_OK;
}

static int check_of(const char *fn, const float *pred, const float *targ, const void *labels, int labels_is_i64,
                    int64_t B, int64_t K, int64_t N)
{
    FFB6D_CHECK_ARG(LOSS_SIZES_OK(B, N) && K >= 1 && K <= FFB6D_ITEM_MAX_KPS && B * K * N * 3 < (1ll << 40),
                    "%s: bad size (B=%lld n_kps=%lld N=%lld; 1 <= n_kps <= %d)", fn, (long long)B, (long long)K,
                    (long long)N, FFB6D_ITEM_MAX_KPS);
    FFB6D_CHECK_ARG(labels_is_i64 == 0 || labels_is_i64 == 1, "%s: labels_is_i64 must be 0 or 1", fn);
    FFB6D_CHECK_ARG(pred && targ && labels, "%s: null pointer", fn);
    FFB6D_CHECK_ARG(aligned(pred, 4) && aligned(targ, 4) && aligned(labels, labels_is_i64 ? 8 : 4),
                    "%s: misaligned pointer", fn);
    return FFB6D_OK;
}

static size_t of_smem(int64_t K) { return (size_t)(OP * K * 3 + OP) * sizeof(float); }

extern "C" int ffb6d_of_l1_loss_fwd(const float *pred, const float *targ, const void *labels, int labels_is_i64,
                                    const uint8_t *valid, int64_t B, int64_t n_kps, int64_t N, float *out,
                                    float *count, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    const int rc = check_of("of_l1_loss_fwd", pred, targ, labels, labels_is_i64, B, n_kps, N);
    if (rc) return rc;
    FFB6D_CHECK_ARG(out && count && workspace, "of_l1_loss_fwd: null pointer");
    FFB6D_CHECK_ARG(aligned(out, 4) && aligned(count, 4) && aligned(workspace, 16), "of_l1_loss_fwd: misaligned pointer");
    const size_t need = of_ws_bytes(B, N, n_kps);
    if (workspace_bytes < need) {
        set_error("of_l1_loss_fwd: workspace of %zu bytes, %zu needed", workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int tiles = (int)ceil_div(N, OP);
    const size_t parts = (size_t)B * tiles;
    double *part_s = static_cast<double *>(workspace);
    unsigned *part_n = reinterpret_cast<unsigned *>(static_cast<char *>(workspace) +
                                                    align_up(parts * n_kps * sizeof(double), 16));
    FFB6D_OPTIN_SMEM(of_fwd_kernel, of_smem(FFB6D_ITEM_MAX_KPS));
    of_fwd_kernel<<<dim3((unsigned)tiles, (unsigned)B), OTH, of_smem(n_kps), st>>>(
        pred, targ, labels, labels_is_i64, valid, (int)n_kps, (int)N, part_s, part_n);
    FFB6D_LAUNCH_OK("of_fwd_kernel");
    of_finalize_kernel<<<(unsigned)B, 32, 0, st>>>(part_s, part_n, valid, (int)n_kps, tiles, out, count);
    FFB6D_LAUNCH_OK("of_finalize_kernel");
    return FFB6D_OK;
}

extern "C" int ffb6d_of_l1_loss_bwd(const float *pred, const float *targ, const void *labels, int labels_is_i64,
                                    const uint8_t *valid, int64_t B, int64_t n_kps, int64_t N, const float *count,
                                    const float *grad_out, float *grad_pred, ffb6d_stream_t stream)
{
    const int rc = check_of("of_l1_loss_bwd", pred, targ, labels, labels_is_i64, B, n_kps, N);
    if (rc) return rc;
    FFB6D_CHECK_ARG(count && grad_out && grad_pred, "of_l1_loss_bwd: null pointer");
    FFB6D_CHECK_ARG(aligned(count, 4) && aligned(grad_out, 4) && aligned(grad_pred, 4),
                    "of_l1_loss_bwd: misaligned pointer");
    FFB6D_OPTIN_SMEM(of_bwd_kernel, of_smem(FFB6D_ITEM_MAX_KPS));
    of_bwd_kernel<<<dim3((unsigned)ceil_div(N, OP), (unsigned)B), OTH, of_smem(n_kps), (cudaStream_t)stream>>>(
        pred, targ, labels, labels_is_i64, valid, (int)n_kps, (int)N, count, grad_out, grad_pred);
    FFB6D_LAUNCH_OK("of_bwd_kernel");
    return FFB6D_OK;
}
