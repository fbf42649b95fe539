// api.cu -- library bookkeeping, KNN dispatch and the host-pointer entry points
// that carry the reference's own signatures (NN/knn_.h:2-16).
#include "common.cuh"
#include "knn_common.cuh"

#include <atomic>
#include <mutex>
#include <string.h>
#include <stdlib.h>

namespace ffb6d {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int current_device()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        dev = 0;
    }
    return dev;
}

const DeviceInfo &device_info()
{
    static DeviceInfo info[kMaxDevices];
    static std::atomic<unsigned long long> known{0};
    const int dev = current_device() & (kMaxDevices - 1);
    if (!((known.load(std::memory_order_acquire) >> dev) & 1ull)) {
        DeviceInfo d;
        if (cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.num_sms < 1) {
            cudaGetLastError();
            d.num_sms = 132;   // H100 SXM
        }
        if (cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
            cudaGetLastError();
            d.max_smem_optin = 48 * 1024;
        }
        info[dev] = d;   // racing threads write identical values
        known.fetch_or(1ull << dev, std::memory_order_release);
    }
    return info[dev];
}

const Env &env()
{
    static const Env e = [] {
        Env v;
        auto on = [](const char *n) { const char *x = getenv(n); return x && *x && strcmp(x, "0") != 0; };
        v.check_indices = on("FFB6D_CHECK_INDICES");
        return v;
    }();
    return e;
}

// Grow-only device scratch used ONLY by the blocking *_host entry points (the
// device-pointer API never allocates).  One per process, guarded by a mutex:
// the host entry points are serialised, like the GIL-holding Cython shim they
// replace (NN/knn.pyx:71-109).
struct HostScratch {
    std::mutex mu;
    void *buf[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t cap[4] = {0, 0, 0, 0};
    int device = -1;
    int get(int slot, size_t bytes, void **out)
    {
        int dev = 0;
        FFB6D_CUDA(cudaGetDevice(&dev));
        if (dev != device) {  // buffers belong to another device: drop them
            for (int s = 0; s < 4; ++s) {
                if (buf[s]) {
                    cudaSetDevice(device);
                    cudaFree(buf[s]);
                    cudaSetDevice(dev);
                }
                buf[s] = nullptr;
                cap[s] = 0;
            }
            device = dev;
        }
        if (bytes > cap[slot]) {
            if (buf[slot]) FFB6D_CUDA(cudaFree(buf[slot]));
            buf[slot] = nullptr;
            cap[slot] = 0;
            const size_t want = align_up(bytes + bytes / 4, 1 << 20);
            FFB6D_CUDA(cudaMalloc(&buf[slot], want));
            cap[slot] = want;
        }
        *out = buf[slot];
        return FFB6D_OK;
    }
};
static HostScratch g_scratch;

static int knn_dispatch(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                        int K, void *idx_out, int idx_is_i64, void *ws, size_t ws_bytes, int algo,
                        cudaStream_t st)
{
    FFB6D_CHECK_ARG(B >= 0 && S >= 0 && Q >= 0, "knn: negative size (B=%lld S=%lld Q=%lld)",
                    (long long)B, (long long)S, (long long)Q);
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "knn: K=%d outside [1,%d]", K, FFB6D_MAX_K);
    FFB6D_CHECK_ARG(S < (1ll << 31) && Q < (1ll << 31) && B < 65536, "knn: size too large");
    FFB6D_CHECK_ARG(algo >= 0 && algo <= 2, "knn: unknown algo %d", algo);
    if (B == 0 || Q == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(query && idx_out, "knn: null query/idx_out");
    FFB6D_CHECK_ARG(S == 0 || support, "knn: null support");
    if (algo == 0) algo = knn_grid_workspace_bytes(B, S, Q, K) ? 2 : 1;
    if (algo == 2) {
        const size_t need = knn_grid_workspace_bytes(B, S, Q, K);
        if (need == 0) {
            algo = 1;  // the grid declines tiny problems
        } else {
            if (!ws || ws_bytes < need) {
                set_error("knn: workspace of %zu bytes required, %zu given", need, ws_bytes);
                return FFB6D_ERR_WORKSPACE;
            }
            return knn_grid_launch(support, query, B, S, Q, K, idx_out, idx_is_i64, ws, ws_bytes, st);
        }
    }
    return knn_brute_launch(support, query, B, S, Q, K, idx_out, idx_is_i64, st);
}

}  // namespace ffb6d

using namespace ffb6d;

extern "C" {

int ffb6d_version(void) { return 3; }
const char *ffb6d_last_error(void) { return g_err; }
uint64_t ffb6d_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
int ffb6d_check_indices_enabled(void) { return env().check_indices ? 1 : 0; }

int ffb6d_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

size_t ffb6d_knn_workspace_bytes(int64_t B, int64_t S, int64_t Q, int K)
{
    if (B <= 0 || S <= 0 || Q <= 0 || K < 1 || K > FFB6D_MAX_K) return 0;
    return knn_grid_workspace_bytes(B, S, Q, K);
}

int ffb6d_knn_batch(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                    int K, void *idx_out, int idx_is_i64, void *workspace, size_t workspace_bytes,
                    ffb6d_stream_t stream)
{
    return knn_dispatch(support, query, B, S, Q, K, idx_out, idx_is_i64, workspace,
                        workspace_bytes, 0, (cudaStream_t)stream);
}

int ffb6d_knn_batch_algo(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                         int K, void *idx_out, int idx_is_i64, void *workspace,
                         size_t workspace_bytes, int algo, ffb6d_stream_t stream)
{
    return knn_dispatch(support, query, B, S, Q, K, idx_out, idx_is_i64, workspace,
                        workspace_bytes, algo, (cudaStream_t)stream);
}

size_t ffb6d_knn_grid_bytes(int64_t B, int64_t S)
{
    if (B <= 0 || S <= 0) return 0;
    return knn_grid_store_bytes(B, S);
}

size_t ffb6d_knn_grid_query_bytes(int64_t B, int64_t Q)
{
    if (B <= 0 || Q <= 0) return 0;
    return knn_grid_query_bytes(B, Q);
}

int ffb6d_knn_grid_build(const float *support, int64_t B, int64_t S, int K_hint, void *grid,
                         size_t grid_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 1 && S >= 1 && B < 65536 && S < (1ll << 31), "knn_grid_build: bad size");
    FFB6D_CHECK_ARG(K_hint >= 1 && K_hint <= FFB6D_MAX_K, "knn_grid_build: K_hint=%d outside [1,%d]",
                    K_hint, FFB6D_MAX_K);
    FFB6D_CHECK_ARG(support && grid, "knn_grid_build: null pointer");
    return knn_grid_build(support, B, S, K_hint, grid, grid_bytes, (cudaStream_t)stream);
}

int ffb6d_knn_grid_query(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                         int K, void *idx_out, int idx_is_i64, const void *grid, size_t grid_bytes,
                         void *scratch, size_t scratch_bytes, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && S >= 1 && Q >= 0 && B < 65536 && S < (1ll << 31) && Q < (1ll << 31),
                    "knn_grid_query: bad size");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "knn_grid_query: K=%d outside [1,%d]", K, FFB6D_MAX_K);
    if (B == 0 || Q == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(support && query && idx_out && grid && scratch, "knn_grid_query: null pointer");
    return knn_grid_query(support, query, B, S, Q, K, idx_out, idx_is_i64, grid, grid_bytes, scratch,
                          scratch_bytes, (cudaStream_t)stream);
}

int ffb6d_knn_grid_query_organized(const float *support, const float *query, int64_t B, int64_t S, int64_t Q,
                                   int K, void *idx_out, int idx_is_i64, const void *grid, size_t grid_bytes,
                                   void *scratch, size_t scratch_bytes, int64_t query_width, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && S >= 1 && Q >= 0 && B < 65536 && S < (1ll << 31) && Q < (1ll << 31),
                    "knn_grid_query: bad size");
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "knn_grid_query: K=%d outside [1,%d]", K, FFB6D_MAX_K);
    FFB6D_CHECK_ARG(query_width >= 0 && (query_width == 0 || Q % query_width == 0),
                    "knn_grid_query: query_width=%lld does not divide Q=%lld", (long long)query_width, (long long)Q);
    if (B == 0 || Q == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(support && query && idx_out && grid && scratch, "knn_grid_query: null pointer");
    return knn_grid_query(support, query, B, S, Q, K, idx_out, idx_is_i64, grid, grid_bytes, scratch,
                          scratch_bytes, (cudaStream_t)stream, query_width);
}

void ffb6d_knn_grid_tune(float cell_scale, int quantile) { knn_grid_tune(cell_scale, quantile); }
void ffb6d_knn_grid_tune_k1(float cell_scale_k1) { knn_grid_tune_k1(cell_scale_k1); }

int ffb6d_knn_batch_host(const float *batch_data, size_t batch_size, size_t npts, size_t dim,
                         const float *queries, size_t nqueries, size_t K, long *batch_indices)
{
    FFB6D_CHECK_ARG(dim == 3, "knn_batch_host: dim=%zu, only 3 is supported", dim);
    FFB6D_CHECK_ARG(K >= 1 && K <= FFB6D_MAX_K, "knn_batch_host: K=%zu outside [1,%d]", K,
                    FFB6D_MAX_K);
    if (batch_size == 0 || nqueries == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(queries && batch_indices && (npts == 0 || batch_data),
                    "knn_batch_host: null pointer");
    if (ffb6d_device_count() == 0) {
        set_error("knn_batch_host: no CUDA device visible");
        return FFB6D_ERR_NO_DEVICE;
    }
    std::lock_guard<std::mutex> lock(g_scratch.mu);
    const size_t sup_b = batch_size * npts * 3 * sizeof(float);
    const size_t qry_b = batch_size * nqueries * 3 * sizeof(float);
    const size_t idx_b = batch_size * nqueries * K * sizeof(long);
    const size_t ws_b = ffb6d_knn_workspace_bytes((int64_t)batch_size, (int64_t)npts,
                                                  (int64_t)nqueries, (int)K);
    void *d_sup, *d_qry, *d_idx, *d_ws;
    int rc;
    if ((rc = g_scratch.get(0, sup_b ? sup_b : 16, &d_sup))) return rc;
    if ((rc = g_scratch.get(1, qry_b, &d_qry))) return rc;
    if ((rc = g_scratch.get(2, idx_b, &d_idx))) return rc;
    if ((rc = g_scratch.get(3, ws_b ? ws_b : 16, &d_ws))) return rc;
    cudaStream_t st = 0;
    if (sup_b) FFB6D_CUDA(cudaMemcpyAsync(d_sup, batch_data, sup_b, cudaMemcpyHostToDevice, st));
    FFB6D_CUDA(cudaMemcpyAsync(d_qry, queries, qry_b, cudaMemcpyHostToDevice, st));
    rc = knn_dispatch((const float *)d_sup, (const float *)d_qry, (int64_t)batch_size,
                      (int64_t)npts, (int64_t)nqueries, (int)K, d_idx, 1, d_ws, ws_b, 0, st);
    if (rc) return rc;
    FFB6D_CUDA(cudaMemcpyAsync(batch_indices, d_idx, idx_b, cudaMemcpyDeviceToHost, st));
    FFB6D_CUDA(cudaStreamSynchronize(st));
    return FFB6D_OK;
}

int ffb6d_knn_host(const float *points, size_t npts, size_t dim, const float *queries,
                   size_t nqueries, size_t K, long *indices)
{
    return ffb6d_knn_batch_host(points, 1, npts, dim, queries, nqueries, K, indices);
}

}  // extern "C"
