// common.cuh -- shared helpers for libffb6d_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/ffb6d_b200.h"

namespace ffb6d {

// thread-local error text behind ffb6d_last_error()
void set_error(const char *fmt, ...);
// bumps the process-wide launch counter behind ffb6d_launch_count()
void count_launch(int n = 1);

#define FFB6D_CHECK_ARG(cond, ...)                         \
    do {                                                   \
        if (!(cond)) {                                     \
            ::ffb6d::set_error(__VA_ARGS__);               \
            return FFB6D_ERR_INVALID;                      \
        }                                                  \
    } while (0)

#define FFB6D_CUDA(call)                                                             \
    do {                                                                             \
        cudaError_t e__ = (call);                                                    \
        if (e__ != cudaSuccess) {                                                    \
            ::ffb6d::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                               __FILE__, __LINE__);                                  \
            return FFB6D_ERR_CUDA;                                                   \
        }                                                                            \
    } while (0)

// after a <<<>>> launch
#define FFB6D_LAUNCH_OK(name)                                                          \
    do {                                                                               \
        cudaError_t e__ = cudaGetLastError();                                          \
        if (e__ != cudaSuccess) {                                                      \
            ::ffb6d::set_error("launch of %s failed: %s", name, cudaGetErrorString(e__)); \
            return FFB6D_ERR_CUDA;                                                     \
        }                                                                              \
        ::ffb6d::count_launch();                                                       \
    } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Per-device facts, cached per device ordinal (a process may drive several GPUs: function attributes
// and SM counts belong to the CURRENT device, never to the process).
constexpr int kMaxDevices = 64;
struct DeviceInfo {
    int num_sms;          // 132 on H100 SXM
    int max_smem_optin;   // bytes of dynamic shared memory a kernel may opt into
};
int current_device();                 // cudaGetDevice, 0 on error
const DeviceInfo &device_info();      // of the current device
static inline int num_sms() { return device_info().num_sms; }

// One-time (per kernel instantiation AND per device) opt-in to more than 48 KB of dynamic shared
// memory.  Not a stream operation, so it is safe under CUDA-graph capture.
#define FFB6D_OPTIN_SMEM(kern, bytes)                                                              \
    do {                                                                                           \
        static std::atomic<unsigned long long> done__{0};                                          \
        const int dev__ = ::ffb6d::current_device() & (::ffb6d::kMaxDevices - 1);                  \
        if (!((done__.load(std::memory_order_relaxed) >> dev__) & 1ull)) {                         \
            FFB6D_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                            (int)(bytes)));                                        \
            done__.fetch_or(1ull << dev__, std::memory_order_relaxed);                             \
        }                                                                                          \
    } while (0)

// train.cu: weight gradient of narrow layers (used by ffb6d_fusion_mlp_wgrad, fusion_mlp.cu)
int wgrad_small_launch(const float *grad_z, const float *x1, int64_t C1, const float *x2, int64_t C2, int64_t B, int64_t Co,
                       int64_t P, float *grad_w, cudaStream_t st);
// ... and of ffb6d_fusion_mlp_wgrad_det: its split count (SM count dependent), and the launch that stores each split's
// partial into part + split * Co * (C1 + C2)
int64_t wgrad_small_splits(int64_t B, int64_t P);
int wgrad_small_det_launch(const float *grad_z, const float *x1, int64_t C1, const float *x2, int64_t C2, int64_t B,
                           int64_t Co, int64_t P, float *part, cudaStream_t st);

// Experiment switches, read ONCE per process (never in a launch path; results never depend on them).
struct Env {
    bool gather_direct;     // FFB6D_GATHER_DIRECT=1: K-lane gathers through the older direct kernel
    bool check_indices;     // FFB6D_CHECK_INDICES=1: validate gather indices (synchronises; debugging aid)
    bool grid_thread_search;
    bool subset_nn;         // FFB6D_SUBSET_NN=1: ffb6d_build_indices reads cld_interp_idx{0,1} off the self searches (ffb6d_knn_subset_nn)
    float grid_scale, grid_scale_k1;
    int grid_quantile;
};
const Env &env();

// The reference distance: nanoflann L2_Adaptor::evalMetric tail loop for dim 3
// (NN/nanoflann.hpp:343-346): result = 0; result += d0*d0; += d1*d1; += d2*d2 in fp32,
// compiled without FMA.  The _rn intrinsics are never contracted by nvcc.
__device__ __forceinline__ float ref_sqdist(float qx, float qy, float qz, float sx, float sy,
                                            float sz)
{
    const float dx = __fsub_rn(qx, sx);
    const float dy = __fsub_rn(qy, sy);
    const float dz = __fsub_rn(qz, sz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

}  // namespace ffb6d
