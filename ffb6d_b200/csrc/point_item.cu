// point_item.cu -- the sampled points' network input and pose-training targets (sm_90a).
//
// The half of the datasets' get_item that reads `choose` (datasets/ycb/ycb_dataset.py:237-247, 348-386 ==
// datasets/linemod/linemod_dataset.py:284-293, 398-436): for point p of frame b at pixel px = choose[b,p]
//   cld_rgb_nrm[b,:,p] = (xyz, rgb[px], nrm[px])         xyz = dpt_2_pcld's float64 point, rounded once
//   labels_pt[b,p]     = labels[px]
//   kp_targ_ofst[b,p]  = xyz64 - kps[i],  ctr_targ_ofst[b,p] = xyz64 - ctr[i]
// where i is the LAST object slot whose class id equals labels[px] (get_pose_gt_info loops over the objects and a
// later one overwrites an earlier one), and +0.0 where no slot matches.  The cloud is float64 in the reference
// (int pixel grid minus a float64 intrinsic) and so are the posed keypoints: the offsets are formed in float64 from
// the UNROUNDED point and cast once, as `kp_targ_ofst.astype(np.float32)` does.  Rounding the point first changes
// about a sixth of the offsets.
//
// Layout: one thread per point, ITEM_TILE points per CTA.  cld_rgb_nrm [B,9,N] and labels_pt [B,N] are point-major,
// so per-thread stores are already coalesced.  The offsets [B,N,n_kps,3] and [B,N,3] are point-minor: a thread's
// outputs go to a padded shared-memory row first, and the CTA then writes its tile as one contiguous run.  The
// label -> slot table (labels are uint8: 256 entries) is built once per CTA.
#include "backproject.cuh"

namespace ffb6d {

constexpr int ITEM_TILE = 64;

// shared floats of a tile's staged offsets: keypoint rows padded to an odd length (no bank conflicts), then centres
static inline int item_row_len(int n_kps) { return (3 * n_kps) | 1; }
static inline size_t item_smem_bytes(int n_kps) { return (size_t)ITEM_TILE * (item_row_len(n_kps) + 3) * sizeof(float); }

__global__ void __launch_bounds__(ITEM_TILE)
point_item_kernel(const float *__restrict__ depth, int H, int W, const double *__restrict__ intr, int intr_per_frame,
                  const int *__restrict__ choose, int N, const uint8_t *__restrict__ rgb,
                  const uint8_t *__restrict__ labels, const float *__restrict__ nrm, const int *__restrict__ obj_cls,
                  const double *__restrict__ obj_kps, const double *__restrict__ obj_ctr, int n_obj, int n_kps,
                  float *__restrict__ cld_rgb_nrm, int *__restrict__ labels_pt, float *__restrict__ kp_targ_ofst,
                  float *__restrict__ ctr_targ_ofst)
{
    extern __shared__ float stage[];
    __shared__ int slot_of[256];
    const int b = blockIdx.y, t = threadIdx.x;
    const int p0 = blockIdx.x * ITEM_TILE, p = p0 + t;
    const int K3 = 3 * n_kps, row_len = K3 | 1;
    float *kst = stage, *cst = stage + ITEM_TILE * row_len;

    for (int i = t; i < 256; i += ITEM_TILE) slot_of[i] = -1;
    __syncthreads();
    const int *cls = obj_cls + (size_t)b * n_obj;
    for (int i = t; i < n_obj; i += ITEM_TILE) {
        const int c = __ldg(cls + i);
        if (c >= 0 && c < 256) atomicMax(&slot_of[c], i);     // the last slot of a class wins
    }
    __syncthreads();

    if (p < N) {
        const size_t HW = (size_t)H * W;
        const int px = __ldg(choose + (size_t)b * N + p);
        const double *k = intr + (intr_per_frame ? (size_t)b * 4 : 0);
        double xyz[3];
        backproject_px64(depth + b * HW, W, px / W, px % W, k[0], k[1], k[2], k[3], xyz);
        const size_t pix = b * HW + px;
        float *o = cld_rgb_nrm + (size_t)b * 9 * N + p;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            o[(size_t)c * N] = __double2float_rn(xyz[c]);
            o[(size_t)(3 + c) * N] = (float)__ldg(rgb + pix * 3 + c);
            o[(size_t)(6 + c) * N] = __ldg(nrm + pix * 3 + c);
        }
        const int lab = __ldg(labels + pix);
        labels_pt[(size_t)b * N + p] = lab;
        const int s = slot_of[lab];
        float *kr = kst + t * row_len, *cr = cst + t * 3;
        if (s >= 0) {
            const double *kp = obj_kps + ((size_t)b * n_obj + s) * K3;
            for (int j = 0; j < K3; j += 3) {
#pragma unroll
                for (int c = 0; c < 3; ++c) kr[j + c] = __double2float_rn(__dsub_rn(xyz[c], __ldg(kp + j + c)));
            }
            const double *ct = obj_ctr + ((size_t)b * n_obj + s) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) cr[c] = __double2float_rn(__dsub_rn(xyz[c], __ldg(ct + c)));
        } else {
            for (int j = 0; j < K3; ++j) kr[j] = 0.0f;
#pragma unroll
            for (int c = 0; c < 3; ++c) cr[c] = 0.0f;
        }
    }
    __syncthreads();

    const int cnt = min(ITEM_TILE, N - p0);
    float *kout = kp_targ_ofst + ((size_t)b * N + p0) * K3;
    for (int i = t; i < cnt * K3; i += ITEM_TILE) kout[i] = kst[(i / K3) * row_len + i % K3];
    float *cout = ctr_targ_ofst + ((size_t)b * N + p0) * 3;
    for (int i = t; i < cnt * 3; i += ITEM_TILE) cout[i] = cst[i];
}

}  // namespace ffb6d

using namespace ffb6d;

static inline bool aligned(const void *p, size_t a) { return ((uintptr_t)p % a) == 0; }

extern "C" int ffb6d_point_item(const float *depth_m, int64_t B, int64_t H, int64_t W, const double *intrinsics,
                                int intrinsics_per_frame, const int *choose, int64_t N, const uint8_t *rgb,
                                const uint8_t *labels, const float *nrm, const int *obj_cls, const double *obj_kps,
                                const double *obj_ctr, int64_t n_obj, int64_t n_kps, float *cld_rgb_nrm,
                                int *labels_pt, float *kp_targ_ofst, float *ctr_targ_ofst, ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && B < 65536 && H >= 1 && W >= 1 && H * W < (1ll << 31) && N >= 0 && N < (1ll << 31),
                    "point_item: bad size (B=%lld H=%lld W=%lld N=%lld)", (long long)B, (long long)H, (long long)W,
                    (long long)N);
    FFB6D_CHECK_ARG(n_kps >= 1 && n_kps <= FFB6D_ITEM_MAX_KPS, "point_item: n_kps=%lld outside [1, %d]",
                    (long long)n_kps, FFB6D_ITEM_MAX_KPS);
    FFB6D_CHECK_ARG(n_obj >= 1 && n_obj <= FFB6D_ITEM_MAX_OBJ, "point_item: n_obj=%lld outside [1, %d]",
                    (long long)n_obj, FFB6D_ITEM_MAX_OBJ);
    FFB6D_CHECK_ARG(intrinsics_per_frame == 0 || intrinsics_per_frame == 1,
                    "point_item: intrinsics_per_frame must be 0 or 1");
    if (B == 0 || N == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(depth_m && intrinsics && choose && rgb && labels && nrm && obj_cls && obj_kps && obj_ctr &&
                    cld_rgb_nrm && labels_pt && kp_targ_ofst && ctr_targ_ofst, "point_item: null pointer");
    FFB6D_CHECK_ARG(aligned(intrinsics, 8) && aligned(obj_kps, 8) && aligned(obj_ctr, 8) && aligned(depth_m, 4) &&
                    aligned(choose, 4) && aligned(nrm, 4) && aligned(obj_cls, 4) && aligned(cld_rgb_nrm, 4) &&
                    aligned(labels_pt, 4) && aligned(kp_targ_ofst, 4) && aligned(ctr_targ_ofst, 4),
                    "point_item: misaligned pointer");
    dim3 grid((unsigned)ceil_div(N, ITEM_TILE), (unsigned)B);
    point_item_kernel<<<grid, ITEM_TILE, item_smem_bytes((int)n_kps), (cudaStream_t)stream>>>(
        depth_m, (int)H, (int)W, intrinsics, intrinsics_per_frame, choose, (int)N, rgb, labels, nrm, obj_cls, obj_kps,
        obj_ctr, (int)n_obj, (int)n_kps, cld_rgb_nrm, labels_pt, kp_targ_ofst, ctr_targ_ofst);
    FFB6D_LAUNCH_OK("point_item_kernel");
    return FFB6D_OK;
}
