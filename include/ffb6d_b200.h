/*
 * ffb6d_b200.h -- C ABI of libffb6d_b200.so: the H100 (sm_90a) implementation of
 * FFB6D's bidirectional-fusion hot path (KNN index build, gather + max-pool /
 * nearest-feature gather, RandLA set-abstraction ops).
 *
 * Every entry point is extern "C", takes plain pointers and sizes, returns
 * FFB6D_OK (0) or a negative error code, and never throws.  ffb6d_last_error()
 * returns a thread-local, human readable message for the last failure.
 *
 * "Reference" citations below are relative to /root/reference/ffb6d/ of
 * ethnhe/FFB6D @ e90baf73.  NN/ = models/RandLA/utils/nearest_neighbors/,
 * GS/ = models/RandLA/utils/cpp_wrappers/.
 *
 * Pointer conventions
 *   *_host entry points take HOST pointers and have the reference's own C++
 *   signatures (NN/knn_.h:2-26): they are what the reference's Cython shim
 *   (NN/knn.pyx:8-31) would bind instead of cpp_knn*.  They copy in, run the
 *   CUDA kernels on the current device's default stream, copy out and
 *   synchronise before returning -- the caller-visible behaviour of the
 *   reference (blocking, caller-allocated output).
 *   All other entry points take DEVICE pointers plus a cudaStream_t passed as
 *   an opaque void* (NULL = default stream), are asynchronous, and never
 *   allocate: temporary storage is caller-provided (see *_workspace_bytes).
 *
 * Index dtype: idx_is_i64 != 0 means int64 ("long", what NN/knn.pyx:93 allocates
 * and what torch.gather consumes), 0 means int32 (what the datasets store,
 * datasets/ycb/ycb_dataset.py:283-309).
 *
 * Feature layouts for the gather ops (the reference tensors are NCHW
 * [B,C,S,1], models/ffb6d.py:159-194):
 *   FFB6D_LAYOUT_NCS  feat[b][c][s]  (contiguous NCHW; point axis fastest)
 *   FFB6D_LAYOUT_NSC  feat[b][s][c]  (torch channels_last view of the same
 *                                     NCHW tensor; channel axis fastest)
 * The output uses the layout of the input.
 */
#ifndef FFB6D_B200_H_
#define FFB6D_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FFB6D_OK              0
#define FFB6D_ERR_INVALID    -1   /* bad argument (shape, K, null pointer, layout) */
#define FFB6D_ERR_CUDA       -2   /* a CUDA runtime call or kernel launch failed  */
#define FFB6D_ERR_WORKSPACE  -3   /* workspace missing or too small               */
#define FFB6D_ERR_NO_DEVICE  -4   /* no CUDA device visible                       */

#define FFB6D_LAYOUT_NCS 0
#define FFB6D_LAYOUT_NSC 1

#define FFB6D_MAX_K 64            /* largest supported neighbour count */

typedef void *ffb6d_stream_t;     /* cudaStream_t */

/* ---- library ------------------------------------------------------------ */
int ffb6d_version(void);                 /* ABI version, bumped on signature change */
const char *ffb6d_last_error(void);      /* thread-local message of the last failure */
int ffb6d_device_count(void);            /* number of CUDA devices, 0 if none / no driver */
/* number of kernels this library has launched in this process (all threads).
 * bench.py reports it as gpu_launches. */
uint64_t ffb6d_launch_count(void);

/* ---- KNN index build ---------------------------------------------------- */
/*
 * Exact K nearest neighbours of every query among the support points of the
 * same batch item, ascending squared distance, fp32 arithmetic identical to
 * nanoflann's L2_Adaptor for dim 3 (NN/nanoflann.hpp:343-346, no FMA).
 * Replaces cpp_knn_batch / cpp_knn_batch_omp (NN/knn_.cxx:72-135).
 *   support [B,S,3] f32, query [B,Q,3] f32 -> idx_out [B,Q,K] int32|int64
 * Ties (exactly equal fp32 distances) are ordered by ascending support index
 * (the reference orders them by KD-tree traversal; see DESIGN.md "tie contract").
 * K > S: slots >= S are written as 0, as the reference leaves them (NN/knn_.cxx:120-121).
 * Workspace: ffb6d_knn_workspace_bytes(B,S,Q,K) bytes of device memory, 256-byte
 * aligned; may be NULL when that function returns 0.
 */
size_t ffb6d_knn_workspace_bytes(int64_t B, int64_t S, int64_t Q, int K);
int ffb6d_knn_batch(const float *support, const float *query,
                    int64_t B, int64_t S, int64_t Q, int K,
                    void *idx_out, int idx_is_i64,
                    void *workspace, size_t workspace_bytes,
                    ffb6d_stream_t stream);

/* Same, selecting the algorithm explicitly (testing / benchmarking):
 * algo 0 = automatic, 1 = tiled brute force, 2 = uniform-grid search. */
int ffb6d_knn_batch_algo(const float *support, const float *query,
                         int64_t B, int64_t S, int64_t Q, int K,
                         void *idx_out, int idx_is_i64,
                         void *workspace, size_t workspace_bytes,
                         int algo, ffb6d_stream_t stream);

/*
 * Build-once / query-many form of the same search, for callers that search one support
 * cloud several times (the FFB6D schedule searches each pyramid level 2-4 times,
 * datasets/ycb/ycb_dataset.py:275-308).  The grid (uniform-cell index of `support`) is
 * written by ffb6d_knn_grid_build into caller memory of ffb6d_knn_grid_bytes(B,S) bytes and
 * is read-only afterwards: queries may run concurrently on any streams ordered after the
 * build.  K_hint only tunes the cell size (performance); results never depend on it.  Each
 * query call needs its own scratch of ffb6d_knn_grid_query_bytes(B,Q) bytes.  `support`
 * must be the array the grid was built from.  Results are identical to ffb6d_knn_batch.
 */
size_t ffb6d_knn_grid_bytes(int64_t B, int64_t S);
size_t ffb6d_knn_grid_query_bytes(int64_t B, int64_t Q);
int ffb6d_knn_grid_build(const float *support, int64_t B, int64_t S, int K_hint,
                         void *grid, size_t grid_bytes, ffb6d_stream_t stream);
int ffb6d_knn_grid_query(const float *support, const float *query,
                         int64_t B, int64_t S, int64_t Q, int K,
                         void *idx_out, int idx_is_i64,
                         const void *grid, size_t grid_bytes,
                         void *scratch, size_t scratch_bytes, ffb6d_stream_t stream);
/* The same search with a layout hint: the Q queries of every batch item are the pixels of an image with
 * rows of `query_width` points, row after row (the stride pyramids of the organised cloud,
 * ycb_dataset.py:253-267).  For K = 1 the 32 queries of an 8x4 pixel tile then share one candidate set.
 * Results are identical to ffb6d_knn_grid_query; query_width = 0 means "no particular order". */
int ffb6d_knn_grid_query_organized(const float *support, const float *query,
                                   int64_t B, int64_t S, int64_t Q, int K,
                                   void *idx_out, int idx_is_i64,
                                   const void *grid, size_t grid_bytes,
                                   void *scratch, size_t scratch_bytes,
                                   int64_t query_width, ffb6d_stream_t stream);

/*
 * The whole index build of a batch in one call: the 22 searches of datasets/ycb/ycb_dataset.py:269-309
 * (== datasets/linemod/linemod_dataset.py:313-353) on `stream`, one grid per (support set, K class).
 *   cld  [B,N0,3]: the sampled, shuffled clouds; level i of the pyramid = the first N0/4^i rows (:278)
 *   img2/img4/img8 [B,(H/sr)*(W/sr),3]: stride-sr sub-grids of the organised cloud (:253-267;
 *                  ffb6d_backproject writes them), zero rows at holes
 *   out[22]: device buffers in the reference's call order -- for i = 0..3: cld_nei_idx{i} [B,N_i,K],
 *            cld_interp_idx{i} [B,N_i,1], r2p_ds_nei_idx{i} [B,N_{i+1},K], p2r_ds_nei_idx{i} [B,HW(sr_i),1]
 *            (sr = 4,8,8,8); then for i = 0..2: r2p_up_nei_idx{i} [B,N_{3-i},K], p2r_up_nei_idx{i}
 *            [B,HW(sr_i),1] (sr = 4,2,2); int32, or int64 with idx_is_i64.  cld_sub_idx{i} is the
 *            first N_{i+1} rows of cld_nei_idx{i} (:279).
 * N0 a multiple of 256, H and W multiples of 8.  workspace: ffb6d_build_indices_workspace_bytes.
 */
size_t ffb6d_build_indices_workspace_bytes(int64_t B, int64_t N0, int64_t H, int64_t W, int K);
int ffb6d_build_indices(const float *cld, const float *img2, const float *img4, const float *img8,
                        int64_t B, int64_t N0, int64_t H, int64_t W, int K,
                        void *const *out, int idx_is_i64, void *workspace, size_t workspace_bytes,
                        ffb6d_stream_t stream);

/* Performance knobs of the grid search (never affect results): the cell edge is
 * cell_scale x the `quantile`-th smallest (0..31) of 32 sampled K-th-neighbour distances.
 * Non-positive / negative arguments leave a knob unchanged.  Defaults 1.0 and 17. */
void ffb6d_knn_grid_tune(float cell_scale, int quantile);
/* Same knob for the grids built for K = 1 searches (default 2.5). */
void ffb6d_knn_grid_tune_k1(float cell_scale_k1);

/* HOST-pointer twins with the reference's exact signatures (NN/knn_.h:2-16);
 * dim must be 3.  `long` is int64 on LP64, as in the reference. */
int ffb6d_knn_batch_host(const float *batch_data, size_t batch_size, size_t npts, size_t dim,
                         const float *queries, size_t nqueries, size_t K, long *batch_indices);
int ffb6d_knn_host(const float *points, size_t npts, size_t dim,
                   const float *queries, size_t nqueries, size_t K, long *indices);

/* ---- gather + max-pool / nearest gather -------------------------------- */
/*
 * out[b,c,q] = max_k feat[b,c,idx[b,q,k]]                       (K >= 1)
 * Replaces FFB6D.random_sample / Network.random_sample (models/ffb6d.py:159-177,
 * models/RandLA/RandLANet.py:87-102) and, with K == 1, FFB6D.nearest_interpolation
 * (models/ffb6d.py:179-194, RandLANet.py:104-117) and the final `choose` gather
 * (models/ffb6d.py:309-312).  Pure selection: results are bitwise equal to the
 * reference (NaN propagates like torch.max).
 *   feat [B,C,S] f32 in `layout`, idx [B,Q,K] -> out [B,C,Q] f32 in `layout`.
 * B < 65536, C <= 65535*8, S, Q < 2^31; with FFB6D_LAYOUT_NSC also B*Q <= 8*(2^31 - 1).
 * Indices must lie in [0,S).  The forward kernels do not check them (an offender reads a stale or
 * foreign element where torch.gather raises a device assert); the backward kernels skip offenders.
 * Debugging aid: ffb6d_check_indices below, or FFB6D_CHECK_INDICES=1 in the environment, which runs
 * that check (and synchronises the stream) in front of every gather entry point.
 */
int ffb6d_gather_max_fwd(const float *feat, const void *idx, int idx_is_i64,
                         int64_t B, int64_t C, int64_t S, int64_t Q, int K,
                         int layout, float *out, ffb6d_stream_t stream);
/* Validates `count` indices against [0,S): returns FFB6D_ERR_INVALID (with the number of offenders
 * in ffb6d_last_error) if any lies outside.  Blocking: synchronises `stream`; not capturable. */
int ffb6d_check_indices(const void *idx, int idx_is_i64, int64_t count, int64_t S, ffb6d_stream_t stream);
/* 1 if this process's library runs that check in front of every gather (FFB6D_CHECK_INDICES as it read the
 * environment once, at its first use), else 0.  Such gathers synchronise and cannot be captured in a CUDA graph. */
int ffb6d_check_indices_enabled(void);
/* Name of the kernel ffb6d_gather_max_fwd launches for a shape (for profiling tools). */
const char *ffb6d_gather_kernel_name(int64_t B, int64_t C, int64_t S, int64_t Q, int K, int layout);
/*
 * Backward of the above as autograd defines it for gather + max: grad_feat is
 * zero-filled, then grad_out[b,c,q] is added at the arg-max neighbour (the first
 * maximal k).  fp32 atomic adds: summation order is not deterministic, exactly
 * as the reference's torch.gather backward on CUDA (ffb6d_gather_max_bwd_det below is the deterministic one).
 */
int ffb6d_gather_max_bwd(const float *feat, const void *idx, int idx_is_i64,
                         const float *grad_out,
                         int64_t B, int64_t C, int64_t S, int64_t Q, int K,
                         int layout, float *grad_feat, ffb6d_stream_t stream);

/*
 * out[b,n,k,:] = pc[b,idx[b,n,k],:]        channels-last neighbour gather
 * Replaces Building_block.gather_neighbour (models/RandLA/RandLANet.py:225-234).
 *   pc [B,S,D] f32, idx [B,N,K] -> out [B,N,K,D] f32
 */
int ffb6d_gather_neighbour_fwd(const float *pc, const void *idx, int idx_is_i64,
                               int64_t B, int64_t S, int64_t D, int64_t N, int K,
                               float *out, ffb6d_stream_t stream);
int ffb6d_gather_neighbour_bwd(const float *grad_out, const void *idx, int idx_is_i64,
                               int64_t B, int64_t S, int64_t D, int64_t N, int K,
                               float *grad_pc, ffb6d_stream_t stream);

/*
 * Relative position encoding of RandLA's local spatial encoding
 * (models/RandLA/RandLANet.py:216-223):
 *   out[b,n,k,:] = [ ||xyz_n - xyz_j||, xyz_n - xyz_j, xyz_n, xyz_j ],  j = idx[b,n,k]
 *   xyz [B,N,3] f32, idx [B,N,K] -> out [B,N,K,10] f32
 * The norm is sqrt((dx*dx + dy*dy) + dz*dz) with round-to-nearest fp32 ops, the
 * order torch.sum uses for a length-3 reduction.
 */
int ffb6d_relative_pos_encoding_fwd(const float *xyz, const void *idx, int idx_is_i64,
                                    int64_t B, int64_t N, int K,
                                    float *out, ffb6d_stream_t stream);
/* Same values written channel-major, out [B,10,N,K] -- what the reference obtains with
 * .permute((0,3,1,2)).contiguous() before the first LFA conv (RandLANet.py:197-198). */
int ffb6d_relative_pos_encoding_cm_fwd(const float *xyz, const void *idx, int idx_is_i64,
                                       int64_t B, int64_t N, int K,
                                       float *out, ffb6d_stream_t stream);

/* ---- fusion 1x1 MLP (tensor cores) ---------------------------------------- */
/*
 * out[b,co,p] = act( scale[co] * sum_ci W[co,ci] * cat(x1,x2)[b,ci,p] + shift[co] )
 * Replaces torch.cat + pt_utils.Conv2d(kernel_size=(1,1), bn=True) with frozen (eval)
 * BatchNorm statistics (models/pytorch_utils.py:75-129,168-201; built models/ffb6d.py:55-80,
 * 104-129; applied :246-262, 282-298): scale = gamma/sqrt(var+eps), shift = beta - mean*scale.
 * Hopper wgmma TF32 tensor cores with 3xTF32 operand splitting: agrees with the fp32 path to ~1e-6
 * relative (the 1e-5 contract).  x1 [B,C1,P], x2 [B,C2,P] or NULL (C2 = 0), weight [Co,C1+C2]
 * row-major, out [B,Co,P]; all f32, NCHW (point axis contiguous).
 * act: 0 none, 1 ReLU (the fusion layers), 2 LeakyReLU(negative_slope) (RandLA's pt_utils.Conv2d,
 * models/RandLA/pytorch_utils.py:163-197: conv -> BN(eps 1e-6) -> LeakyReLU(0.2)).
 *
 * The weights are prepared once (inference: weights are constants), so the layer call allocates
 * nothing.  ffb6d_fusion_mlp_pack splits weight [Co,Ci] into its TF32 hi/lo parts and lays them out
 * as the kernel's shared-memory tiles (`packed`: device, 16-byte aligned,
 * ffb6d_fusion_mlp_pack_bytes(Co, Ci) bytes); ffb6d_fusion_mlp_fwd_packed then streams those tiles
 * with bulk-async (TMA) copies.
 */
size_t ffb6d_fusion_mlp_pack_bytes(int64_t Co, int64_t Ci);
int ffb6d_fusion_mlp_pack(const float *weight, int64_t Co, int64_t Ci, void *packed, size_t packed_bytes,
                          ffb6d_stream_t stream);
int ffb6d_fusion_mlp_fwd_packed(const float *x1, int64_t C1, const float *x2, int64_t C2,
                                const void *packed, const float *scale, const float *shift,
                                int64_t B, int64_t Co, int64_t P, int act, float negative_slope,
                                float *out, ffb6d_stream_t stream);

/*
 * The packed layer with the two epilogue extras of the restructured fusion stage (SURVEY.md §8f-3):
 *   out = act( scale * ( W * cat(x1, x2) + addend[b, add_idx[b, p], :] ) + shift )
 * The reference computes rgb' = p2r_fuse(cat(rgb, nearest_interpolation(p2r_pre(p), idx)))
 * (models/ffb6d.py:246-253, 282-289).  The 1x1 conv is linear and the interpolation a pure selection, so
 * W * cat(rgb, y[idx]) = W1 * rgb + (W2 * y)[idx]: the small product Z = W2 * y is computed on the N_{i+1}
 * points (one call with out_layout = FFB6D_LAYOUT_NSC, so that Z is stored [B, NA, Co], a point's channels
 * contiguous), and the big layer runs over K = C_r only and adds Z[idx[p]] in its epilogue -- the
 * interpolated map is never materialised and the layer's FLOPs halve.
 *   addend   [B, NA, Co] f32 channels-last, or NULL;   add_idx [B, P] int32 / int64 (with addend)
 *   out_layout: FFB6D_LAYOUT_NCS -> out [B, Co, P] (NCHW), FFB6D_LAYOUT_NSC -> out [B, P, Co]
 */
int ffb6d_fusion_mlp_fwd_ex(const float *x1, int64_t C1, const float *x2, int64_t C2,
                            const void *packed, const float *scale, const float *shift,
                            int64_t B, int64_t Co, int64_t P, int act, float negative_slope,
                            const float *addend, const void *add_idx, int add_idx_is_i64, int64_t NA,
                            int out_layout, float *out, ffb6d_stream_t stream);

/* ---- training mode of the 1x1 layers (batch-statistics BatchNorm, backward) ---------------------------
 * Reference: pt_utils.Conv2d = conv1x1(bias=False) -> BatchNorm2d -> activation, trained with autograd
 * (models/pytorch_utils.py:75-129; RandLA flavour models/RandLA/pytorch_utils.py:35-111, eps 1e-6,
 * momentum 0.99; train_ycb.py:464-470 runs backward + Adam over them).  The layer is composed of
 *   z = W * cat(x1, x2)                 ffb6d_fusion_mlp_fwd_ex (scale 1, shift 0, act 0), z is kept
 *   y = act(BN_batch(z))                ffb6d_bn_train_fwd   (also updates the running statistics)
 * and backwards
 *   dz, dgamma, dbeta from dy           ffb6d_bn_train_bwd
 *   dW = sum_b dz_b * X_b^T             ffb6d_fusion_mlp_wgrad (wgmma, split-K, fp32 atomics into dW)
 *   dX = W^T * dz                       ffb6d_fusion_mlp_fwd_ex with the packed transposed weight
 * stats [C][4] f32 = (mean, 1/sqrt(var+eps), gamma/sqrt(var+eps), beta) per channel, written by the forward
 * and read by the backward; workspace: ffb6d_bn_workspace_bytes(C, P) bytes of device memory.
 * act: 0 none, 1 ReLU, 2 LeakyReLU(negative_slope).  gamma / beta / running_* may be NULL. */
size_t ffb6d_bn_workspace_bytes(int64_t C, int64_t P);
int ffb6d_bn_train_fwd(const float *z, int64_t B, int64_t C, int64_t P, const float *gamma, const float *beta,
                       float eps, float momentum, float *running_mean, float *running_var,
                       int act, float negative_slope, float *stats, float *y,
                       void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
int ffb6d_bn_train_bwd(const float *z, const float *grad_y, const float *stats, int64_t B, int64_t C, int64_t P,
                       int act, float negative_slope, float *grad_gamma, float *grad_beta, float *grad_z,
                       void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
/* The same BatchNorm with the statistics of the batch of every rank of a process group (torch's
 * nn.SyncBatchNorm).  The caller gathers one fp64 row per rank between the two halves of each direction:
 *   forward   ffb6d_bn_sync_moments  z -> moments [2C+1] = (n, mean[C], M2[C]) of this rank's B*P values
 *             (all-gather the rows in rank order into gathered [W][2C+1])
 *             ffb6d_bn_sync_fwd      combines the W rows in rank order in fp64 (Chan's parallel formula), writes
 *                                    stats, the running statistics (unbiased variance of the global count) and the
 *                                    global count *count (device, fp64), then y as ffb6d_bn_train_fwd
 *   backward  ffb6d_bn_sync_bwd_sums z, grad_y, stats -> sums [2C] = (sum g'[C], sum g' * xhat[C]) of this rank,
 *                                    and this rank's grad_gamma / grad_beta (left to the caller's gradient all-reduce)
 *             (all-gather the rows into gathered [W][2C])
 *             ffb6d_bn_sync_bwd      adds the W rows in rank order in fp64, divides by *count once, writes grad_z
 * Every rank combines the same rows in the same order, so all ranks hold bit-identical stats and running
 * statistics.  No allocation, no host synchronisation.  workspace: ffb6d_bn_workspace_bytes(C, P); moments, sums,
 * gathered and count 8-byte aligned, stats 16-byte aligned; 1 <= W <= 65536.  A rank with no values is not
 * supported (B, P >= 1). */
int ffb6d_bn_sync_moments(const float *z, int64_t B, int64_t C, int64_t P, double *moments,
                          void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
int ffb6d_bn_sync_fwd(const float *z, int64_t B, int64_t C, int64_t P, const double *gathered, int64_t W,
                      const float *gamma, const float *beta, float eps, float momentum, float *running_mean,
                      float *running_var, int act, float negative_slope, float *stats, double *count, float *y,
                      ffb6d_stream_t stream);
int ffb6d_bn_sync_bwd_sums(const float *z, const float *grad_y, const float *stats, int64_t B, int64_t C, int64_t P,
                           int act, float negative_slope, double *sums, float *grad_gamma, float *grad_beta,
                           void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
int ffb6d_bn_sync_bwd(const float *z, const float *grad_y, const float *stats, int64_t B, int64_t C, int64_t P,
                      const double *gathered, int64_t W, const double *count, int act, float negative_slope,
                      float *grad_z, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
/* grad_z = grad_y * act'(z) for a layer with an activation but no BatchNorm. */
int ffb6d_act_bwd(const float *z, const float *grad_y, int64_t n, int act, float negative_slope, float *grad_z,
                  ffb6d_stream_t stream);
/* grad_w [Co, C1+C2] = sum over frames of grad_z [B,Co,P] * cat(x1, x2)^T; grad_w is overwritten. */
int ffb6d_fusion_mlp_wgrad(const float *grad_z, const float *x1, int64_t C1, const float *x2, int64_t C2,
                           int64_t B, int64_t Co, int64_t P, float *grad_w, ffb6d_stream_t stream);

/* Backward of the gathered addend of the restructured fusion stage (ffb6d_fusion_mlp_fwd_ex with addend):
 * the transpose of the K = 1 pixel -> point gather, a deterministic segment sum
 *   out[b, c, s] = sum over pixels p with idx[b, p] = s of grad[b, c, p]
 * ffb6d_segment_plan turns idx [B,P] (int32 / int64, values in [0, NA); other values belong to no segment) into a
 * CSR per frame in `plan` (device, 16-byte aligned, ffb6d_segment_plan_bytes(B, P, NA) bytes; 0 for bad sizes):
 * int32 offsets [NA+1], then the pixels of every segment in ascending order.  ffb6d_segment_sum reads
 * grad [B,C,P] f32 (NCHW) and writes out [B,C,NA] f32 (NCS) with a plan made for the same B, P, NA.
 * Every output element is written exactly once (no atomics on out; an empty segment gets 0.0); the sum runs in
 * fp64 in plan order and is rounded once to fp32.  No allocation, no host synchronisation (capturable in a CUDA
 * graph); bit-identical from run to run and from replay to replay.  Sizes, null pointers, plan bytes and
 * alignment are checked before any launch (FFB6D_ERR_INVALID, text in ffb6d_last_error). */
size_t ffb6d_segment_plan_bytes(int64_t B, int64_t P, int64_t NA);
int ffb6d_segment_plan(const void *idx, int idx_is_i64, int64_t B, int64_t P, int64_t NA, void *plan,
                       size_t plan_bytes, ffb6d_stream_t stream);
int ffb6d_segment_sum(const float *grad, const void *plan, size_t plan_bytes, int64_t B, int64_t C, int64_t P,
                      int64_t NA, float *out, ffb6d_stream_t stream);

/* Deterministic backward (what a caller runs when torch.use_deterministic_algorithms(True) is set; the atomic
 * entry points above and below stay as they are).  None of these allocates or synchronises with the host: they can
 * be captured in a CUDA graph, and their results are bit-identical from run to run and from replay to replay.
 * Sizes, null pointers, alignment, workspace bytes and idx_is_i64 are checked before any launch (FFB6D_ERR_INVALID).
 *
 * ffb6d_segment_csr builds the CSR of ffb6d_segment_plan -- int32 offsets [NA+1], then the entries of every segment
 * in ascending position; out-of-range indices belong to no segment -- in work and memory linear in P + NA (the
 * plan above keeps NA x ceil(P/1024) counters).  Frame b starts at byte b * ffb6d_segment_csr_bytes(1, P, NA) of
 * `plan` (16-byte aligned); scratch follows the entries.  ffb6d_segment_sum_csr is ffb6d_segment_sum on that
 * layout (same kernel, same results). */
size_t ffb6d_segment_csr_bytes(int64_t B, int64_t P, int64_t NA);
int ffb6d_segment_csr(const void *idx, int idx_is_i64, int64_t B, int64_t P, int64_t NA, void *plan,
                      size_t plan_bytes, ffb6d_stream_t stream);
int ffb6d_segment_sum_csr(const float *grad, const void *plan, size_t plan_bytes, int64_t B, int64_t C, int64_t P,
                          int64_t NA, float *out, ffb6d_stream_t stream);
/* ffb6d_gather_max_bwd without atomics: grad_feat[b,c,s] = the sum of grad_out[b,c,q] over the rows q whose
 * arg-max neighbour (the rule of ffb6d_gather_max_bwd: a NaN wins, else the first strict maximum) is s.  A CSR of
 * idx flattened to [B, Q*K] and, for K > 1, a uint8 arg-max map go into `workspace` (16-byte aligned,
 * ffb6d_gather_max_bwd_det_workspace_bytes; 0 for bad sizes); the sum runs in fp64 in ascending (q, k) and is
 * rounded once; every element of grad_feat is written once (0.0 where nothing lands).  Layouts as the atomic one. */
size_t ffb6d_gather_max_bwd_det_workspace_bytes(int64_t B, int64_t C, int64_t S, int64_t Q, int K);
int ffb6d_gather_max_bwd_det(const float *feat, const void *idx, int idx_is_i64, const float *grad_out,
                             int64_t B, int64_t C, int64_t S, int64_t Q, int K, int layout, void *workspace,
                             size_t workspace_bytes, float *grad_feat, ffb6d_stream_t stream);
/* ffb6d_gather_neighbour_bwd without atomics: the CSR of idx [B, N*K] and the segment sum over the channels of
 * grad_out [B,N,K,D]; workspace: ffb6d_gather_neighbour_bwd_det_workspace_bytes(B, S, N, K) bytes. */
size_t ffb6d_gather_neighbour_bwd_det_workspace_bytes(int64_t B, int64_t S, int64_t N, int K);
int ffb6d_gather_neighbour_bwd_det(const float *grad_out, const void *idx, int idx_is_i64, int64_t B, int64_t S,
                                   int64_t D, int64_t N, int K, void *workspace, size_t workspace_bytes,
                                   float *grad_pc, ffb6d_stream_t stream);
/* ffb6d_fusion_mlp_wgrad without atomics: the same CTAs, tiles, numerics and split count, but each split stores
 * its partial dW into its own slice of `workspace`, and wgrad_split_reduce_kernel adds the slices in split order in
 * fp64 and rounds once.  The split count depends on the shape and on the SM count of the current device (never on
 * timing), so ffb6d_fusion_mlp_wgrad_det_workspace_bytes(C1, C2, B, Co, P) must be asked on the device that runs
 * the call, and results are bit-identical between runs on GPUs with the same SM count. */
size_t ffb6d_fusion_mlp_wgrad_det_workspace_bytes(int64_t C1, int64_t C2, int64_t B, int64_t Co, int64_t P);
int ffb6d_fusion_mlp_wgrad_det(const float *grad_z, const float *x1, int64_t C1, const float *x2, int64_t C2,
                               int64_t B, int64_t Co, int64_t P, void *workspace, size_t workspace_bytes,
                               float *grad_w, ffb6d_stream_t stream);

/*
 * Attentive pooling core of RandLA's Att_pooling (models/RandLA/RandLANet.py:243-248):
 *   out[b,c,n] = sum_k f[b,c,n,k] * softmax_k(att[b,c,n,:])[k],   f = cat(f1, f2) along channels
 *   f1 [B,C1,N,K], f2 [B,C2,N,K] or NULL, att [B,C1+C2,N,K] -> out [B,C1+C2,N]   (f32, K <= 64)
 * (the scores `att` come from the layer's fc = 1x1 conv, i.e. ffb6d_fusion_mlp_fwd_ex with act 0).
 */
int ffb6d_att_pool_fwd(const float *f1, int64_t C1, const float *f2, int64_t C2, const float *att,
                       int64_t B, int64_t N, int K, float *out, ffb6d_stream_t stream);
/* Backward of the above: grad_f[k] = g * s[k], grad_att[k] = s[k] * g * (f[k] - out), s = softmax_k(att).
 * grad_f1 [B,C1,N,K], grad_f2 [B,C2,N,K] (NULL iff C2 == 0), grad_att [B,C1+C2,N,K]; grad_out [B,C1+C2,N,1]. */
int ffb6d_att_pool_bwd(const float *f1, int64_t C1, const float *f2, int64_t C2, const float *att,
                       const float *grad_out, int64_t B, int64_t N, int K,
                       float *grad_f1, float *grad_f2, float *grad_att, ffb6d_stream_t stream);

/*
 * One fused kernel per attentive pooling of RandLA's local feature aggregation (inference, BatchNorm folded):
 *   f_xyz = mlp1(relative_pos_encoding(xyz, idx)) [-> mlp2]          (models/RandLA/RandLANet.py:197-199, 207, 216-223)
 *   f_cat = cat(gather_neighbour(feature, idx), f_xyz)                (:200-205, 208-212)
 *   out   = mlp(sum_K f_cat * softmax_K(fc(f_cat)))                   (:243-250)
 * A warp owns a point; nothing of size N*K is written to memory.
 *   xyz [B,N,3]; idx [B,N,16]; feature [B,Dh,N] (Dh = d/2 in {16, 32, 64}); w_x1 [Dh,10], w_x2 [Dh,Dh] or NULL
 *   (NULL: first pooling of a Building_block), w_fc [2Dh,2Dh], w_out [Do,2Dh] (Do <= 2Dh); scale_* / shift_*: the
 *   folded BatchNorm of mlp1 / mlp2 / the output mlp; LeakyReLU(negative_slope) after each of them.
 *   out [B,Do,N] f32.
 */
int ffb6d_lfa_att_pool_fused(const float *xyz, const void *idx, int idx_is_i64, const float *feature,
                             const float *w_x1, const float *scale_x1, const float *shift_x1,
                             const float *w_x2, const float *scale_x2, const float *shift_x2,
                             const float *w_fc, const float *w_out, const float *scale_out, const float *shift_out,
                             int64_t B, int64_t N, int K, int64_t Dh, int64_t Do, float negative_slope,
                             float *out, ffb6d_stream_t stream);

/*
 * The attentive pooling of a Building_block in training (models/RandLA/RandLANet.py:200-212, 243-248), with the
 * position MLPs' output f_xyz given:
 *   x_k   = cat(feature[b, :, idx[b,n,k]], f_xyz[b, :, n, k])          (d = 2 Dh channels)
 *   f_agg = sum_k x_k * softmax_k(w_fc . x_k)
 * A warp owns a point; nothing of size N*K is written by the forward.
 *   feature [B,Dh,N]; idx [B,N,16] int32 / int64 (values in [0, N)); f_xyz [B,Dh,N,16]; w_fc [2Dh,2Dh];
 *   Dh in {16, 32, 64}, K = 16; f_agg [B,2Dh,N].  All f32, dense.
 * ffb6d_lfa_train_bwd recomputes x, the logits and the softmax s from the same inputs and, with g = grad_agg
 * [B,2Dh,N], dlogit = s * g * (x - f_agg) and dx = g * s + w_fc^T . dlogit, writes
 *   grad_edge  [B,Dh,N*16]  the feature half of dx, one row per edge (n, k): the gradient of the K = 1 gather
 *                           feature[:, :, idx.reshape(B, N*16)]; the caller scatters it onto the points
 *                           (ffb6d_gather_max_bwd or ffb6d_gather_max_bwd_det with K = 1, Q = N*16, S = N)
 *   grad_f_xyz [B,Dh,N,16]  the f_xyz half of dx
 *   grad_w_fc  [2Dh,2Dh]    sum dlogit . x^T, overwritten; without atomics: one partial per CTA in `workspace`,
 *                           summed in CTA order in fp64 and rounded once, so bit-identical from run to run
 * grad_edge and grad_f_xyz 16-byte aligned; workspace: ffb6d_lfa_train_bwd_workspace_bytes(B, N, K, Dh) bytes,
 * 16-byte aligned, asked on the device that runs the call (the partial count follows its SM count; 0 for sizes the
 * calls reject or when there is no device).  B < 65536, N < 2^31.  No allocation, no host synchronisation.
 */
int ffb6d_lfa_train_fwd(const float *feature, const void *idx, int idx_is_i64, const float *f_xyz,
                        const float *w_fc, int64_t B, int64_t N, int K, int64_t Dh, float *f_agg,
                        ffb6d_stream_t stream);
size_t ffb6d_lfa_train_bwd_workspace_bytes(int64_t B, int64_t N, int K, int64_t Dh);
int ffb6d_lfa_train_bwd(const float *feature, const void *idx, int idx_is_i64, const float *f_xyz,
                        const float *w_fc, const float *grad_agg, int64_t B, int64_t N, int K, int64_t Dh,
                        float *grad_edge, float *grad_f_xyz, float *grad_w_fc, void *workspace,
                        size_t workspace_bytes, ffb6d_stream_t stream);

/* ---- depth map -> searched point sets ------------------------------------- */
/*
 * Back-projection of the depth image and extraction of the four point sets the fusion
 * schedule searches, replacing dpt_2_pcld + the `choose` sampling + the stride pyramids of the
 * datasets (datasets/ycb/ycb_dataset.py:165-176, 237, 253-267).  float64 arithmetic like numpy's,
 * rounded once to float32: bit-identical to the reference's arrays.
 *   depth [B,H,W] f32 metres (0 = hole), intrinsics (fx, fy, cx, cy) as float64: 4 values shared
 *   by the batch (intrinsics_per_frame = 0) or [B,4]; choose [B,N] int32 flat pixel indices
 *   -> cld [B,N,3]; pyr2 [B,(H/2)*(W/2),3]; pyr4; pyr8   (f32; holes are signed zeros)
 */
int ffb6d_backproject(const float *depth, int64_t B, int64_t H, int64_t W,
                      const double *intrinsics, int intrinsics_per_frame,
                      const int *choose, int64_t N,
                      float *cld, float *pyr2, float *pyr4, float *pyr8, ffb6d_stream_t stream);

/*
 * The sampled points' network input and pose-training targets: the part of the datasets' get_item that reads
 * `choose` (datasets/ycb/ycb_dataset.py:237-247 with get_pose_gt_info :348-386; datasets/linemod/
 * linemod_dataset.py:284-293, 398-436).  For point p of frame b at pixel px = choose[b,p]:
 *   cld_rgb_nrm [B,9,N] f32: channels 0-2 the point of ffb6d_backproject (same float64 arithmetic, rounded once:
 *                            bitwise equal to its cld), 3-5 rgb[px] as float, 6-8 nrm[px]
 *   labels_pt   [B,N] i32:   labels[px]
 *   kp_targ_ofst [B,N,n_kps,3], ctr_targ_ofst [B,N,3] f32: the float64 point minus obj_kps[b,i] / obj_ctr[b,i],
 *                            rounded once, for i the LAST slot with obj_cls[b,i] == labels[px]; +0.0 where none is
 *   depth_m [B,H,W] f32 metres, intrinsics as ffb6d_backproject, choose [B,N] int32 (trusted, as there);
 *   rgb [B,H,W,3] u8; labels [B,H,W] u8; nrm [B,H,W,3] f32; obj_cls [B,n_obj] i32 class id per slot (< 0: empty);
 *   obj_kps [B,n_obj,n_kps,3] f64 and obj_ctr [B,n_obj,3] f64 posed keypoints and centres.
 * 1 <= n_kps <= FFB6D_ITEM_MAX_KPS, 1 <= n_obj <= FFB6D_ITEM_MAX_OBJ.  Sizes, null pointers and alignment are
 * checked before any launch (FFB6D_ERR_INVALID).  No allocation, no host synchronisation (capturable in a CUDA
 * graph); deterministic.
 */
#define FFB6D_ITEM_MAX_KPS 32
#define FFB6D_ITEM_MAX_OBJ 256
int ffb6d_point_item(const float *depth_m, int64_t B, int64_t H, int64_t W,
                     const double *intrinsics, int intrinsics_per_frame,
                     const int *choose, int64_t N,
                     const uint8_t *rgb, const uint8_t *labels, const float *nrm,
                     const int *obj_cls, const double *obj_kps, const double *obj_ctr,
                     int64_t n_obj, int64_t n_kps,
                     float *cld_rgb_nrm, int *labels_pt, float *kp_targ_ofst, float *ctr_targ_ofst,
                     ffb6d_stream_t stream);

/*
 * The network-input half of ffb6d_point_item, for frames without labels or objects (inference):
 *   cld_rgb_nrm [B,9,N] f32, bitwise what ffb6d_point_item writes for the same depth_m, intrinsics, choose, rgb
 *   and nrm.  Arguments as there; the same size limits.  Sizes, null pointers and alignment are checked before any
 *   launch (FFB6D_ERR_INVALID).  No allocation, no host synchronisation (capturable in a CUDA graph); deterministic.
 */
int ffb6d_point_input(const float *depth_m, int64_t B, int64_t H, int64_t W,
                      const double *intrinsics, int intrinsics_per_frame,
                      const int *choose, int64_t N,
                      const uint8_t *rgb, const float *nrm,
                      float *cld_rgb_nrm, ffb6d_stream_t stream);

/*
 * Valid-pixel compaction + seeded point sampling on the device: replaces the reference's CPU recipe
 * (datasets/ycb/ycb_dataset.py:218-235: `nonzero()` of the depth mask, a random subset of N valid pixels --
 * or all of them repeated cyclically ('wrap') when fewer exist --, then a random permutation).
 *   depth [B,H,W] f32 (valid where > min_depth) -> choose [B,N] int32 flat pixel indices, the `choose`
 *   input of ffb6d_backproject; valid_count [B] int32 (device, may be NULL) = number of valid pixels.
 * Deterministic per (seed, frame index).  Same distribution as the reference (uniform subset, uniform order);
 * numpy's own random stream is not reproduced.  workspace: ffb6d_sample_pixels_workspace_bytes(B,H,W) bytes.
 */
size_t ffb6d_sample_pixels_workspace_bytes(int64_t B, int64_t H, int64_t W);
int ffb6d_sample_pixels(const float *depth, int64_t B, int64_t H, int64_t W, float min_depth, int64_t N,
                        uint64_t seed, int *choose, int *valid_count, void *workspace, size_t workspace_bytes,
                        ffb6d_stream_t stream);
/* ffb6d_sample_pixels with the seed read on the device from seed_dev (one uint64, 8-byte aligned), so that a
 * captured CUDA graph takes a new seed per replay.  Same checks; for equal seed values, the same bits. */
int ffb6d_sample_pixels_dseed(const float *depth, int64_t B, int64_t H, int64_t W, float min_depth, int64_t N,
                              const uint64_t *seed_dev, int *choose, int *valid_count, void *workspace,
                              size_t workspace_bytes, ffb6d_stream_t stream);

/*
 * Depth completion of the raw sensor depth, replacing the CPU call
 * `dpt_um = bs_utils.fill_missing(dpt_um, cam_scale, 1)` of datasets/ycb/ycb_dataset.py:204
 * (utils/basic_utils.py:467-487 -> ip_basic's fill_in_multiscale,
 * utils/ip_basic/ip_basic/depth_map_utils_ycb.py:290-443, with max_depth 3.0, no extrapolation and the
 * bilateral blur -- the only configuration the datasets use).
 *   depth_raw [B,H,W] uint16 (the depth PNG's values), cam_scale > 0 raw units per metre
 *   -> filled_raw [B,H,W] f32 (fill_missing's return, raw units; may be NULL)
 *   -> depth_m    [B,H,W] f32 (the dataset's dpt_m = filled_raw / cam_scale, metres; may be NULL)
 * Every pixel the final bilateral blur does not write is bit-identical to the reference; the blurred ones
 * use exact float64 weights where OpenCV interpolates a table, and differ from it by at most 2e-6 m.
 * Any H, W >= 1.  No allocation, no host synchronisation (capturable in a CUDA graph); deterministic.
 * workspace: ffb6d_fill_depth_workspace_bytes(B,H,W) bytes.  FFB6D_ERR_INVALID on bad sizes, cam_scale <= 0
 * or both outputs NULL; FFB6D_ERR_WORKSPACE on a missing or small workspace.
 */
size_t ffb6d_fill_depth_workspace_bytes(int64_t B, int64_t H, int64_t W);
int ffb6d_fill_depth(const uint16_t *depth_raw, int64_t B, int64_t H, int64_t W, float cam_scale,
                     float *filled_raw, float *depth_m, void *workspace, size_t workspace_bytes,
                     ffb6d_stream_t stream);

/*
 * Surface normals of a millimetre depth map (DESIGN.md §4.30): the least-squares depth-gradient fit of OpenCV's
 * LINEMOD (`accumBilateral`) with the camera's fx, fy, not quantised.  An opt-in stand-in for the datasets'
 * `normalSpeed.depth_normal(dpt_mm, fx, fy, k_size, distance_threshold, difference_threshold, point_into_surface)`
 * (datasets/ycb/ycb_dataset.py:207-210); whether that package computes the same is not known.  For pixel (y, x) with
 * d = depth_mm[b,y,x] and r = k_size:
 *   d == 0 or d >= distance_threshold -> (0, 0, 0).  Otherwise over the 8 offsets (dx, dy) in {-r, 0, r}^2 \ {(0,0)}
 *   inside the image, delta = D[y+dy,x+dx] - d; where |delta| < difference_threshold, in int64:
 *   A0 += dx dx, A1 += dx dy, A2 += dy dy, b0 += dx delta, b1 += dy delta.  det = A0 A2 - A1^2, ddx = A2 b0 - A1 b1,
 *   ddy = A0 b1 - A1 b0; det == 0 -> (0, 0, 0).  In float64 without contraction: nx = fx ddx, ny = fy ddy,
 *   nz = -(double)(det d), s = sqrt((nx nx + ny ny) + nz nz); nrm = (nx/s, ny/s, nz/s), each rounded once to float32,
 *   negated when point_into_surface is 1.
 *   depth_mm [B,H,W] uint16; intrinsics (fx, fy, cx, cy) float64 on the device, [4] (intrinsics_per_frame = 0) or
 *   [B,4] (only fx, fy are read); nrm [B,H,W,3] float32.
 * 0 <= B <= FFB6D_NRM_MAX_FRAMES (B = 0 is a no-op), 1 <= H <= FFB6D_NRM_MAX_HEIGHT, 1 <= W, H W <=
 * FFB6D_NRM_MAX_FRAME_PIXELS; 1 <= k_size <= FFB6D_NRM_MAX_KSIZE; 1 <= distance_threshold <= 65536;
 * 1 <= difference_threshold <= 65535; intrinsics_per_frame, point_into_surface in {0, 1}; depth_mm 2-byte, intrinsics
 * 8-byte, nrm 4-byte aligned.  Checked before any launch (FFB6D_ERR_INVALID).  One launch, no allocation, no host
 * synchronisation (capturable in a CUDA graph); deterministic.
 *
 * ffb6d_depth_to_mm: depth_mm[i] = (uint16)trunc(depth[i] / divisor) over n floats, the division a float32 IEEE one:
 * the YCB dataset's `(dpt_um / 10).astype(np.uint16)` of the completed depth (ycb_dataset.py:207) with divisor 10.
 * Quotients outside [0, 65535] and NaN saturate (0 or 65535).  0 <= n <= FFB6D_NRM_MAX_FRAMES FFB6D_NRM_MAX_FRAME_PIXELS
 * (n = 0 is a no-op); 0 < divisor < inf; depth 4-byte, depth_mm 2-byte aligned.
 */
#define FFB6D_NRM_MAX_KSIZE 16
#define FFB6D_NRM_MAX_FRAMES 65535
#define FFB6D_NRM_MAX_HEIGHT (65535 * 8 - 1)
#define FFB6D_NRM_MAX_FRAME_PIXELS 2147483647ll
int ffb6d_depth_normal(const uint16_t *depth_mm, int64_t B, int64_t H, int64_t W,
                       const double *intrinsics, int intrinsics_per_frame,
                       int k_size, int distance_threshold, int difference_threshold, int point_into_surface,
                       float *nrm, ffb6d_stream_t stream);
int ffb6d_depth_to_mm(const float *depth, int64_t n, float divisor, uint16_t *depth_mm, ffb6d_stream_t stream);

/*
 * Synthetic RGB-D frames of vertex-coloured meshes (DESIGN.md §4.31): a z-buffer rasteriser, the GPU stand-in for
 * the LineMOD `render` pickles (datasets/linemod/linemod_dataset.py:202-212).  Per frame b and slot s < M:
 *   m = mesh_idx[b,s] (-1: empty slot; any value outside [0, n_meshes) draws nothing), RT = RTs[b,s] (float32 [3,4],
 *   object to camera, metres), label[b,s] (uint8).
 * Vertex stage, float64 without contraction: X = ((r0 x + r1 y) + r2 z) + t per row; the vertex is culled when
 *   !(Z >= z_near) or Z is not finite (only non-finite poses or vertices make it so); u = fx (X/Z) + cx,
 *   v = fy (Y/Z) + cy; culled when !(|u| <= 2^14 && |v| <= 2^14) (guard band); U = rint(256 u), V = rint(256 v) as
 *   integers (1/256 pixel, ties to even).  A face with a culled vertex is not drawn (culled, not clipped).
 * Coverage: pixel (col i, row j) samples P = (256 i, 256 j).  With E(a, b, P) = (b.x - a.x)(P.y - a.y) -
 *   (b.y - a.y)(P.x - a.x): w0 = E(V1, V2, P), w1 = E(V2, V0, P), w2 = E(V0, V1, P), A = E(V0, V1, V2) (exact
 *   integers).  A == 0: not drawn.  A < 0: A and every w negated (both windings draw).  P is covered when every
 *   w_k > 0, or w_k == 0 on an owned edge: with (dx, dy) = sign(A) (b - a) of the edge's E(a, b, .), owned is
 *   dy < 0 || (dy == 0 && dx > 0) (the top-left rule: of two faces sharing an edge exactly one draws it).
 * Depth and colour, float64 without contraction: p_k = w_k (1/Z_k), S = (p0 + p1) + p2, depth = fl32(A / S);
 *   colour channel c = clamp(floor((((p0 c0 + p1 c1) + p2 c2) / S) + 0.5), 0, 255) of the vertices' (r, g, b).
 * Visibility: the least key (bits(depth) << 32) | (s max_faces + f) of a pixel wins: the nearest depth, ties to the
 *   lower (slot, face).  Empty pixels are 0 in every output.
 * Mesh table: xyz [V_total,3] float32 metres, vrgb [V_total,3] uint8, faces [F_total,3] int32 (mesh-local vertex
 *   indices, checked by the caller: 0 <= index < the mesh's vertex count), vert_off / face_off [n_meshes + 1] int64
 *   (mesh k owns rows [off[k], off[k+1])); max_verts / max_faces: the largest vertex / face count of a mesh.
 * intrinsics (fx, fy, cx, cy) float64 on the device, [4] (intrinsics_per_frame = 0) or [B,4]; active [B] uint8 or
 *   NULL (every frame): an inactive frame's outputs are not written.  Exactly one of depth [B,H,W] float32 metres and
 *   depth_mm [B,H,W] uint16 = min(trunc(fl32(depth * 1000.0f)), 65535) (LineMOD's `dpt_mm`) is non-NULL; rgb
 *   [B,H,W,3] uint8, labels [B,H,W] uint8.
 * 0 <= B <= FFB6D_RND_MAX_FRAMES (B = 0 is a no-op), 1 <= H, W, H W <= FFB6D_RND_MAX_FRAME_PIXELS,
 * 1 <= M <= FFB6D_RND_MAX_SLOTS, 1 <= n_meshes, 1 <= max_verts <= FFB6D_RND_MAX_MESH_VERTS, 1 <= max_faces,
 * M max_faces <= FFB6D_RND_MAX_FRAME_FACES (the key's 32-bit index), B M max_faces < 2^62; 0.001 <= z_near < inf;
 * intrinsics_per_frame in {0, 1}; every pointer aligned to its element, workspace to 16 bytes.  Checked before any
 * launch (FFB6D_ERR_INVALID; FFB6D_ERR_WORKSPACE below ffb6d_render_workspace_bytes).  Launch shapes depend on the
 * arguments only: one memset and four launches, no allocation, no host synchronisation (capturable in a CUDA graph).
 * Deterministic: the result does not depend on the order of the atomics.  ffb6d_render_workspace_bytes returns 0
 * for sizes the entry point refuses.
 */
#define FFB6D_RND_MAX_FRAMES 65535
#define FFB6D_RND_MAX_FRAME_PIXELS 2147483647ll
#define FFB6D_RND_MAX_SLOTS 4096
#define FFB6D_RND_MAX_MESH_VERTS 2147483647ll
#define FFB6D_RND_MAX_FRAME_FACES 4294967296ll
#define FFB6D_RND_GUARD_BAND 16384
#define FFB6D_RND_BIG_FACE_PIXELS 256
#define FFB6D_RND_QUEUE_CAP (1 << 20)
size_t ffb6d_render_workspace_bytes(int64_t B, int64_t M, int64_t H, int64_t W, int64_t max_verts, int64_t max_faces);
int ffb6d_render_rgbd(const float *xyz, const uint8_t *vrgb, const int32_t *faces, const int64_t *vert_off,
                      const int64_t *face_off, int64_t n_meshes, int64_t max_verts, int64_t max_faces,
                      const int32_t *mesh_idx, const float *RTs, const uint8_t *label, int64_t B, int64_t M,
                      const double *intrinsics, int intrinsics_per_frame, int64_t H, int64_t W, double z_near,
                      const uint8_t *active, float *depth, uint16_t *depth_mm, uint8_t *rgb, uint8_t *labels,
                      void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);

/*
 * ORB keypoints of cv2.ORB_create()'s defaults (DESIGN.md §4.32; oracle/orb_oracle.py restates every step), the 2D
 * stage of the reference's textured keypoint tool (utils/dataset_tools/rgbd_rnder_sift_kp3ds.py:138-166).
 * ffb6d_orb_detect: rgb [B,H,W,3] uint8 -> per frame b, count[b] keypoints in pt [B,cap,2] float32 (x, y image
 *   coordinates), octave [B,cap] int32 and response [B,cap] float32 (Harris), level then raster order; entries past
 *   count[b] hold scratch (candidates of the Harris cut); pt, octave and response may be NULL when cap = 0.
 *   cap = ffb6d_orb_capacity(H, W) = sum over the 8 levels of ceil(w_l' / 2) ceil(h_l' / 2), w_l' = max(w_l - 62, 0)
 *   (the border-filtered level): strict 3x3 non-maximum suppression keeps at most one point per 2x2 block, so the
 *   output can never overflow, however many points the tie-inclusive cuts keep.
 *   Grey (3735 B + 19235 G + 9798 R + 2^14) >> 15; level l of size cvRound(W (1 / s_l)) x cvRound(H (1 / s_l)),
 *   s_l = float32(pow(double(1.2f), l)), is INTER_LINEAR_EXACT of level l-1; FAST-9/16 at threshold 20 with strict
 *   3x3 non-maximum suppression; 31 <= x < w_l - 31, 31 <= y < h_l - 31; every point whose FAST score is >= the
 *   (2 n_l)-th best; Harris (7x7, k = 0.04, integer sums, float32 rounded per operation); every point whose response
 *   is >= the n_l-th best, n_l = nfeaturesPerLevel of 500 features; pt = float32(x_l) s_l.
 *   2 <= H, W <= FFB6D_ORB_MAX_SIDE, 0 <= B <= FFB6D_ORB_MAX_FRAMES (B = 0 is a no-op), cap as above.
 * ffb6d_orb_lift: the keypoints of B = n_obj views renders (object o's views are frames o views ... o views + views
 *   - 1) lifted into the object frame as the tool does: pixel (u, v) = (int(pt.x), int(pt.y)), z = depth[b, v, u]
 *   (float32 metres), x = ((u - cx) z) / fx, y = ((v - cy) z) / fy in float64 without contraction; kept when x is
 *   finite and z > 1e-8 (and the pixel lies in the frame); q = p - t, out_j = (q0 R0j + q1 R1j) + q2 R2j with the
 *   view's RTs [B,3,4] float64 (object to camera), rounded once to float32.  cloud [n_obj, views cap, 3] float32
 *   holds each object's points, views in order, keypoints in order; n_points [n_obj] int32 their number (entries past
 *   it are not written).  intrinsics (fx, fy, cx, cy) float64, [4] or [B,4].  1 <= views, B = n_obj views,
 *   n_obj <= FFB6D_ORB_MAX_OBJECTS, views cap < 2^31.
 * Arguments are checked before any launch (FFB6D_ERR_INVALID; FFB6D_ERR_WORKSPACE below
 * ffb6d_orb_workspace_bytes, which like ffb6d_orb_capacity returns 0 for sizes the entry point refuses).  Launch
 * shapes depend on the arguments only and neither entry point synchronises: both can be captured in a CUDA graph.
 * Deterministic: no atomic decides an output position.
 */
#define FFB6D_ORB_MAX_FRAMES 65535
#define FFB6D_ORB_MIN_SIDE 2
#define FFB6D_ORB_MAX_SIDE 8192
#define FFB6D_ORB_LEVELS 8
#define FFB6D_ORB_MAX_OBJECTS 65535
int64_t ffb6d_orb_capacity(int64_t H, int64_t W);
size_t ffb6d_orb_workspace_bytes(int64_t B, int64_t H, int64_t W);
int ffb6d_orb_detect(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, int32_t *count, float *pt, int32_t *octave,
                     float *response, int64_t cap, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
int ffb6d_orb_lift(const int32_t *count, const float *pt, int64_t cap, const float *depth, int64_t B, int64_t H,
                   int64_t W, const double *intrinsics, int intrinsics_per_frame, const double *RTs, int64_t views,
                   float *cloud, int32_t *n_points, ffb6d_stream_t stream);

/* ---- keypoint voting and pose fitting (the step after the network) -------- */
/*
 * Gaussian mean shift of G independent vote sets, replacing MeanShiftTorch.fit
 * (ffb6d/utils/meanshift_pytorch.py:28-57) as cal_frame_poses / cal_frame_poses_lm call it once per keypoint
 * and once for the centre (ffb6d/utils/pvn3d_eval_utils_kpls.py:89-90, 124-137, 245-258).  One persistent
 * kernel runs all G sets to convergence (max shift < bandwidth * 1e-3, or max_iter + 1 rounds, :30-47) without
 * the N x N matrices and without a host round trip per iteration.
 *   votes [G,N,3] f32; valid: u8 mask of the points that vote (the reference's votes[mask]), [N] shared by the
 *   sets (valid_stride = 0), one row per set (valid_stride >= N elements between rows), or NULL (all vote)
 *   -> centres [G,3] f32: the mode with the most modes within one bandwidth (lowest index on ties);
 *      labels [G,N] u8: 1 where a point's mode lies within one bandwidth of it (0 for non-voting points);
 *      iters [G] i32: rounds run; modes [G,N,3] f32 or NULL: every point's converged position
 *      (`ret_mid_res=True`; rows of non-voting points are 0).
 * A set without voting points gets centre (0,0,0) and 0 rounds.  Floating point: the sums run in another order
 * than torch's, agreement is to about the stop threshold (tests/test_gpu_pose.py), not bitwise.
 * G <= 64.  workspace: ffb6d_mean_shift_workspace_bytes(G, N) bytes.
 */
size_t ffb6d_mean_shift_workspace_bytes(int64_t G, int64_t N);
int ffb6d_mean_shift_fit(const float *votes, const unsigned char *valid, int64_t valid_stride, int64_t G, int64_t N,
                         float bandwidth, int max_iter, float *centres, unsigned char *labels, int *iters,
                         float *modes, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);

/*
 * Least-squares rigid transform mapping point set A onto B (Kabsch / SVD), replacing best_fit_transform
 * (ffb6d/utils/pvn3d_eval_utils_kpls.py:28-59), batched over G objects; float64 arithmetic like numpy's.
 *   A, B [G,M,3] f32 (mesh keypoints, voted keypoints) -> T [G,3,4] f64 = [R | t], det R = +1.
 */
int ffb6d_best_fit_transform(const float *A, const float *B, int64_t G, int64_t M, double *T, ffb6d_stream_t stream);

/*
 * The poses of every object of B frames, replacing cal_frame_poses (ffb6d/utils/pvn3d_eval_utils_kpls.py:65-160;
 * LineMOD's cal_frame_poses_lm, :220-284, is the call with n_cls = 2 on the mask `mask == 1` and refine_thr = NULL).
 *   pcld [B,N,3] f32; mask [B,N] int64 predicted class ids; ctr_of [B,1,N,3], kp_of [B,n_kps,N,3] f32 offsets;
 *   mesh_kps [n_cls,R,3] f32 object-frame keypoints, R = n_kps + use_ctr, the centre last; has_mesh [n_cls] u8;
 *   refine_thr [n_cls] f32 (class c's 0.8 x radius, rounded as float32(float64(r) * 0.8)) or NULL: no refinement
 *   -> present [B,n_cls] u8: class c >= 1 has a point in the unrefined mask (the reference's pred_cls_ids);
 *      count [B,n_cls] i32: the class's points after refinement;
 *      kps [B,n_cls,R,3] f32: the voted keypoints, then the centre when use_ctr;
 *      poses [B,n_cls,3,4] f64: the Kabsch fit of mesh_kps[c] onto kps[b,c] (ffb6d_best_fit_transform's kernel).
 * Per frame, as the reference: with refine_thr, every present class's centre votes (pcld - ctr_of) are fitted, and
 * an object point takes the class of the nearest of those centres (lowest class id on distance ties, distance
 * |pred_ctr - ctr| formed as a difference) when it is below refine_thr of that class.  Then every class with points
 * fits its centre votes (centre + inlier labels; with no label set the class's first point is kept, as the
 * reference's `ctr_labels[0] = 1`) and its n_kps keypoint vote sets, over the labelled points when ctr_filter.
 * Every vote set is compacted in ascending point order from pcld - of in fp32, so its centre and labels are
 * bitwise those of ffb6d_mean_shift_fit on the same set: the same arithmetic, over a device-built set table.
 * Rows without a fit: an absent class gets zeros; a present class left without points the identity pose and zero
 * keypoints.  A mask id outside [0, n_cls) makes that frame's poses and keypoints NaN (present and count 0), and a
 * present class with has_mesh 0 gets a NaN pose and keypoints, without a fault; other rows are unaffected.
 * Three stages with refinement (two without), each one cooperative launch over every set of every frame
 * (DESIGN.md §4.25); results are deterministic and do not depend on the other frames of the batch.
 * 0 <= B (B = 0 is a no-op), 1 <= N <= FFB6D_VOTE_MAX_POINTS, 2 <= n_cls <= FFB6D_VOTE_MAX_CLASSES,
 * 1 <= n_kps <= FFB6D_VOTE_MAX_KPS, B * n_cls * n_kps <= FFB6D_VOTE_MAX_SETS, n_kps * B * N <=
 * FFB6D_VOTE_MAX_SLOTS (the int32 offsets of the packed points); use_ctr, ctr_filter in {0, 1}; bandwidth > 0
 * finite, max_iter >= 0; pointers aligned to their element, the workspace to 256 bytes.
 * workspace: ffb6d_vote_poses_workspace_bytes(B, N, n_cls, n_kps) bytes (FFB6D_ERR_WORKSPACE if missing or
 * smaller).  Arguments are checked before any launch (FFB6D_ERR_INVALID); no allocation, no host synchronisation
 * (capturable in a CUDA graph).
 */
#define FFB6D_VOTE_MAX_POINTS ((1 << 24) - 1)
#define FFB6D_VOTE_MAX_CLASSES 1024
#define FFB6D_VOTE_MAX_KPS 64
#define FFB6D_VOTE_MAX_SETS (1 << 24)
#define FFB6D_VOTE_MAX_SLOTS 2147483647
size_t ffb6d_vote_poses_workspace_bytes(int64_t B, int64_t N, int64_t n_cls, int64_t n_kps);
int ffb6d_vote_poses(const float *pcld, const int64_t *mask, const float *ctr_of, const float *kp_of,
                     const float *mesh_kps, const unsigned char *has_mesh, const float *refine_thr, int64_t B,
                     int64_t N, int64_t n_cls, int64_t n_kps, int use_ctr, int ctr_filter, float bandwidth, int max_iter,
                     unsigned char *present, int *count, float *kps, double *poses, void *workspace,
                     size_t workspace_bytes, ffb6d_stream_t stream);

/* ---- farthest point sampling (object keypoints) -------------------------- */
/*
 * Farthest point sampling of G clouds, replacing the reference's farthest_point_sampling /
 * farthest_point_sampling_init_center (utils/dataset_tools/fps/src/farthest_point_sampling.cpp:166-204, called by
 * fps/fps_utils.py:8-23 for the keypoints of utils/dataset_tools/gen_obj_info.py:86-117).  Bitwise the reference's
 * selection: squared distances (p - q).(p - q) summed x, y, z in round-to-nearest fp32 without FMA; the arg-max
 * takes the first index with a strictly greater min_dist from (index 0, 0.f), so when every remaining distance is 0
 * (duplicate points, S > n) index 0 is selected again.
 *   pts [G,P,3] f32; n_points_per_cloud [G] int32 (device) or NULL: cloud g is its first n_g points, 1 <= n_g <= P
 *   (NULL: every cloud has P); start [G] int32 (device): the first index of each cloud (the reference draws it with
 *   rand()), unread with init_center, which starts from the point farthest from the centre of the bounding box
 *   -> idx_out [G,S] int32.  A cloud whose n_g or start lies out of range gets a row of -1.
 * One thread-block cluster of ceil(P / 14336) CTAs per cloud keeps it in shared memory (DESIGN.md §4.22).
 * 1 <= G <= FFB6D_FPS_MAX_CLOUDS, 1 <= P <= FFB6D_FPS_MAX_POINTS, 1 <= S <= FFB6D_FPS_MAX_SAMPLES; pointers 4-byte
 * aligned.  The kernel needs no workspace: ffb6d_farthest_point_sampling_workspace_bytes returns 0 and ws may be
 * NULL.  Sizes and pointers are checked before the launch (FFB6D_ERR_INVALID); one launch, no allocation, no host
 * synchronisation (capturable in a CUDA graph); deterministic.
 */
#define FFB6D_FPS_MAX_CLUSTER 8
#define FFB6D_FPS_MAX_POINTS (FFB6D_FPS_MAX_CLUSTER * 14336)
#define FFB6D_FPS_MAX_SAMPLES FFB6D_FPS_MAX_POINTS
#define FFB6D_FPS_MAX_CLOUDS 65535
size_t ffb6d_farthest_point_sampling_workspace_bytes(int64_t G, int64_t P, int64_t S);
int ffb6d_farthest_point_sampling(const float *pts, const int *n_points_per_cloud, int64_t G, int64_t P, int64_t S,
                                  const int *start, int init_center, int *idx_out, void *ws, size_t ws_bytes,
                                  ffb6d_stream_t stream);

/* ---- pose scoring (ADD / ADD-S) ------------------------------------------ */
/*
 * ADD and ADD-S of M predicted poses, replacing Basic_Utils.cal_add_cuda / cal_adds_cuda (utils/basic_utils.py:
 * 651-669) as eval_metric / eval_metric_lm call them once per object (utils/pvn3d_eval_utils_kpls.py:162-195,
 * 287-304).  For object m with mesh points x_i, the rows mesh_off[c] .. mesh_off[c+1] of mesh_pts, c = obj_mesh[m],
 * and the poses P = pred_RT[m], G = gt_RT[m]:
 *   add[m]  = mean_i |P x_i - G x_i|
 *   adds[m] = mean_i min_j |P x_j - G x_i|
 *   mesh_pts [sum of mesh sizes, 3] f32; mesh_off [n_meshes + 1] int32 with mesh_off[n_meshes] <= the rows of
 *   mesh_pts; obj_mesh [M] int32; pred_RT, gt_RT [M,3,4] f32 row-major -> add, adds [M] f32.
 * d = P x_j - G x_i is formed before |d|^2 (no |a|^2 + |b|^2 - 2 a.b), the min is taken over squared distances with
 * NaN propagating like torch.min, and one sqrt follows; sums run in fp64 in a fixed order, rounded once to f32, so
 * results are deterministic and pred_RT == gt_RT gives 0 exactly.  A non-finite value in an object's poses or
 * points gives that object NaN.  So does, without a fault, an obj_mesh[m] outside [0, n_meshes), a negative or
 * decreasing offset, or a mesh of 0 or more than max_points points; other objects are unaffected.
 * max_points is the host's bound on every scored mesh's size: it sets the grid (ceil(max_points /
 * FFB6D_POSE_EVAL_GT_TILE) x M CTAs, DESIGN.md §4.24) without a sync.
 * 0 <= M <= FFB6D_POSE_EVAL_MAX_OBJECTS (M = 0 is a no-op), 1 <= max_points <= FFB6D_POSE_EVAL_MAX_POINTS,
 * 1 <= n_meshes <= FFB6D_POSE_EVAL_MAX_MESHES when M > 0; pointers 4-byte aligned, the workspace 16-byte aligned.
 * workspace: ffb6d_pose_add_adds_workspace_bytes(M, max_points) bytes (FFB6D_ERR_WORKSPACE if missing or smaller).
 * Arguments are checked before any launch (FFB6D_ERR_INVALID); two launches, no allocation, no host
 * synchronisation (capturable in a CUDA graph).
 */
#define FFB6D_POSE_EVAL_GT_TILE 512
#define FFB6D_POSE_EVAL_PRED_TILE 512
#define FFB6D_POSE_EVAL_MAX_OBJECTS 65535
#define FFB6D_POSE_EVAL_MAX_POINTS 1048576
#define FFB6D_POSE_EVAL_MAX_MESHES 2147483646
size_t ffb6d_pose_add_adds_workspace_bytes(int64_t M, int64_t max_points);
int ffb6d_pose_add_adds(const float *mesh_pts, const int32_t *mesh_off, int64_t n_meshes, int64_t max_points,
                        const int32_t *obj_mesh, const float *pred_RT, const float *gt_RT, int64_t M, float *add,
                        float *adds, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);

/* ---- the test run's record and summary ------------------------------------ */
/*
 * The per-object lists of the reference's TorchEval (utils/pvn3d_eval_utils_kpls.py:326-505) as a device table, and
 * its summary (cal_auc / cal_lm_add over Basic_Utils.cal_auc, utils/basic_utils.py:642-649), DESIGN.md §4.29.
 *
 * The table: rows [capacity, FFB6D_EVAL_ROW_WORDS] int32 and state [4] int64 (device, zeroed by the caller to start
 * a run): state[0] the rows used, state[1] the frames recorded, state[2] the overflow flag.  A row's words:
 *   0 class id (int32), or -1 for a skipped slot; 1 frame index (state[1] at the batch + b); 2 the class was
 *   predicted (0 / 1); 3 ADD, 4 ADD-S, 5 keypoint error (float32 bits); 6..17 the scored predicted pose [3,4]
 *   (float32 bits); 18, 19 zero.
 *
 * ffb6d_eval_record: one batch of B frames x n_obj object slots; slot (b, j) is written to row state[0] + b n_obj + j
 * (the reference's list order, with no atomic in it), then state[0] += B n_obj and state[1] += B.  A slot is skipped
 * when valid[b] == 0 (valid [B] u8, or NULL: every frame), and
 *   YCB (obj_id = 0): from the frame's first zero cls_ids[b, j] on (cls_ids [B, n_obj] int32); the slot's class
 *     c = cls_ids[b, j] is predicted when 0 <= c < n_cls and present[b, c] (present [B, n_cls] u8, the vote's); its
 *     keypoint error is mean_k |gt_kps[b, j, k] - kps[b, c, k]| in f32 (kps [B, n_cls, R, 3] f32 with R >= n_kps + 1,
 *     gt_kps [B, n_obj, n_kps, 3] f32; kps = 0 when c was not predicted); add, adds [B, n_obj] f32 and pred_RT
 *     [B, n_obj, 3, 4] f32 are placed as given;
 *   LineMOD (obj_id > 0): every slot but 0, which gets class obj_id, presence present[b, 1], add[b], adds[b],
 *     pred_RT[b] and keypoint error 0; cls_ids, kps and gt_kps are unread (may be NULL).
 * The frame table (optional; both or neither): frame_flags [frame_capacity, n_cls] u8 gets present[b, c] | 2 valid[b]
 * and frame_poses [frame_capacity, n_cls, 3, 4] f64 the vote's poses [B, n_cls, 3, 4] at frame state[1] + b.
 * If the batch does not fit (state[0] + B n_obj > capacity, or state[1] + B > frame_capacity with the frame table),
 * nothing is written but state[2] = 1.  One launch (one CTA).
 *
 * ffb6d_eval_auc: over the rows r < min(state[0], capacity) whose class c lies in [1, n_cls):
 *   auc [3, n_cls] f64: cal_auc of ADD, ADD-S and ADD(-S) (ADD-S where sym[c] != 0, sym [n_cls] u8 or NULL) per
 *     class, class 0 over every counted row: distances > 0.1 are misses (exactly 0.1 counts), the accuracy is the f32
 *     cumulative count over n, the area is VOCap's in f64, times 1000; no distance gives 0, a NaN distance NaN;
 *   pct [2, n_cls] f64: the percentage of ADD, ADD-S < lm_thr per class (cal_lm_add; NaN for an empty class);
 *   kp [2] f64: the sum of the rows' keypoint errors and their count (mean_kp_err).
 * The distances are ordered with CUB's radix sort; every sum runs in fp64 in a fixed order (deterministic).
 * workspace: ffb6d_eval_auc_workspace_bytes(capacity, n_cls) bytes, 256-byte aligned.  Four launches.
 *
 * Both: 1 <= capacity, frame_capacity <= FFB6D_EVAL_MAX_ROWS; 1 <= n_cls <= FFB6D_VOTE_MAX_CLASSES; B n_obj <=
 * FFB6D_POSE_EVAL_MAX_OBJECTS; YCB 1 <= n_kps <= FFB6D_VOTE_MAX_KPS.  Arguments are checked before any launch
 * (FFB6D_ERR_INVALID); no allocation, no host synchronisation (capturable in a CUDA graph).
 */
#define FFB6D_EVAL_ROW_WORDS 20
#define FFB6D_EVAL_MAX_ROWS (1 << 24)
int ffb6d_eval_record(const int32_t *cls_ids, const uint8_t *valid, const uint8_t *present, const float *kps,
                      const double *poses, const float *gt_kps, const float *pred_RT, const float *add,
                      const float *adds, int64_t B, int64_t n_obj, int64_t n_cls, int64_t R, int64_t n_kps,
                      int64_t obj_id, int32_t *rows, int64_t capacity, int64_t *state, double *frame_poses,
                      uint8_t *frame_flags, int64_t frame_capacity, ffb6d_stream_t stream);
size_t ffb6d_eval_auc_workspace_bytes(int64_t capacity, int64_t n_cls);
int ffb6d_eval_auc(const int32_t *rows, const int64_t *state, int64_t capacity, int64_t n_cls, const uint8_t *sym,
                   double lm_thr, double *auc, double *pct, double *kp, void *workspace, size_t workspace_bytes,
                   ffb6d_stream_t stream);

/* ---- pose and label drawing ---------------------------------------------- */
/*
 * Projection and drawing of S point sets, replacing Basic_Utils.project_p3d and draw_p2ds (utils/basic_utils.py:
 * 268-295) as demo.py's cal_view_pred_pose (demo.py:116-145) and the trainers' view_labels (train_ycb.py:189-204)
 * call them once per object or frame (DESIGN.md §4.26).
 * The set table: set s is the rows start[s] .. start[s] + count[s] of a point table of n_rows rows (start, count
 * [S] int32, device), drawn only where enable[s] != 0 (enable [S] u8, or NULL: every set).  Outputs are padded to
 * [S, max_rows, ...], row r of set s at s * max_rows + r.  A disabled set, and one with a negative start or count,
 * count > max_rows or start + count > n_rows, is empty: it projects to padding and draws nothing, without a fault.
 *
 * ffb6d_project_p3d: pts [n_rows,3] f32 (pts_f64 = 0) or f64 (1); pose [S,3,4] f64 or NULL; K [3,3] f64 and
 *   cam_scale [1] f64 shared (per_set = 0) or K [S,3,3] and cam_scale [S] (per_set = 1), all device
 *   -> p2ds [S,max_rows,2] int32, (u, v) per row, (INT32_MIN, INT32_MIN) at padding.  Bitwise numpy's float64 code:
 *   with a pose, y_j = fma(x2, R[j][2], fma(x1, R[j][1], x0 * R[j][0])) + t_j and y * cam_scale in f64; without,
 *   x * cam_scale in the points' dtype (f32 points times (float)cam_scale, numpy's casting of a Python float), then
 *   promoted; p_j = fma(z, K[j][2], fma(y, K[j][1], x * K[j][0])); p_2 < 1e-8 -> 1.0 (NaN stays); u = rint(p_0 /
 *   p_2), v = rint(p_1 / p_2) (IEEE division, half to even); the int32 cast of x86's cvttsd2si: NaN and values
 *   outside [-2^31, 2^31) give INT32_MIN.  One launch.
 * ffb6d_draw_p2ds: draws into img [B,H,W,3] u8 (in place) the filled circle of cv2.circle(img, (x, y), radius[s],
 *   colour, -1) (LINE_8, shift 0: OpenCV's integer midpoint circle, clipped to the image) at every row of every set,
 *   x = clip(u, 0, W), y = clip(v, 0, H) (inclusive bounds, as the reference), in frame frame[s] (frame, radius [S]
 *   int32, device).  colors [S,3] u8 (color_per_row = 0) or [S,max_rows,3] (1).  Where circles overlap within a
 *   frame the last in (set, row) order wins; no other pixel is written.  A set whose frame lies outside [0, B) or
 *   whose radius lies outside [0, FFB6D_VIS_MAX_RADIUS] draws nothing.  n_rows and start only decide, as above,
 *   whether a set is empty.  A memset of the workspace and two launches (mark the winning key per pixel with
 *   atomicMax, then paint); the result does not depend on scheduling.
 *   workspace: ffb6d_draw_p2ds_workspace_bytes(B, H, W) = B H W 8 bytes, 8-byte aligned (FFB6D_ERR_WORKSPACE if
 *   missing or smaller); the query returns 0 for sizes out of range.
 * 0 <= S <= FFB6D_VIS_MAX_SETS (S = 0 is a no-op), 1 <= max_rows <= FFB6D_VIS_MAX_ROWS, 0 <= n_rows <=
 * FFB6D_VIS_MAX_TABLE_ROWS, 0 <= B <= FFB6D_VIS_MAX_FRAMES (B = 0 is a no-op), 1 <= H, W <= FFB6D_VIS_MAX_SIDE;
 * flags 0 or 1; pointers aligned to their element, p2ds to 8 bytes.  Arguments are checked before any launch
 * (FFB6D_ERR_INVALID); no allocation, no host synchronisation (capturable in a CUDA graph).
 */
#define FFB6D_VIS_MAX_RADIUS 64
#define FFB6D_VIS_MAX_SIDE 16384
#define FFB6D_VIS_MAX_SETS (1 << 24)
#define FFB6D_VIS_MAX_ROWS (1 << 24)
#define FFB6D_VIS_MAX_TABLE_ROWS 2147483647
#define FFB6D_VIS_MAX_FRAMES 65535
int ffb6d_project_p3d(const void *pts, int pts_f64, int64_t n_rows, const int32_t *start, const int32_t *count,
                      const unsigned char *enable, int64_t S, int64_t max_rows, const double *pose, const double *K,
                      const double *cam_scale, int per_set, int32_t *p2ds, ffb6d_stream_t stream);
size_t ffb6d_draw_p2ds_workspace_bytes(int64_t B, int64_t H, int64_t W);
int ffb6d_draw_p2ds(unsigned char *img, int64_t B, int64_t H, int64_t W, const int32_t *p2ds, int64_t S,
                    int64_t max_rows, const int32_t *frame, const int32_t *start, const int32_t *count,
                    const unsigned char *enable, int64_t n_rows, const int32_t *radius, const unsigned char *colors,
                    int color_per_row, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);

/* ---- grid subsampling --------------------------------------------------- */
/*
 * Voxel-grid barycentre subsampling, replaces grid_subsampling()
 * (GS/cpp_subsampling/grid_subsampling/grid_subsampling.cpp:5-106) behind
 * DataProcessing.grid_sub_sampling (models/RandLA/helper_tool.py:199-219).
 * HOST pointers (the reference op is numpy-in / numpy-out).
 *   points [N,3] f32, features [N,fdim] f32 or NULL, classes [N,ldim] i32 or NULL
 *   -> sub_points [M,3], sub_features [M,fdim], sub_classes [M,ldim]; outputs must
 *      have room for N rows; *M_out receives M.
 * Rows are emitted by ascending voxel key (the reference's order is that of a
 * libstdc++ unordered_map and is unspecified).  Per-voxel sums are accumulated in
 * input order, so barycentres and mean features are bitwise equal to the
 * reference; among labels tied for the maximal count the smallest is chosen.
 */
int ffb6d_grid_subsample_host(const float *points, size_t N,
                              const float *features, size_t fdim,
                              const int *classes, size_t ldim,
                              float sampleDl,
                              float *sub_points, float *sub_features, int *sub_classes,
                              size_t *M_out);

/*
 * Synthetic-frame augmentation (datasets/ycb/ycb_dataset.py:79-163, datasets/linemod/linemod_dataset.py:114-186).
 *
 * ffb6d_rgb_add_noise: the datasets' rgb_add_noise for a batch, rgb [B,H,W,3] u8 -> out [B,H,W,3] u8 (out may
 *   equal rgb).  Each frame has a float64 record of FFB6D_AUG_REC_LEN slots (layout: ffb6d_b200/augment.py) drawn on
 *   the host: HSV factors, the sharpen 3x3, the motion-blur kernel (a x a, a <= FFB6D_AUG_MAX_KSIZE), the Gaussian
 *   blur's fixed-point taps and the noise flags.  plan_host [B,REC_LEN] is what is validated (layout version, flags,
 *   kernel sizes, taps); plan_dev holds the same bytes on the device and is what the kernels read.  The normal draws
 *   are Philox4x32-10 of (seed, frame b, stage 2*pass / 2*pass+1, pixel, channel), or, when noise is not NULL, the
 *   given [2,B,H,W,3] f64 fields.  work: B*H*W*3 bytes of device scratch, aliasing neither rgb nor out.  Given the
 *   record and the same normals the output is bitwise OpenCV's and numpy's, except that filter2D takes a DFT path
 *   for kernels of 130 or more taps (a >= 12), where OpenCV may differ by 1 (DESIGN.md §4.14).
 * ffb6d_add_real_back: add_real_back for a batch.  mode [B] u8 (device): bit 0 composes the depth
 *   (dpt where dpt > 0, else back_dpt where the background pixel is kept, else 0), bit 1 with bit 0 also the colour
 *   (back_rgb where labels == 0 and the background pixel is kept, 0 where it is not).  The background keeps a pixel
 *   where back_labels <= 0 (YCB) or back_labels[...,0] < 255 (LineMOD).  labels [B,H,W] u8, back_labels
 *   [B,H,W,back_label_channels] u8 (1 or 3), dpt / back_dpt / dpt_out [B,H,W] u16.  Outputs may equal inputs.
 * ffb6d_aug_noise_field: out [B,H,W,3] f64 = the normals ffb6d_rgb_add_noise draws for (seed, frame, stage).
 * All three need 0 <= B < 65536, 32 <= H <= 524280 (65535 tiles of 8 rows), 32 <= W < 2^20 and H*W*3 < 2^31, check sizes and null pointers before any launch (FFB6D_ERR_INVALID), allocate nothing and
 * do not synchronise the host (capturable in a CUDA graph); they are deterministic.
 */
#define FFB6D_AUG_VERSION 1
#define FFB6D_AUG_REC_LEN 1024
#define FFB6D_AUG_MAX_KSIZE 30
#define FFB6D_AUG_YCB 0
#define FFB6D_AUG_LINEMOD 1
int ffb6d_rgb_add_noise(const uint8_t *rgb, int64_t B, int64_t H, int64_t W,
                        const double *plan_host, const double *plan_dev, uint64_t seed, const double *noise,
                        uint8_t *out, uint8_t *work, ffb6d_stream_t stream);
/* ffb6d_rgb_add_noise with the seed read on the device from seed_dev (one uint64, 8-byte aligned): a captured
 * CUDA graph takes a new seed per replay.  Same checks; for equal seed values, the same bits. */
int ffb6d_rgb_add_noise_dseed(const uint8_t *rgb, int64_t B, int64_t H, int64_t W,
                              const double *plan_host, const double *plan_dev, const uint64_t *seed_dev,
                              const double *noise, uint8_t *out, uint8_t *work, ffb6d_stream_t stream);
/* The record checks of ffb6d_rgb_add_noise alone, on the host, without a launch: plan_host [B,REC_LEN] f64,
 * 0 <= B < 65536.  0 or FFB6D_ERR_INVALID with ffb6d_rgb_add_noise's ffb6d_last_error() text for a bad record.
 * A caller that replays a captured call (whose records are copied to plan_dev) checks each batch with it. */
int ffb6d_rgb_noise_check_records(const double *plan_host, int64_t B);
int ffb6d_add_real_back(const uint8_t *rgb, const uint8_t *labels, const uint16_t *dpt,
                        const uint8_t *back_rgb, const uint8_t *back_labels, int back_label_channels,
                        const uint16_t *back_dpt, const uint8_t *mode, int dataset,
                        int64_t B, int64_t H, int64_t W, uint8_t *rgb_out, uint16_t *dpt_out, ffb6d_stream_t stream);
int ffb6d_aug_noise_field(uint64_t seed, int64_t B, int64_t H, int64_t W, int stage, double *out,
                          ffb6d_stream_t stream);

/*
 * Colour jitter of training frames: torchvision's ColorJitter(0.2, 0.2, 0.2, 0.05) on a PIL RGB image
 * (datasets/ycb/ycb_dataset.py:34, 190-193; datasets/linemod/linemod_dataset.py:35, 220-223), bitwise as
 * torchvision 0.26 with Pillow 12.2 computes it (DESIGN.md §4.15).
 *   rgb [B,H,W,3] u8 -> out [B,H,W,3] u8 (out may equal rgb, but may not overlap it otherwise).
 *   plan_host / plan_dev [B,FFB6D_JITTER_PLAN_LEN] f64, the same bytes on the host (validated) and on the device
 *   (read by the kernels): slots 0-3 the order of the ops (a permutation of 0 brightness, 1 contrast, 2 saturation,
 *   3 hue), slots 4-7 the brightness, contrast and saturation factors (finite, >= 0, <= FLT_MAX) and the hue
 *   factor (|hue| <= 0.5), as ColorJitter.get_params draws them (ffb6d_b200/augment.py draw_color_jitter).
 *   active [B] u8 (device): frames with 0 are copied through unchanged.
 *   work [B] int64 (device, 8-byte aligned, overlapping neither image): the frames' sums of L, zeroed by the call.
 * 1 <= B < 65536, 1 <= H, W < 2^20, H*W*3 < 2^31.  Sizes, null pointers, alignment and every plan are checked before
 * any launch (FFB6D_ERR_INVALID).  A memset and two launches; no allocation, no host synchronisation (capturable in a
 * CUDA graph); deterministic.
 */
#define FFB6D_JITTER_PLAN_LEN 8
int ffb6d_color_jitter(const uint8_t *rgb, int64_t B, int64_t H, int64_t W, const double *plan_host,
                       const double *plan_dev, const uint8_t *active, uint8_t *out, int64_t *work,
                       ffb6d_stream_t stream);
/* The plan checks of ffb6d_color_jitter alone, on the host, without a launch: plan_host [B,FFB6D_JITTER_PLAN_LEN]
 * f64, 1 <= B < 65536.  0 or FFB6D_ERR_INVALID with ffb6d_color_jitter's ffb6d_last_error() text for a bad plan. */
int ffb6d_color_jitter_check_plans(const double *plan_host, int64_t B);

/*
 * FFB6D's training loss (models/loss.py:12-90, combined as train_ycb.py:237-253): FocalLoss and the offset L1 loss
 * of_l1_loss / OFLoss, each with an optional per-frame mask valid [B] u8 (device; NULL: every frame).  A frame with
 * valid[b] == 0 adds nothing to any sum or count and gets zero gradients, so every output equals the reference's on
 * the sub-batch of valid frames.  Labels [B,N] int32 or int64 (labels_is_i64).
 *
 * ffb6d_focal_loss_fwd: logits [B,C,N] (layout 0, the head's) or [B,N,C] (layout 1: the reference's reshaped rows,
 *   e.g. an [M,C] input as B = 1, N = M); 1 <= C <= 256; gamma finite, >= 0; alpha [C] f32 (device) or NULL.
 *   pt = exp(logpt) is a constant of the backward, as the reference's Variable(logpt.data.exp()).  Writes the loss
 *   (mean over the M counted points when size_average, else the sum), acc = (arg-max == label) / M with the lowest
 *   index winning ties, count = M (int64, for the backward) and lse [B,N] (0 on masked frames).  With M = 0 (every
 *   frame masked) loss and acc are 0 and the backward writes zeros.  A label outside [0, C) is not read through: its
 *   term and its gradients are NaN.  workspace: ffb6d_loss_workspace_bytes(B, N, any n_kps), 16-byte aligned.
 * ffb6d_focal_loss_bwd: grad_logits (same layout) from the saved lse and count and the upstream grad_loss [1]
 *   (device): dz_j = g_t [j == t] - exp(z_j - lse) g_t, g_t = -(1 - pt)^gamma alpha[t] g / M (g when not
 *   size_average).  One launch.
 * ffb6d_of_l1_loss_fwd: pred [B,n_kps,N,3] (the head's layout), targ [B,N,n_kps,3] (the item's layout),
 *   w_n = labels[b,n] > 0; 1 <= n_kps <= FFB6D_ITEM_MAX_KPS.  out [B,n_kps] = S_bk / (float(cnt_b) + 1e-3f) with
 *   S_bk = sum_n sum_c w_n |pred - targ| (fp64) and cnt_b = sum_n w_n, saved in count [B] f32 (0 on masked frames,
 *   whose out is 0).  workspace: ffb6d_loss_workspace_bytes(B, N, n_kps), 16-byte aligned.
 * ffb6d_of_l1_loss_bwd: grad_pred [B,n_kps,N,3] = (g_bk / (count_b + 1e-3f)) * w_n * sign(pred - targ) in fp32,
 *   sign(0) = 0, for any upstream grad_out [B,n_kps] (device): bitwise the reference's autograd.  One launch.
 * 1 <= B < 65536, 1 <= N < 2^31 - 128.  Sizes, null pointers and alignment are checked before any launch
 * (FFB6D_ERR_INVALID; a short workspace FFB6D_ERR_WORKSPACE).  A forward is two launches (partials per CTA, then
 * one finalize that adds them in a fixed order); no allocation, no host synchronisation (capturable in a CUDA
 * graph), no atomics (deterministic).  ffb6d_loss_workspace_bytes returns 0 for sizes the calls reject.
 */
size_t ffb6d_loss_workspace_bytes(int64_t B, int64_t N, int64_t n_kps);
int ffb6d_focal_loss_fwd(const float *logits, int layout, const void *labels, int labels_is_i64,
                         const uint8_t *valid, int64_t B, int64_t C, int64_t N, float gamma, const float *alpha,
                         int size_average, float *loss, float *acc, int64_t *count, float *lse,
                         void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
int ffb6d_focal_loss_bwd(const float *logits, int layout, const void *labels, int labels_is_i64,
                         const uint8_t *valid, int64_t B, int64_t C, int64_t N, float gamma, const float *alpha,
                         int size_average, const float *lse, const int64_t *count, const float *grad_loss,
                         float *grad_logits, ffb6d_stream_t stream);
int ffb6d_of_l1_loss_fwd(const float *pred, const float *targ, const void *labels, int labels_is_i64,
                         const uint8_t *valid, int64_t B, int64_t n_kps, int64_t N, float *out, float *count,
                         void *workspace, size_t workspace_bytes, ffb6d_stream_t stream);
int ffb6d_of_l1_loss_bwd(const float *pred, const float *targ, const void *labels, int labels_is_i64,
                         const uint8_t *valid, int64_t B, int64_t n_kps, int64_t N, const float *count,
                         const float *grad_out, float *grad_pred, ffb6d_stream_t stream);

/*
 * The PSP head of FFB6D's image branch at inference (models/cnn/pspnet.py:7-31, 108-112; DESIGN.md §4.17).
 *
 * ffb6d_psp_pool: AdaptiveAvgPool2d at the sizes 1, 2, 3 and 6 of x [B,C,H,W] f32 in one read, with torch's bins
 *   (bin i of s over n: [floor(i n / s), ceil((i + 1) n / s)), overlapping where s does not divide n).  out holds the
 *   50 B C bins scale-major: [B,C,1,1], [B,C,2,2], [B,C,3,3], [B,C,6,6] one after the other, each block equal to
 *   adaptive_avg_pool2d(x, s).  Sums in fp64.  1 <= B, C; B C < 2^31; 1 <= H <= 1024; 1 <= W < 2^24.  One launch.
 * ffb6d_psp_bottleneck_fwd: out [B,Co,H,W] = relu(W_f x + bias + sum_s up_s(T_s)), the bottleneck of PSPModule with
 *   its concat split by input block (W = [W_1|W_2|W_3|W_6|W_f]) and the stage convs moved behind the pooling:
 *   T_s = W_s C_s pool_s(x).  packed = ffb6d_fusion_mlp_pack of W_f [Co, C]; bias [Co]; table [B*50, Co] f32, the
 *   four T_s channels-last, in the block order of ffb6d_psp_pool ([B, s*s, Co] for s = 1, 2, 3, 6, e.g. made by
 *   ffb6d_fusion_mlp_fwd_ex with out_layout FFB6D_LAYOUT_NSC).  up_s is torch's bilinear upsampling with
 *   align_corners=False, all four taps read (a NaN at a zero-weight tap propagates, as in torch).  3xTF32 on wgmma,
 *   like the fusion layers.  1 <= B < 65536; H + W <= 3072; B * 50 * Co < 2^31.  One launch.
 * ffb6d_conv1x1_log_softmax_fwd: out [B,Co,P] = log_softmax(W x + bias, dim=1) for x [B,Ci,P] f32, packed =
 *   ffb6d_fusion_mlp_pack of W [Co, Ci], bias [Co]; 1 <= Co <= 128 (every channel of a pixel in one output tile).
 *   out = y - max - log(sum exp(y - max)) per pixel, NaN / +-inf propagate as torch's log_softmax.  One launch.
 * All three check sizes and null pointers before any launch (FFB6D_ERR_INVALID); no allocation, no host
 * synchronisation (capturable in a CUDA graph), no atomics.
 */
int ffb6d_psp_pool(const float *x, int64_t B, int64_t C, int64_t H, int64_t W, float *out, ffb6d_stream_t stream);
int ffb6d_psp_bottleneck_fwd(const float *x, int64_t B, int64_t C, int64_t H, int64_t W, const void *packed,
                             const float *bias, int64_t Co, const float *table, float *out, ffb6d_stream_t stream);
int ffb6d_conv1x1_log_softmax_fwd(const float *x, int64_t B, int64_t Ci, int64_t P, const void *packed,
                                  const float *bias, int64_t Co, float *out, ffb6d_stream_t stream);

/*
 * The backward of the PSP head and of PSPUpsample's upsampling, for training (DESIGN.md §4.18).  All four check
 * sizes, null pointers and 4-byte alignment before any launch (FFB6D_ERR_INVALID); one launch each, no allocation,
 * no host synchronisation (capturable in a CUDA graph), no atomics: every output element is written once, its sum
 * taken in a fixed order, so results are bit-identical from run to run (torch.use_deterministic_algorithms).
 *
 * ffb6d_psp_bottleneck_bwd: backward of ffb6d_psp_bottleneck_fwd from grad_out and the forward's out [B,Co,H,W]:
 *   grad_z = threshold_backward(grad_out, out, 0) (0 where out <= 0, grad_out elsewhere, as torch's ReLU backward on
 *   its result); grad_table [B*50, Co], laid out as the forward's table, = the adjoint of sum_s up_s(T_s) applied to
 *   grad_z, with the forward's taps, every tap's product added (weight 0 too); grad_sum [B*Co] = the sum of each
 *   (frame, channel) plane of grad_z (the bias gradient is its sum over the frames).  Sums in fp64.
 *   1 <= B, Co; H, W <= 1024 with H*104 + (H + W)*64 <= 227 KB of shared memory; B Co < 2^31.
 * ffb6d_psp_pool_bwd: adjoint of ffb6d_psp_pool: grad_x [B,C,H,W] += sum over the bins of the four sizes that contain
 *   a pixel of grad_pooled[bin] / area(bin), grad_pooled in ffb6d_psp_pool's block order.  grad_x must hold a value
 *   (e.g. the bottleneck's input gradient W_f^T grad_z); the sum is in fp64, rounded once into it.
 *   H <= 1024, W <= 16384, B C < 2^31.
 * ffb6d_log_softmax_bwd: grad_in = grad_out - exp(out) * sum_c grad_out per pixel, for out, grad_out [B,C,P]
 *   (channel stride P; torch's _log_softmax_backward_data, NaN / +-inf propagating as there).  B < 65536.
 * ffb6d_upsample_bilinear2d_bwd: backward of upsample_bilinear2d(align_corners=True) from grad_out [B,C,Ho,Wo] to
 *   grad_in [B,C,Hi,Wi] (written, not added), with torch's float taps (scale = (float)(in-1)/(out-1), 0 when out == 1),
 *   weight-0 taps included.  Every size < 2^24.
 */
int ffb6d_psp_bottleneck_bwd(const float *grad_out, const float *out, int64_t B, int64_t Co, int64_t H, int64_t W,
                             float *grad_z, float *grad_table, float *grad_sum, ffb6d_stream_t stream);
int ffb6d_psp_pool_bwd(const float *grad_pooled, int64_t B, int64_t C, int64_t H, int64_t W, float *grad_x,
                       ffb6d_stream_t stream);
int ffb6d_log_softmax_bwd(const float *grad_out, const float *out, int64_t B, int64_t C, int64_t P, float *grad_in,
                          ffb6d_stream_t stream);
int ffb6d_upsample_bilinear2d_bwd(const float *grad_out, int64_t B, int64_t C, int64_t Hi, int64_t Wi, int64_t Ho,
                                  int64_t Wo, float *grad_in, ffb6d_stream_t stream);

/*
 * PSPUpsample (x2 bilinear upsampling with align_corners=True, 3x3 conv with padding 1, BatchNorm, PReLU) at the
 * input's resolution (DESIGN.md §4.23): conv3x3(up(x)) + b = b + sum_t S_t(up(W_t x)), W_t = W[:, :, ky, kx],
 * t = 3 ky + kx, S_t the shift to tap t on the upsampled grid.  The stacked product T = [W_0; ..; W_8] x of a chunk
 * of Cc output channels co0 .. co0 + Cc - 1 (row t Cc + j = W[co0 + j, :, ky, kx]) is ffb6d_fusion_mlp_fwd_ex with
 * the packed stacked weight; T is [B, 9 Cc, Hi, Wi].  Ho = 2 Hi, Wo = 2 Wi.  The taps are torch's float taps (as
 * ffb6d_upsample_bilinear2d_bwd), all four read even at weight 0.  Every call checks sizes (1 <= B, Co, Cc, Hi, Wi;
 * 0 <= co0, co0 + Cc <= Co; Hi, Wi < 2^23; B Co, 9 B Cc < 2^31), null pointers and 4-byte alignment before any
 * launch (FFB6D_ERR_INVALID); one launch each, no allocation, no host synchronisation, no atomics: every output
 * element is written once, its sum taken in a fixed order.
 *
 * ffb6d_upconv_taps_fwd: out[b, co0 + j, y, x] = act(affine(bias[co] + sum_t sum_4 lambda T[b, t Cc + j, src])) into
 *   out [B, Co, Ho, Wo] (the chunk's channels only).  bias may be NULL (0); scale and shift (folded eval BatchNorm,
 *   v * scale + shift) both or neither; alpha (PReLU's one weight, read on the device) may be NULL (no activation).
 * ffb6d_upconv_taps_bwd: the adjoint, grad_table [B, 9 Cc, Hi, Wi] = up^T(S_t^T grad_z[:, co0 + j]) from
 *   grad_z [B, Co, Ho, Wo], sums in fp64.
 * ffb6d_prelu_fwd: y = x > 0 ? x : alpha[0] x over n elements (x may be y).  n < 2^50.
 * ffb6d_bn_prelu_bwd: the backward of PReLU(u), u the training BatchNorm's output, recomputed from z [B, C, P] and the
 *   stats [C, 4] of ffb6d_bn_train_fwd / ffb6d_bn_sync_fwd (16-byte aligned) as those kernels compute it: grad_u =
 *   u > 0 ? grad_y : alpha grad_y, and grad_alpha_part [B C] fp64 (8-byte aligned), each (frame, channel) row's sum of
 *   u grad_y where u <= 0, added in a fixed order.  B C < 2^31.
 */
int ffb6d_upconv_taps_fwd(const float *table, int64_t B, int64_t Co, int64_t co0, int64_t Cc, int64_t Hi, int64_t Wi,
                          const float *bias, const float *scale, const float *shift, const float *alpha, float *out,
                          ffb6d_stream_t stream);
int ffb6d_upconv_taps_bwd(const float *grad_z, int64_t B, int64_t Co, int64_t co0, int64_t Cc, int64_t Hi, int64_t Wi,
                          float *grad_table, ffb6d_stream_t stream);
int ffb6d_prelu_fwd(const float *x, int64_t n, const float *alpha, float *y, ffb6d_stream_t stream);
int ffb6d_bn_prelu_bwd(const float *z, const float *grad_y, const float *stats, int64_t B, int64_t C, int64_t P,
                       const float *alpha, float *grad_u, double *grad_alpha_part, ffb6d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FFB6D_B200_H_ */
