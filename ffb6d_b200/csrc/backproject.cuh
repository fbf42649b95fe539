// backproject.cuh -- the one back-projection of a depth pixel, shared by backproject.cu and point_item.cu.
//
// Arithmetic is the reference's dpt_2_pcld (datasets/ycb/ycb_dataset.py:165-176), which numpy evaluates in
// float64 (integer pixel grid minus a float64 intrinsic): x = ((col - cx) * d) / fx, y = ((row - cy) * d) / fy,
// z = d, each multiplied by the validity mask (d > 1e-8 ? 1 : 0 -- holes become signed zeros).
#pragma once
#include "common.cuh"

namespace ffb6d {

// the float64 point, unrounded: what get_pose_gt_info subtracts the keypoints from
__device__ __forceinline__ void backproject_px64(const float *__restrict__ depth, int W, int row, int col,
                                                 double fx, double fy, double cx, double cy, double *o)
{
    const float d = __ldg(depth + (size_t)row * W + col);
    const double msk = (d > 1e-8f) ? 1.0 : 0.0;
    const double dd = (double)d;
    o[0] = __dmul_rn(__ddiv_rn(__dmul_rn((double)col - cx, dd), fx), msk);
    o[1] = __dmul_rn(__ddiv_rn(__dmul_rn((double)row - cy, dd), fy), msk);
    o[2] = __dmul_rn(dd, msk);
}

// the same point rounded once to float32, where the reference casts (`cld.astype(np.float32)`)
__device__ __forceinline__ void backproject_px(const float *__restrict__ depth, int W, int row, int col,
                                               double fx, double fy, double cx, double cy, float *o)
{
    double v[3];
    backproject_px64(depth, W, row, col, fx, fy, cx, cy, v);
    o[0] = __double2float_rn(v[0]);
    o[1] = __double2float_rn(v[1]);
    o[2] = __double2float_rn(v[2]);
}

}  // namespace ffb6d
