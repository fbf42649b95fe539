// psp.cuh -- the bin and tap conventions of PSPModule (models/cnn/pspnet.py:19-31), shared by the pyramid pooling and
// its adjoint (psp.cu), the restructured bottleneck's epilogue (fusion_mlp.cu) and its adjoint (psp.cu), so that the
// forward and the backward of the PSP head cannot disagree on a bin bound or a tap (DESIGN.md 4.17, 4.18).
#pragma once

namespace ffb6d {

// the four sizes k = 0..3 (s = 1, 2, 3, 6): the size, its first range among the 12, its first bin among the 50
__device__ __forceinline__ int psp_size_k(int k) { return (k == 0) ? 1 : (k == 1) ? 2 : (k == 2) ? 3 : 6; }
__device__ __forceinline__ int psp_first_range(int k) { return (k == 0) ? 0 : (k == 1) ? 1 : (k == 2) ? 3 : 6; }
__device__ __forceinline__ int psp_bin_offset(int k) { return (k == 0) ? 0 : (k == 1) ? 1 : (k == 2) ? 5 : 14; }
// the size index of range r of the 12
__device__ __forceinline__ int psp_range_size_k(int r) { return (r == 0) ? 0 : (r < 3) ? 1 : (r < 6) ? 2 : 3; }

// range r of the 12 adaptive-average ranges of the four sizes along an axis of length n: sizes 1 (r = 0), 2 (1-2),
// 3 (3-5), 6 (6-11).  torch's bins (aten/src/ATen/native/AdaptiveAveragePooling.cpp): bin i of s covers
// [floor(i n / s), ceil((i + 1) n / s)), overlapping where s does not divide n and repeating where n < s.
__device__ __forceinline__ void pool_range(int r, int n, int &lo, int &hi, int &s, int &i)
{
    const int k = psp_range_size_k(r);
    s = psp_size_k(k);
    i = r - psp_first_range(k);
    lo = (int)(((long long)i * n) / s);
    hi = (int)(((long long)(i + 1) * n + s - 1) / s);
}

// bin t of the 50, in the block order of the pooling's output: size index k, size s, the size's first bin off among
// the 50, row bin i and column bin j (t = off + i * s + j)
__device__ __forceinline__ void psp_bin(int t, int &k, int &s, int &off, int &i, int &j)
{
    k = (t == 0) ? 0 : (t < 5) ? 1 : (t < 14) ? 2 : 3;
    s = psp_size_k(k);
    off = psp_bin_offset(k);
    i = (t - off) / s;
    j = (t - off) % s;
}

// one output coordinate's two source taps along one axis (torch upsample_bilinear2d, align_corners=False)
struct PspTap {
    int i0, i1;
    float l0, l1;
};

__device__ __forceinline__ PspTap psp_tap(int dst, int out_size, int in_size)
{
    // area_pixel_compute_source_index: src = (in / out) * (dst + 0.5) - 0.5, clamped at 0; in double like the
    // float64 reference, so that the tap index agrees with it wherever src is not within round-off of an integer
    double src = (double)in_size / (double)out_size * ((double)dst + 0.5) - 0.5;
    if (src < 0.0) src = 0.0;
    PspTap t;
    t.i0 = min((int)src, in_size - 1);
    t.i1 = t.i0 + ((t.i0 < in_size - 1) ? 1 : 0);
    const double l1 = src - (double)t.i0;
    t.l1 = (float)l1;
    t.l0 = (float)(1.0 - l1);
    return t;
}

// One axis of upsample_bilinear2d with align_corners=True (PSPUpsample's x2), in torch's float arithmetic: scale =
// (float)(in - 1) / (out - 1) (0 when out == 1), src = scale * dst, i0 = (int)src, i1 = i0 + (i0 < in - 1),
// lambda1 = src - i0, lambda0 = 1 - lambda1.  Shared by the upsampling's adjoint (psp.cu) and the restructured
// upsample + 3x3 conv (upconv.cu), so that both read the taps torch's forward reads.
struct AcAxis {
    float scale;
    int in, out;
    __device__ __forceinline__ int i0(int dst) const
    {
        return min((int)__fmul_rn(scale, (float)dst), in - 1);
    }
    // the first dst whose i0 is >= t (out if none)
    __device__ __forceinline__ int first_ge(int t) const
    {
        int d = (scale > 0.f) ? (int)fmin((double)t / (double)scale, (double)out) : (t <= 0 ? 0 : out);
        d = max(0, min(d, out));
        while (d > 0 && i0(d - 1) >= t) --d;
        while (d < out && i0(d) < t) ++d;
        return d;
    }
    // the two source coordinates of dst and their weights
    __device__ __forceinline__ void taps(int dst, int &a0, int &a1, float &l0, float &l1) const
    {
        const float src = __fmul_rn(scale, (float)dst);
        a0 = min((int)src, in - 1);
        a1 = a0 + ((a0 < in - 1) ? 1 : 0);
        l1 = __fsub_rn(src, (float)a0);
        l0 = __fsub_rn(1.f, l1);
    }
    // the weights with which dst taps v: i0(dst) == v contributes lambda0, i1(dst) == v lambda1
    __device__ __forceinline__ void tap(int dst, int v, bool &h0, float &l0, bool &h1, float &l1) const
    {
        int a, a1;
        taps(dst, a, a1, l0, l1);
        h0 = (a == v);
        h1 = (a1 == v);
    }
};

__device__ __forceinline__ AcAxis ac_axis(int in, int out)
{
    return AcAxis{(out > 1) ? (float)(in - 1) / (float)(out - 1) : 0.f, in, out};
}

}  // namespace ffb6d
