// fuse_frames.cu -- LineMOD's `fuse` frames on the device (sm_90a), DESIGN.md §4.34: object crops of real frames
// pasted into a frame.
//
// The specification is the header's (ffb6d_fuse_rgbd) and oracle/fuse_oracle.py restates it in numpy.  One launch,
// gather form: a CTA loads its frame's slot records into shared memory, then each thread owns output pixels (a
// grid-stride loop) and walks the records from the last slot to the first, stopping at the first crop that holds
// the pixel with its silhouette set.  Every output byte is written at most once and nothing is atomic, so the frames
// are bitwise the oracle's whatever the schedule.
#include "common.cuh"

#include <algorithm>

namespace ffb6d {
namespace {

constexpr int kThreads = 256;
constexpr unsigned kMaxGridX = 65535;

// one slot of one frame: where its crop sits in the frame and in the planes; h = w = 0 pastes nothing
struct __align__(16) Slot {
    long long off;      // the crop's first pixel in the planes
    int row, col;       // the crop's top-left corner in the frame
    int h, w;
    int label;
    int pad;
};
static_assert(sizeof(Slot) == 32, "slot records are 32 bytes");

struct Args {
    const uint8_t *crop_rgb;
    const uint16_t *crop_dpt;
    const uint8_t *crop_sil;
    const int64_t *crop_off;
    const int32_t *crop_hw;
    int64_t n_crops;
    const int32_t *crop;
    const int32_t *offset;
    const uint8_t *label;
    int M, H, W;
    const uint8_t *active;
    uint16_t *dpt_mm;
    uint8_t *rgb, *labels;
};

__global__ void __launch_bounds__(kThreads) fuse_kernel(Args a)
{
    extern __shared__ Slot slots[];
    const int64_t b = blockIdx.y;
    if (a.active && a.active[b] == 0) return;               // uniform over the CTA
    for (int s = threadIdx.x; s < a.M; s += kThreads) {
        const int64_t bs = b * a.M + s;
        const int c = __ldg(a.crop + bs);
        Slot t = {0, 0, 0, 0, 0, 0, 0};
        if (c >= 0 && c < a.n_crops) {
            t.off = __ldg(a.crop_off + c);
            t.h = __ldg(a.crop_hw + 2 * (int64_t)c);
            t.w = __ldg(a.crop_hw + 2 * (int64_t)c + 1);
            t.row = __ldg(a.offset + 2 * bs);
            t.col = __ldg(a.offset + 2 * bs + 1);
            t.label = __ldg(a.label + bs);
        }
        slots[s] = t;
    }
    __syncthreads();
    const int64_t HW = (int64_t)a.H * a.W;
    for (int64_t px = blockIdx.x * (int64_t)kThreads + threadIdx.x; px < HW; px += (int64_t)gridDim.x * kThreads) {
        const int r = (int)px / a.W, c = (int)px % a.W;     // H W < 2^31
        for (int s = a.M - 1; s >= 0; --s) {
            const Slot &t = slots[s];
            // r - row and c - col in int64: any int32 offset; a negative difference wraps above every size
            const unsigned long long dr = (unsigned long long)((long long)r - t.row);
            const unsigned long long dc = (unsigned long long)((long long)c - t.col);
            if (dr >= (unsigned long long)t.h || dc >= (unsigned long long)t.w) continue;
            const int64_t q = t.off + (int64_t)dr * t.w + (int64_t)dc;
            if (!__ldg(a.crop_sil + q)) continue;
            const int64_t o = b * HW + px;
            a.dpt_mm[o] = __ldg(a.crop_dpt + q);
            uint8_t *rgb = a.rgb + o * 3;
            const uint8_t *src = a.crop_rgb + q * 3;
            rgb[0] = __ldg(src);
            rgb[1] = __ldg(src + 1);
            rgb[2] = __ldg(src + 2);
            a.labels[o] = (uint8_t)t.label;
            break;
        }
    }
}

static inline bool aligned(const void *p, size_t a) { return ((uintptr_t)p % a) == 0; }

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" int ffb6d_fuse_rgbd(const uint8_t *crop_rgb, const uint16_t *crop_dpt, const uint8_t *crop_sil,
                               const int64_t *crop_off, const int32_t *crop_hw, int64_t n_crops, const int32_t *crop,
                               const int32_t *offset, const uint8_t *label, int64_t B, int64_t M, int64_t H, int64_t W,
                               const uint8_t *active, uint16_t *dpt_mm, uint8_t *rgb, uint8_t *labels,
                               ffb6d_stream_t stream)
{
    FFB6D_CHECK_ARG(B >= 0 && B <= FFB6D_FUSE_MAX_FRAMES && H >= 1 && W >= 1 && H <= FFB6D_FUSE_MAX_FRAME_PIXELS &&
                        W <= FFB6D_FUSE_MAX_FRAME_PIXELS && H * W <= FFB6D_FUSE_MAX_FRAME_PIXELS && M >= 1 &&
                        M <= FFB6D_FUSE_MAX_SLOTS,
                    "fuse_rgbd: bad size (B=%lld M=%lld H=%lld W=%lld)", (long long)B, (long long)M, (long long)H,
                    (long long)W);
    FFB6D_CHECK_ARG(n_crops >= 1 && n_crops <= FFB6D_FUSE_MAX_CROPS, "fuse_rgbd: n_crops=%lld outside [1, 2^31)",
                    (long long)n_crops);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG(crop_rgb && crop_dpt && crop_sil && crop_off && crop_hw && crop && offset && label && dpt_mm &&
                        rgb && labels, "fuse_rgbd: null pointer");
    FFB6D_CHECK_ARG(aligned(crop_dpt, 2) && aligned(crop_off, 8) && aligned(crop_hw, 4) && aligned(crop, 4) &&
                        aligned(offset, 4) && aligned(dpt_mm, 2), "fuse_rgbd: misaligned pointer");
    Args a;
    a.crop_rgb = crop_rgb;
    a.crop_dpt = crop_dpt;
    a.crop_sil = crop_sil;
    a.crop_off = crop_off;
    a.crop_hw = crop_hw;
    a.n_crops = n_crops;
    a.crop = crop;
    a.offset = offset;
    a.label = label;
    a.M = (int)M;
    a.H = (int)H;
    a.W = (int)W;
    a.active = active;
    a.dpt_mm = dpt_mm;
    a.rgb = rgb;
    a.labels = labels;
    const unsigned gx = (unsigned)std::min<int64_t>(ceil_div(H * W, kThreads), kMaxGridX);
    fuse_kernel<<<dim3(gx, (unsigned)B), kThreads, (size_t)M * sizeof(Slot), (cudaStream_t)stream>>>(a);
    FFB6D_LAUNCH_OK("fuse_kernel");
    return FFB6D_OK;
}
