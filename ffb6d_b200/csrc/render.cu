// render.cu -- z-buffer rasteriser of vertex-coloured meshes on the device (sm_90a), DESIGN.md §4.31.
//
// The specification is the header's (ffb6d_render_rgbd) and oracle/render_oracle.py restates it in numpy.  Every
// float64 operation is a separately rounded _rn intrinsic and the coverage test is exact integer arithmetic, so the
// frames are bitwise the oracle's.
//
// Stages, all with launch shapes that depend on the arguments only:
//   memset     the key buffer to all-ones (empty) and the queue counter to 0;
//   vertex     one thread per (frame, slot, vertex): fixed-point (U, V) and 1/Z into the workspace, 1/Z = 0 if culled
//              (a vertex that is not culled has a finite Z >= z_near, so its 1/Z is positive);
//   raster     faces in a grid-stride loop, one thread per face over its pixel box, atomicMin of the 64-bit key.  A face
//              whose box holds more than FFB6D_RND_BIG_FACE_PIXELS pixels is pushed to a queue instead (when the queue
//              is full the thread draws it itself: slower, same result);
//   drain      a fixed grid of CTAs, one queued face per CTA at a time, its box's pixels over the CTA's threads;
//   resolve    one thread per pixel: the winning face's barycentrics recomputed from the workspace, depth (or dpt_mm),
//              colour and label written with coalesced stores.
// The key is (float32 depth bits << 32) | (slot max_faces + face): the depth is positive, so its bits order as the
// values, and one atomicMin takes the nearest face, a tie the lower (slot, face), whatever the order of the atomics.
#include "common.cuh"

#include <algorithm>
#include <cfloat>

namespace ffb6d {
namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kEmpty = ~0ull;

struct __align__(16) Vtx {
    int U, V;       // 1/256-pixel fixed point
    double iz;      // 1/Z; 0 marks a culled vertex
};

struct Args {
    const float *xyz;
    const uint8_t *vrgb;
    const int32_t *faces;
    const int64_t *vert_off, *face_off;
    int64_t n_meshes, max_verts, max_faces;
    const int32_t *mesh_idx;
    const float *RTs;
    const uint8_t *label;
    int64_t B, M;
    const double *intr;
    int intr_per_frame;
    int H, W;
    double z_near;
    const uint8_t *active;
    float *depth;
    uint16_t *depth_mm;
    uint8_t *rgb, *labels;
    unsigned long long *keys;
    Vtx *vtx;
    unsigned long long *count;
    long long *queue;
};

__device__ __forceinline__ bool frame_on(const Args &a, int64_t b) { return !a.active || a.active[b] != 0; }

// the slot's mesh, or -1 when it draws nothing (empty slot, or an index outside the table)
__device__ __forceinline__ int slot_mesh(const Args &a, int64_t b, int64_t s)
{
    const int m = __ldg(a.mesh_idx + b * a.M + s);
    return (m >= 0 && m < a.n_meshes) ? m : -1;
}

__device__ __forceinline__ long long floor256(long long x) { return x >> 8; }        // arithmetic shift: floor
__device__ __forceinline__ long long ceil256(long long x) { return -((-x) >> 8); }

__global__ void __launch_bounds__(kThreads) vertex_kernel(Args a)
{
    const int64_t total = a.B * a.M * a.max_verts;
    for (int64_t g = blockIdx.x * (int64_t)kThreads + threadIdx.x; g < total; g += (int64_t)gridDim.x * kThreads) {
        const int64_t v = g % a.max_verts, bs = g / a.max_verts, s = bs % a.M, b = bs / a.M;
        if (!frame_on(a, b)) continue;
        const int m = slot_mesh(a, b, s);
        if (m < 0) continue;
        const int64_t v0 = __ldg(a.vert_off + m);
        if (v >= __ldg(a.vert_off + m + 1) - v0) continue;
        const float *p = a.xyz + (v0 + v) * 3;
        const double x = (double)__ldg(p), y = (double)__ldg(p + 1), z = (double)__ldg(p + 2);
        const float *rt = a.RTs + bs * 12;
        double c[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float *row = rt + 4 * r;
            c[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)__ldg(row), x), __dmul_rn((double)__ldg(row + 1), y)),
                                       __dmul_rn((double)__ldg(row + 2), z)),
                             (double)__ldg(row + 3));
        }
        Vtx o = {0, 0, 0.0};
        if (c[2] >= a.z_near && c[2] <= DBL_MAX) {          // culled: nearer than z_near, or not finite
            const double *k = a.intr + (a.intr_per_frame ? b * 4 : 0);
            const double u = __dadd_rn(__dmul_rn(__ldg(k), __ddiv_rn(c[0], c[2])), __ldg(k + 2));
            const double w = __dadd_rn(__dmul_rn(__ldg(k + 1), __ddiv_rn(c[1], c[2])), __ldg(k + 3));
            if (fabs(u) <= (double)FFB6D_RND_GUARD_BAND && fabs(w) <= (double)FFB6D_RND_GUARD_BAND) {
                o.U = (int)__double2ll_rn(__dmul_rn(u, 256.0));
                o.V = (int)__double2ll_rn(__dmul_rn(w, 256.0));
                o.iz = __ddiv_rn(1.0, c[2]);
            }
        }
        a.vtx[g] = o;
    }
}

// One face of one slot in one frame, set up for coverage: its vertices, the sign-normalised doubled area, the owned
// edges and its pixel box.  ok = false when it draws nothing.
struct Face {
    long long x[3], y[3];
    double iz[3];
    long long A;
    long long sgn;
    bool own[3];
    int i0, i1, j0, j1;
    int64_t vbase;
    int f3[3];
};

__device__ __forceinline__ bool setup_face(const Args &a, int64_t b, int64_t s, int64_t f, Face &F)
{
    const int m = slot_mesh(a, b, s);
    if (m < 0) return false;
    const int64_t f0 = __ldg(a.face_off + m);
    if (f >= __ldg(a.face_off + m + 1) - f0) return false;
    const int32_t *fi = a.faces + (f0 + f) * 3;
    F.vbase = (b * a.M + s) * a.max_verts;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        F.f3[k] = __ldg(fi + k);
        const Vtx t = a.vtx[F.vbase + F.f3[k]];
        if (t.iz == 0.0) return false;
        F.x[k] = t.U;
        F.y[k] = t.V;
        F.iz[k] = t.iz;
    }
    const long long A = (F.x[1] - F.x[0]) * (F.y[2] - F.y[0]) - (F.y[1] - F.y[0]) * (F.x[2] - F.x[0]);
    if (A == 0) return false;
    F.sgn = A > 0 ? 1 : -1;
    F.A = A * F.sgn;
#pragma unroll
    for (int k = 0; k < 3; ++k) {           // edge k is E(V[k+1], V[k+2], .), opposite vertex k
        const int p = (k + 1) % 3, q = (k + 2) % 3;
        const long long dx = F.sgn * (F.x[q] - F.x[p]), dy = F.sgn * (F.y[q] - F.y[p]);
        F.own[k] = dy < 0 || (dy == 0 && dx > 0);
    }
    const long long xmin = min(F.x[0], min(F.x[1], F.x[2])), xmax = max(F.x[0], max(F.x[1], F.x[2]));
    const long long ymin = min(F.y[0], min(F.y[1], F.y[2])), ymax = max(F.y[0], max(F.y[1], F.y[2]));
    F.i0 = (int)max(ceil256(xmin), 0ll);
    F.i1 = (int)min(floor256(xmax), (long long)a.W - 1);
    F.j0 = (int)max(ceil256(ymin), 0ll);
    F.j1 = (int)min(floor256(ymax), (long long)a.H - 1);
    return F.i0 <= F.i1 && F.j0 <= F.j1;
}

// the sign-normalised edge values at pixel (i, j); false when the pixel is not covered
__device__ __forceinline__ bool cover(const Face &F, int i, int j, long long w[3])
{
    const long long px = 256ll * i, py = 256ll * j;
    bool in = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int p = (k + 1) % 3, q = (k + 2) % 3;
        w[k] = F.sgn * ((F.x[q] - F.x[p]) * (py - F.y[p]) - (F.y[q] - F.y[p]) * (px - F.x[p]));
        in = in && (w[k] > 0 || (w[k] == 0 && F.own[k]));
    }
    return in;
}

__device__ __forceinline__ void weights(const Face &F, const long long w[3], double p[3], double &S)
{
#pragma unroll
    for (int k = 0; k < 3; ++k) p[k] = __dmul_rn((double)w[k], F.iz[k]);
    S = __dadd_rn(__dadd_rn(p[0], p[1]), p[2]);
}

__device__ __forceinline__ void draw_pixel(const Face &F, int i, int j, unsigned long long *keys, unsigned long long idx,
                                           int W)
{
    long long w[3];
    if (!cover(F, i, j, w)) return;
    double p[3], S;
    weights(F, w, p, S);
    const float d = __double2float_rn(__ddiv_rn((double)F.A, S));
    const unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | idx;
    unsigned long long *k = keys + (int64_t)j * W + i;
    if (key < *k) atomicMin(k, key);      // the plain read only skips atomics that could not win
}

__global__ void __launch_bounds__(kThreads) raster_kernel(Args a)
{
    const int64_t total = a.B * a.M * a.max_faces;
    const int64_t HW = (int64_t)a.H * a.W;
    for (int64_t g = blockIdx.x * (int64_t)kThreads + threadIdx.x; g < total; g += (int64_t)gridDim.x * kThreads) {
        const int64_t f = g % a.max_faces, bs = g / a.max_faces, s = bs % a.M, b = bs / a.M;
        if (!frame_on(a, b)) continue;
        Face F;
        if (!setup_face(a, b, s, f, F)) continue;
        const int64_t box = (int64_t)(F.i1 - F.i0 + 1) * (F.j1 - F.j0 + 1);
        if (box > FFB6D_RND_BIG_FACE_PIXELS) {
            const unsigned long long slot = atomicAdd(a.count, 1ull);
            if (slot < (unsigned long long)FFB6D_RND_QUEUE_CAP) {
                a.queue[slot] = g;
                continue;
            }
        }
        unsigned long long *keys = a.keys + b * HW;
        const unsigned long long idx = (unsigned long long)(s * a.max_faces + f);
        for (int j = F.j0; j <= F.j1; ++j)
            for (int i = F.i0; i <= F.i1; ++i) draw_pixel(F, i, j, keys, idx, a.W);
    }
}

__global__ void __launch_bounds__(kThreads) drain_kernel(Args a)
{
    const unsigned int n = (unsigned int)min(*a.count, (unsigned long long)FFB6D_RND_QUEUE_CAP);
    const int64_t HW = (int64_t)a.H * a.W;
    for (unsigned int e = blockIdx.x; e < n; e += gridDim.x) {
        const int64_t g = a.queue[e];
        const int64_t f = g % a.max_faces, bs = g / a.max_faces, s = bs % a.M, b = bs / a.M;
        Face F;
        if (!setup_face(a, b, s, f, F)) continue;       // not reached: only drawable faces are queued
        const int bw = F.i1 - F.i0 + 1;
        const int64_t box = (int64_t)bw * (F.j1 - F.j0 + 1);
        unsigned long long *keys = a.keys + b * HW;
        const unsigned long long idx = (unsigned long long)(s * a.max_faces + f);
        for (int64_t t = threadIdx.x; t < box; t += kThreads)
            draw_pixel(F, F.i0 + (int)(t % bw), F.j0 + (int)(t / bw), keys, idx, a.W);
    }
}

__global__ void __launch_bounds__(kThreads) resolve_kernel(Args a)
{
    const int64_t b = blockIdx.y;
    if (!frame_on(a, b)) return;
    const int64_t HW = (int64_t)a.H * a.W;
    for (int64_t px = blockIdx.x * (int64_t)kThreads + threadIdx.x; px < HW; px += (int64_t)gridDim.x * kThreads) {
        const int64_t o = b * HW + px;
        const unsigned long long key = a.keys[o];
        float d = 0.0f;
        uint8_t c[3] = {0, 0, 0}, lab = 0;
        if (key != kEmpty) {
            const int64_t idx = (int64_t)(key & 0xffffffffull), s = idx / a.max_faces, f = idx % a.max_faces;
            Face F;
            setup_face(a, b, s, f, F);
            long long w[3];
            const int j = (int)(px / a.W), i = (int)(px % a.W);
            cover(F, i, j, w);
            double p[3], S;
            weights(F, w, p, S);
            d = __uint_as_float((unsigned int)(key >> 32));
            const uint8_t *col = a.vrgb + (__ldg(a.vert_off + slot_mesh(a, b, s))) * 3;
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const double n = __dadd_rn(__dadd_rn(__dmul_rn(p[0], (double)__ldg(col + F.f3[0] * 3 + ch)),
                                                     __dmul_rn(p[1], (double)__ldg(col + F.f3[1] * 3 + ch))),
                                           __dmul_rn(p[2], (double)__ldg(col + F.f3[2] * 3 + ch)));
                const double r = floor(__dadd_rn(__ddiv_rn(n, S), 0.5));
                c[ch] = (uint8_t)fmin(fmax(r, 0.0), 255.0);
            }
            lab = __ldg(a.label + b * a.M + s);
        }
        if (a.depth_mm)
            a.depth_mm[o] = (uint16_t)min(__float2uint_rz(__fmul_rn(d, 1000.0f)), 65535u);
        else
            a.depth[o] = d;
        uint8_t *rgb = a.rgb + o * 3;
        rgb[0] = c[0];
        rgb[1] = c[1];
        rgb[2] = c[2];
        a.labels[o] = lab;
    }
}

// ---------------------------------------------------------------------------------------- textured meshes, §4.35
// The vertex, raster and drain stages above are shared; only the resolve differs: the colour comes from the mesh's
// mipmapped texture through per-vertex UVs (ffb6d_render_rgbd_textured in the header states every step).
struct Tex {
    const float *uv;
    const uint8_t *tex;
    const int32_t *hw;       // (Th, Tw) of level 0 per mesh
    const int64_t *off;      // texel offset of level l of mesh m at m FFB6D_RND_MAX_TEX_LEVELS + l
};

__device__ __forceinline__ int n_levels(int Th, int Tw) { return 32 - __clz(max(Th, Tw)); }
__device__ __forceinline__ int64_t wrap(int64_t n, int64_t size)
{
    const int64_t r = n % size;
    return r < 0 ? r + size : r;
}

// one bilinear sample of level l of mesh m, unrounded, per channel
__device__ __forceinline__ void bilinear(const Tex &t, int m, int l, int Th, int Tw, double u, double v, double c[3])
{
    const int64_t Wl = max(1, Tw >> l), Hl = max(1, Th >> l);
    const double x = __dsub_rn(__dmul_rn(u, (double)Wl), 0.5);
    const double y = __dsub_rn(__dmul_rn(__dsub_rn(1.0, v), (double)Hl), 0.5);
    const double xf = floor(x), yf = floor(y);
    const double fx = __dsub_rn(x, xf), fy = __dsub_rn(y, yf);
    const double gx = __dsub_rn(1.0, fx), gy = __dsub_rn(1.0, fy);
    const double w00 = __dmul_rn(gx, gy), w10 = __dmul_rn(fx, gy), w01 = __dmul_rn(gx, fy), w11 = __dmul_rn(fx, fy);
    const int64_t x0 = wrap((int64_t)xf, Wl), x1 = wrap((int64_t)xf + 1, Wl);
    const int64_t y0 = wrap((int64_t)yf, Hl), y1 = wrap((int64_t)yf + 1, Hl);
    const uint8_t *base = t.tex + 3 * __ldg(t.off + (int64_t)m * FFB6D_RND_MAX_TEX_LEVELS + l);
    const uint8_t *t00 = base + 3 * (y0 * Wl + x0), *t10 = base + 3 * (y0 * Wl + x1);
    const uint8_t *t01 = base + 3 * (y1 * Wl + x0), *t11 = base + 3 * (y1 * Wl + x1);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch)
        c[ch] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(w00, (double)__ldg(t00 + ch)), __dmul_rn(w10, (double)__ldg(t10 + ch))),
                                    __dmul_rn(w01, (double)__ldg(t01 + ch))),
                          __dmul_rn(w11, (double)__ldg(t11 + ch)));
}

// the filtered colour of pixel (i, j) of face F (covered, weights p and S) of mesh m
__device__ __forceinline__ void texel_colour(const Tex &t, const Face &F, int m, const int64_t v0, const double p[3],
                                             double S, uint8_t out[3])
{
    double uk[3], vk[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float *q = t.uv + (v0 + F.f3[k]) * 2;
        uk[k] = (double)__ldg(q);
        vk[k] = (double)__ldg(q + 1);
    }
    const double u = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[0], uk[0]), __dmul_rn(p[1], uk[1])), __dmul_rn(p[2], uk[2])), S);
    const double v = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[0], vk[0]), __dmul_rn(p[1], vk[1])), __dmul_rn(p[2], vk[2])), S);
    double ux = 0.0, uy = 0.0, vx = 0.0, vy = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        // (gx_k (1/Z_k)) and (gy_k (1/Z_k)): the steps of p_k per pixel
        const double sx = __dmul_rn((double)(-256ll * F.sgn * (F.y[b] - F.y[a])), F.iz[k]);
        const double sy = __dmul_rn((double)(256ll * F.sgn * (F.x[b] - F.x[a])), F.iz[k]);
        const double du = __dsub_rn(uk[k], u), dv = __dsub_rn(vk[k], v);
        // k = 0 starts each sum with its first term, so the sums are ((t0 + t1) + t2)
        ux = k ? __dadd_rn(ux, __dmul_rn(sx, du)) : __dmul_rn(sx, du);
        uy = k ? __dadd_rn(uy, __dmul_rn(sy, du)) : __dmul_rn(sy, du);
        vx = k ? __dadd_rn(vx, __dmul_rn(sx, dv)) : __dmul_rn(sx, dv);
        vy = k ? __dadd_rn(vy, __dmul_rn(sy, dv)) : __dmul_rn(sy, dv);
    }
    ux = __ddiv_rn(ux, S);
    uy = __ddiv_rn(uy, S);
    vx = __ddiv_rn(vx, S);
    vy = __ddiv_rn(vy, S);
    const int Th = __ldg(t.hw + 2 * m), Tw = __ldg(t.hw + 2 * m + 1);
    const double fw = (double)Tw, fh = (double)Th;
    const double ax = __dmul_rn(ux, fw), bx = __dmul_rn(vx, fh), ay = __dmul_rn(uy, fw), by = __dmul_rn(vy, fh);
    const double r1 = __dsqrt_rn(__dadd_rn(__dmul_rn(ax, ax), __dmul_rn(bx, bx)));
    const double r2 = __dsqrt_rn(__dadd_rn(__dmul_rn(ay, ay), __dmul_rn(by, by)));
    const double rho = r2 > r1 ? r2 : r1;
    const int L = n_levels(Th, Tw);
    double c[3];
    if (!(rho > 1.0) || rho >= (double)(1 << (L - 1))) {
        bilinear(t, m, rho > 1.0 ? L - 1 : 0, Th, Tw, u, v, c);
    } else {
        const int e = ilogb(rho);
        const double w = __dsub_rn(scalbn(rho, -e), 1.0), w0 = __dsub_rn(1.0, w);
        double c1[3];
        bilinear(t, m, e, Th, Tw, u, v, c);
        bilinear(t, m, e + 1, Th, Tw, u, v, c1);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) c[ch] = __dadd_rn(__dmul_rn(w0, c[ch]), __dmul_rn(w, c1[ch]));
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) out[ch] = (uint8_t)fmin(fmax(floor(__dadd_rn(c[ch], 0.5)), 0.0), 255.0);
}

__global__ void __launch_bounds__(kThreads) resolve_textured_kernel(Args a, Tex t)
{
    const int64_t b = blockIdx.y;
    if (!frame_on(a, b)) return;
    const int64_t HW = (int64_t)a.H * a.W;
    for (int64_t px = blockIdx.x * (int64_t)kThreads + threadIdx.x; px < HW; px += (int64_t)gridDim.x * kThreads) {
        const int64_t o = b * HW + px;
        const unsigned long long key = a.keys[o];
        float d = 0.0f;
        uint8_t c[3] = {0, 0, 0}, lab = 0;
        if (key != kEmpty) {
            const int64_t idx = (int64_t)(key & 0xffffffffull), s = idx / a.max_faces, f = idx % a.max_faces;
            Face F;
            setup_face(a, b, s, f, F);
            long long w[3];
            const int j = (int)(px / a.W), i = (int)(px % a.W);
            cover(F, i, j, w);
            double p[3], S;
            weights(F, w, p, S);
            d = __uint_as_float((unsigned int)(key >> 32));
            const int m = slot_mesh(a, b, s);
            texel_colour(t, F, m, __ldg(a.vert_off + m), p, S, c);
            lab = __ldg(a.label + b * a.M + s);
        }
        if (a.depth_mm)
            a.depth_mm[o] = (uint16_t)min(__float2uint_rz(__fmul_rn(d, 1000.0f)), 65535u);
        else
            a.depth[o] = d;
        uint8_t *rgb = a.rgb + o * 3;
        rgb[0] = c[0];
        rgb[1] = c[1];
        rgb[2] = c[2];
        a.labels[o] = lab;
    }
}

// level l + 1 of every mesh's chain from level l; per_mesh = the largest level-(l + 1) texel count
__global__ void __launch_bounds__(kThreads) mip_kernel(uint8_t *tex, const int32_t *hw, const int64_t *off,
                                                       int64_t n_meshes, int l, int64_t per_mesh)
{
    const int64_t total = n_meshes * per_mesh;
    for (int64_t g = blockIdx.x * (int64_t)kThreads + threadIdx.x; g < total; g += (int64_t)gridDim.x * kThreads) {
        const int64_t m = g / per_mesh, k = g % per_mesh;
        const int Th = __ldg(hw + 2 * m), Tw = __ldg(hw + 2 * m + 1);
        if (l + 1 >= n_levels(Th, Tw)) continue;
        const int64_t Ws = max(1, Tw >> l), Hs = max(1, Th >> l);
        const int64_t Wd = max(1, Tw >> (l + 1)), Hd = max(1, Th >> (l + 1));
        if (k >= Wd * Hd) continue;
        const int64_t i = k % Wd, j = k / Wd;
        const int64_t xa = min(2 * i, Ws - 1), xb = min(2 * i + 1, Ws - 1);
        const int64_t ya = min(2 * j, Hs - 1), yb = min(2 * j + 1, Hs - 1);
        const uint8_t *src = tex + 3 * __ldg(off + m * FFB6D_RND_MAX_TEX_LEVELS + l);
        uint8_t *dst = tex + 3 * __ldg(off + m * FFB6D_RND_MAX_TEX_LEVELS + l + 1) + 3 * k;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const int s = (int)src[3 * (ya * Ws + xa) + ch] + src[3 * (ya * Ws + xb) + ch] + src[3 * (yb * Ws + xa) + ch] +
                          src[3 * (yb * Ws + xb) + ch];
            dst[ch] = (uint8_t)((s + 2) >> 2);
        }
    }
}

static inline bool aligned(const void *p, size_t a) { return ((uintptr_t)p % a) == 0; }

bool sizes_ok(int64_t B, int64_t M, int64_t H, int64_t W, int64_t max_verts, int64_t max_faces)
{
    return B >= 0 && B <= FFB6D_RND_MAX_FRAMES && H >= 1 && W >= 1 && H <= FFB6D_RND_MAX_FRAME_PIXELS &&
           W <= FFB6D_RND_MAX_FRAME_PIXELS && H * W <= FFB6D_RND_MAX_FRAME_PIXELS && M >= 1 &&
           M <= FFB6D_RND_MAX_SLOTS && max_verts >= 1 && max_verts <= FFB6D_RND_MAX_MESH_VERTS && max_faces >= 1 &&
           max_faces <= FFB6D_RND_MAX_FRAME_FACES && M * max_faces <= FFB6D_RND_MAX_FRAME_FACES &&
           (B == 0 || max_faces <= ((int64_t)1 << 62) / (B * M));
}

// workspace layout, each part 16-byte aligned: [counter][keys B H W, rounded up to 16 B][vertices B M max_verts][queue]
constexpr size_t kHead = 16;
inline size_t key_bytes_of(int64_t B, int64_t H, int64_t W)
{
    return align_up((size_t)B * H * W * sizeof(unsigned long long), 16);
}

}  // namespace
}  // namespace ffb6d

using namespace ffb6d;

extern "C" size_t ffb6d_render_workspace_bytes(int64_t B, int64_t M, int64_t H, int64_t W, int64_t max_verts,
                                               int64_t max_faces)
{
    if (!sizes_ok(B, M, H, W, max_verts, max_faces)) return 0;
    return kHead + key_bytes_of(B, H, W) + (size_t)B * M * max_verts * sizeof(Vtx) +
           (size_t)FFB6D_RND_QUEUE_CAP * sizeof(long long);
}

namespace ffb6d {
namespace {

// The argument checks both entry points share, with `name` leading every message: everything but the colour source.
int check_geometry(const char *name, const float *xyz, const int32_t *faces, const int64_t *vert_off,
                   const int64_t *face_off, int64_t n_meshes, int64_t max_verts, int64_t max_faces,
                   const int32_t *mesh_idx, const float *RTs, const uint8_t *label, int64_t B, int64_t M,
                   const double *intrinsics, int intrinsics_per_frame, int64_t H, int64_t W, double z_near,
                   const float *depth, const uint16_t *depth_mm, const uint8_t *rgb, const uint8_t *labels,
                   const void *workspace, const void *colour_src)
{
    FFB6D_CHECK_ARG(sizes_ok(B, M, H, W, max_verts, max_faces),
                    "%s: bad size (B=%lld M=%lld H=%lld W=%lld max_verts=%lld max_faces=%lld)", name, (long long)B,
                    (long long)M, (long long)H, (long long)W, (long long)max_verts, (long long)max_faces);
    FFB6D_CHECK_ARG(n_meshes >= 1 && n_meshes <= 2147483647ll, "%s: n_meshes=%lld outside [1, 2^31)", name,
                    (long long)n_meshes);
    FFB6D_CHECK_ARG(z_near >= 0.001 && z_near < INFINITY, "%s: z_near=%g must be finite and >= 0.001 m", name,
                    z_near);
    FFB6D_CHECK_ARG(intrinsics_per_frame == 0 || intrinsics_per_frame == 1,
                    "%s: intrinsics_per_frame must be 0 or 1", name);
    if (B == 0) return FFB6D_OK;
    FFB6D_CHECK_ARG((depth == nullptr) != (depth_mm == nullptr),
                    "%s: exactly one of depth and depth_mm must be given (null pointer)", name);
    FFB6D_CHECK_ARG(xyz && colour_src && faces && vert_off && face_off && mesh_idx && RTs && label && intrinsics &&
                    rgb && labels, "%s: null pointer", name);
    FFB6D_CHECK_ARG(aligned(xyz, 4) && aligned(faces, 4) && aligned(vert_off, 8) && aligned(face_off, 8) &&
                    aligned(mesh_idx, 4) && aligned(RTs, 4) && aligned(intrinsics, 8) && aligned(depth, 4) &&
                    aligned(depth_mm, 2) && aligned(workspace, 16), "%s: misaligned pointer", name);
    return FFB6D_OK;
}

int check_workspace(const char *name, int64_t B, int64_t M, int64_t H, int64_t W, int64_t max_verts,
                    int64_t max_faces, const void *workspace, size_t workspace_bytes)
{
    const size_t need = ffb6d_render_workspace_bytes(B, M, H, W, max_verts, max_faces);
    if (!workspace || workspace_bytes < need) {
        set_error("%s: workspace of %zu bytes, %zu needed", name, workspace_bytes, need);
        return FFB6D_ERR_WORKSPACE;
    }
    return FFB6D_OK;
}

// The stages before the resolve, shared by both entry points: the workspace carved into `a`, then the memsets and
// the vertex, raster and drain launches.
int enqueue_geometry(Args &a, void *workspace, cudaStream_t st)
{
    char *ws = (char *)workspace;
    const size_t key_bytes = key_bytes_of(a.B, a.H, a.W);     // keeps the Vtx array 16-byte aligned for odd B H W
    a.count = (unsigned long long *)ws;
    a.keys = (unsigned long long *)(ws + kHead);
    a.vtx = (Vtx *)(ws + kHead + key_bytes);
    a.queue = (long long *)(ws + kHead + key_bytes + (size_t)a.B * a.M * a.max_verts * sizeof(Vtx));
    // the queue counter to 0, every key to all-ones (empty)
    FFB6D_CUDA(cudaMemsetAsync(a.count, 0, kHead, st));
    FFB6D_CUDA(cudaMemsetAsync(a.keys, 0xff, key_bytes, st));
    const int64_t grid_cap = (int64_t)num_sms() * 16;
    const unsigned vb = (unsigned)std::min<int64_t>(ceil_div(a.B * a.M * a.max_verts, kThreads), grid_cap);
    vertex_kernel<<<vb, kThreads, 0, st>>>(a);
    FFB6D_LAUNCH_OK("render_vertex_kernel");
    const unsigned rb = (unsigned)std::min<int64_t>(ceil_div(a.B * a.M * a.max_faces, kThreads), grid_cap);
    raster_kernel<<<rb, kThreads, 0, st>>>(a);
    FFB6D_LAUNCH_OK("render_raster_kernel");
    drain_kernel<<<(unsigned)(num_sms() * 4), kThreads, 0, st>>>(a);
    FFB6D_LAUNCH_OK("render_drain_kernel");
    return FFB6D_OK;
}

Args make_args(const float *xyz, const uint8_t *vrgb, const int32_t *faces, const int64_t *vert_off,
               const int64_t *face_off, int64_t n_meshes, int64_t max_verts, int64_t max_faces,
               const int32_t *mesh_idx, const float *RTs, const uint8_t *label, int64_t B, int64_t M,
               const double *intrinsics, int intrinsics_per_frame, int64_t H, int64_t W, double z_near,
               const uint8_t *active, float *depth, uint16_t *depth_mm, uint8_t *rgb, uint8_t *labels)
{
    Args a;
    a.xyz = xyz;
    a.vrgb = vrgb;
    a.faces = faces;
    a.vert_off = vert_off;
    a.face_off = face_off;
    a.n_meshes = n_meshes;
    a.max_verts = max_verts;
    a.max_faces = max_faces;
    a.mesh_idx = mesh_idx;
    a.RTs = RTs;
    a.label = label;
    a.B = B;
    a.M = M;
    a.intr = intrinsics;
    a.intr_per_frame = intrinsics_per_frame;
    a.H = (int)H;
    a.W = (int)W;
    a.z_near = z_near;
    a.active = active;
    a.depth = depth;
    a.depth_mm = depth_mm;
    a.rgb = rgb;
    a.labels = labels;
    return a;
}

inline unsigned resolve_blocks(int64_t H, int64_t W) { return (unsigned)std::min<int64_t>(ceil_div(H * W, kThreads), 1 << 16); }

}  // namespace
}  // namespace ffb6d

extern "C" int ffb6d_render_rgbd(const float *xyz, const uint8_t *vrgb, const int32_t *faces, const int64_t *vert_off,
                                 const int64_t *face_off, int64_t n_meshes, int64_t max_verts, int64_t max_faces,
                                 const int32_t *mesh_idx, const float *RTs, const uint8_t *label, int64_t B, int64_t M,
                                 const double *intrinsics, int intrinsics_per_frame, int64_t H, int64_t W,
                                 double z_near, const uint8_t *active, float *depth, uint16_t *depth_mm, uint8_t *rgb,
                                 uint8_t *labels, void *workspace, size_t workspace_bytes, ffb6d_stream_t stream)
{
    const char *name = "render_rgbd";
    int rc = check_geometry(name, xyz, faces, vert_off, face_off, n_meshes, max_verts, max_faces, mesh_idx, RTs,
                            label, B, M, intrinsics, intrinsics_per_frame, H, W, z_near, depth, depth_mm, rgb, labels,
                            workspace, vrgb);
    if (rc != FFB6D_OK || B == 0) return rc;
    rc = check_workspace(name, B, M, H, W, max_verts, max_faces, workspace, workspace_bytes);
    if (rc != FFB6D_OK) return rc;
    Args a = make_args(xyz, vrgb, faces, vert_off, face_off, n_meshes, max_verts, max_faces, mesh_idx, RTs, label, B,
                       M, intrinsics, intrinsics_per_frame, H, W, z_near, active, depth, depth_mm, rgb, labels);
    cudaStream_t st = (cudaStream_t)stream;
    rc = enqueue_geometry(a, workspace, st);
    if (rc != FFB6D_OK) return rc;
    resolve_kernel<<<dim3(resolve_blocks(H, W), (unsigned)B), kThreads, 0, st>>>(a);
    FFB6D_LAUNCH_OK("render_resolve_kernel");
    return FFB6D_OK;
}

// the texture table's own checks, shared by both textured entry points
static int check_textures(const char *name, const void *tex, const int32_t *tex_hw, const int64_t *tex_off,
                          int64_t max_tex_side)
{
    FFB6D_CHECK_ARG(max_tex_side >= 1 && max_tex_side <= FFB6D_RND_MAX_TEX_SIDE,
                    "%s: max_tex_side=%lld outside [1, %d]", name, (long long)max_tex_side, FFB6D_RND_MAX_TEX_SIDE);
    FFB6D_CHECK_ARG(tex && tex_hw && tex_off, "%s: null pointer (texture table)", name);
    FFB6D_CHECK_ARG(aligned(tex_hw, 4) && aligned(tex_off, 8), "%s: misaligned pointer (texture table)", name);
    return FFB6D_OK;
}

extern "C" int ffb6d_render_texture_mips(uint8_t *tex, const int32_t *tex_hw, const int64_t *tex_off, int64_t n_meshes,
                                         int64_t max_tex_side, ffb6d_stream_t stream)
{
    const char *name = "render_texture_mips";
    FFB6D_CHECK_ARG(n_meshes >= 1 && n_meshes <= 2147483647ll, "%s: n_meshes=%lld outside [1, 2^31)", name,
                    (long long)n_meshes);
    const int rc = check_textures(name, tex, tex_hw, tex_off, max_tex_side);
    if (rc != FFB6D_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t grid_cap = (int64_t)num_sms() * 16;
    for (int l = 0; (max_tex_side >> (l + 1)) >= 1; ++l) {
        const int64_t side = max_tex_side >> (l + 1), per_mesh = side * side;
        const unsigned g = (unsigned)std::min<int64_t>(ceil_div(n_meshes * per_mesh, kThreads), grid_cap);
        mip_kernel<<<g, kThreads, 0, st>>>(tex, tex_hw, tex_off, n_meshes, l, per_mesh);
        FFB6D_LAUNCH_OK("render_mip_kernel");
    }
    return FFB6D_OK;
}

extern "C" int ffb6d_render_rgbd_textured(const float *xyz, const float *uv, const int32_t *faces,
                                          const int64_t *vert_off, const int64_t *face_off, const uint8_t *tex,
                                          const int32_t *tex_hw, const int64_t *tex_off, int64_t max_tex_side,
                                          int64_t n_meshes, int64_t max_verts, int64_t max_faces,
                                          const int32_t *mesh_idx, const float *RTs, const uint8_t *label, int64_t B,
                                          int64_t M, const double *intrinsics, int intrinsics_per_frame, int64_t H,
                                          int64_t W, double z_near, const uint8_t *active, float *depth,
                                          uint16_t *depth_mm, uint8_t *rgb, uint8_t *labels, void *workspace,
                                          size_t workspace_bytes, ffb6d_stream_t stream)
{
    const char *name = "render_rgbd_textured";
    int rc = check_geometry(name, xyz, faces, vert_off, face_off, n_meshes, max_verts, max_faces, mesh_idx, RTs,
                            label, B, M, intrinsics, intrinsics_per_frame, H, W, z_near, depth, depth_mm, rgb, labels,
                            workspace, uv);
    if (rc != FFB6D_OK) return rc;
    FFB6D_CHECK_ARG(max_tex_side >= 1 && max_tex_side <= FFB6D_RND_MAX_TEX_SIDE,
                    "%s: max_tex_side=%lld outside [1, %d]", name, (long long)max_tex_side, FFB6D_RND_MAX_TEX_SIDE);
    if (B == 0) return FFB6D_OK;
    rc = check_textures(name, tex, tex_hw, tex_off, max_tex_side);
    if (rc != FFB6D_OK) return rc;
    FFB6D_CHECK_ARG(aligned(uv, 4), "%s: misaligned pointer (uv)", name);
    rc = check_workspace(name, B, M, H, W, max_verts, max_faces, workspace, workspace_bytes);
    if (rc != FFB6D_OK) return rc;
    Args a = make_args(xyz, nullptr, faces, vert_off, face_off, n_meshes, max_verts, max_faces, mesh_idx, RTs, label,
                       B, M, intrinsics, intrinsics_per_frame, H, W, z_near, active, depth, depth_mm, rgb, labels);
    const Tex t = {uv, tex, tex_hw, tex_off};
    cudaStream_t st = (cudaStream_t)stream;
    rc = enqueue_geometry(a, workspace, st);
    if (rc != FFB6D_OK) return rc;
    resolve_textured_kernel<<<dim3(resolve_blocks(H, W), (unsigned)B), kThreads, 0, st>>>(a, t);
    FFB6D_LAUNCH_OK("render_resolve_textured_kernel");
    return FFB6D_OK;
}
