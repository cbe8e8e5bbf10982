// vpt_temporal.cu -- the sm_90a kernel of vpt_temporal (include/vpt_b200.h, DESIGN.md section 8p): temporal accumulation of a moving
// camera's frames.  Each pixel's history is carried from the previous output through the motion vectors, clipped to the current frame's
// 3x3 neighbourhood and blended with accum's own running-mean arithmetic.  tests/temporal_ref.py restates it in NumPy.
//
//   k_temporal : one thread per pixel: motion (vectors + the environment's motion at infinity), bilinear history fetch, clip, blend,
//                display word; then the layers of vpt_temporal_layers (section 8r), blended with the beauty's taps and L_new
//
// Deterministic: every pixel is one thread reading its taps in a fixed order, no atomics.  Compiled with vpt_kernels.cu's flags
// (--use_fast_math), so the blend's division and the display words are k_resolve's own.  Includes neither vpt_math.cuh nor the trace
// machinery (see vpt_film.cuh).
#include "vpt_kernels.h"
#include "vpt_film.cuh"
#include "vpt_tonemap.cuh"

namespace vpt {

namespace {

__device__ __forceinline__ bool finite3(const float3 c) { return isfinite(c.x) && isfinite(c.y) && isfinite(c.z); }
__device__ __forceinline__ float3 ldg3(const float* p, size_t i) { return make_float3(__ldg(p + 3 * i), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2)); }

// The pixel's film motion v towards the history's camera B: the vectors' premultiplied collision motion plus the uncovered share's
// environment motion.  False: the pixel has no history (the environment's direction is not in front of A or B while M.z < 1).
__device__ __forceinline__ bool pixel_motion(const TemporalArgs& a, const int x, const int y, const float3 m, float2* v)
{
    v->x = m.x; v->y = m.y;
    if (!(m.z < 1.0f)) return true;
    const vpt_u2 res = { (uint32_t)a.width, (uint32_t)a.height };
    const FilmCam A = film_cam(a.a_origin, a.a_llc, a.a_horizontal, a.a_vertical);
    const FilmCam B = film_cam(a.b_origin, a.b_llc, a.b_horizontal, a.b_vertical);
    const float s = __fdiv_rn(__fadd_rn((float)x, 0.5f), (float)a.width), t = __fdiv_rn(__fadd_rn((float)y, 0.5f), (float)a.height);
    const float3 d = make_float3(__fmaf_rn(t, A.v.x, __fmaf_rn(s, A.h.x, A.e.x)), __fmaf_rn(t, A.v.y, __fmaf_rn(s, A.h.y, A.e.y)),
                                 __fmaf_rn(t, A.v.z, __fmaf_rn(s, A.h.z, A.e.z)));
    float2 pa, pb;
    if (!film_project_dir(A, d, res, &pa) || !film_project_dir(B, d, res, &pb)) return false;
    const float w = __fsub_rn(1.0f, m.z);
    v->x = __fmaf_rn(w, __fsub_rn(pb.x, pa.x), m.x);
    v->y = __fmaf_rn(w, __fsub_rn(pb.y, pa.y), m.y);
    return true;
}

// The bilinear footprint of q - 1/2, q = (x + 1/2, y + 1/2) + v: the first tap (x0, y0) and the fractions (fx, fy); tap k = 2 j + i is
// (x0 + i, y0 + j) with weight tap_weight(fx, fy, i, j).  False: no history (v not finite, or q outside [0, W] x [0, H]).
__device__ __forceinline__ bool footprint(const TemporalArgs& a, const int x, const int y, const float2 v, int* x0, int* y0, float* fx, float* fy)
{
    if (!isfinite(v.x) || !isfinite(v.y)) return false;
    const float qx = __fadd_rn(__fadd_rn((float)x, 0.5f), v.x), qy = __fadd_rn(__fadd_rn((float)y, 0.5f), v.y);
    if (!(qx >= 0.0f && qx <= (float)a.width && qy >= 0.0f && qy <= (float)a.height)) return false;
    const float px = __fsub_rn(qx, 0.5f), py = __fsub_rn(qy, 0.5f);
    const float fx0 = floorf(px), fy0 = floorf(py);
    *fx = __fsub_rn(px, fx0); *fy = __fsub_rn(py, fy0);
    *x0 = (int)fx0; *y0 = (int)fy0;
    return true;
}

__device__ __forceinline__ float tap_weight(const float fx, const float fy, const int i, const int j)
{
    return __fmul_rn(i ? fx : __fsub_rn(1.0f, fx), j ? fy : __fsub_rn(1.0f, fy));
}

// The history at q: the footprint's taps that lie in the frame, weigh more than 0 and hold a finite colour, renormalised; *len the least
// history length among them; *used the taps used (bit k = 2 j + i), *sw their weights' sum in tap order.  The layers are blended with
// exactly these taps (tap_mean).  False: no history.
__device__ __forceinline__ bool fetch_history(const TemporalArgs& a, const int x, const int y, const float2 v, float3* h, float* len,
                                              unsigned* used, float* sw_out)
{
    int x0, y0;
    float fx, fy;
    if (!footprint(a, x, y, v, &x0, &y0, &fx, &fy)) return false;
    float sw = 0.0f, l = 0.0f;
    float3 sh = make_float3(0.0f, 0.0f, 0.0f);
    unsigned u = 0u;
    #pragma unroll
    for (int j = 0; j < 2; ++j) {
        #pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int tx = x0 + i, ty = y0 + j;
            const float w = tap_weight(fx, fy, i, j);
            if (!(w > 0.0f) || tx < 0 || ty < 0 || tx >= a.width || ty >= a.height) continue;
            const size_t tp = (size_t)ty * a.width + tx;
            const float3 c = ldg3(a.history, tp);
            if (!finite3(c)) continue;
            const float tl = __ldg(a.history_len + tp);
            l = sw > 0.0f ? fminf(l, tl) : tl;
            sw = __fadd_rn(sw, w);
            sh = make_float3(__fmaf_rn(w, c.x, sh.x), __fmaf_rn(w, c.y, sh.y), __fmaf_rn(w, c.z, sh.z));
            u |= 1u << (2 * j + i);
        }
    }
    if (!(sw > 0.0f)) return false;
    *h = make_float3(__fdiv_rn(sh.x, sw), __fdiv_rn(sh.y, sw), __fdiv_rn(sh.z, sw));
    *len = l;
    *used = u; *sw_out = sw;
    return true;
}

// The taps fetch_history used, for the layers: footprint, used mask and weight sum
struct Taps {
    int      x0, y0;
    unsigned used;
    float    fx, fy, sw;
};

// Channel ch of an nc-channel history plane at the beauty's taps: sum(w H) / sum(w) in the beauty's order and arithmetic
__device__ __forceinline__ float tap_mean(const TemporalArgs& a, const Taps& t, const float* plane, const unsigned nc, const unsigned ch)
{
    const float* q = plane + ((ptrdiff_t)t.y0 * a.width + t.x0) * (ptrdiff_t)nc + ch;   // tap 0, which may lie outside the frame
    const unsigned row = (unsigned)a.width * nc;
    float s = 0.0f;
    #pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (!((t.used >> k) & 1u)) continue;
        const int i = k & 1, j = k >> 1;
        s = __fmaf_rn(tap_weight(t.fx, t.fy, i, j), __ldg(q + (j * row + i * nc)), s);
    }
    return __fdiv_rn(s, t.sw);
}

// accum's running mean as resolve_pixel writes it, accum + (value - accum) / (float)(iteration + 1), with len for iteration + 1
__device__ __forceinline__ float blend(const float h, const float c, const float len) { return h + (c - h) / len; }

// h clamped per channel to mu +- gamma sigma of the current frame's finite colours in the 3x3 window (clipped at the frame edge)
__device__ __forceinline__ float3 clip_history(const TemporalArgs& a, const int x, const int y, const float3 h)
{
    float3 c[9];
    int n = 0;
    float3 sum = make_float3(0.0f, 0.0f, 0.0f);
    #pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
        #pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int tx = x + dx, ty = y + dy;
            const int k = (dy + 1) * 3 + dx + 1;
            c[k] = make_float3(NAN, NAN, NAN);
            if (tx < 0 || ty < 0 || tx >= a.width || ty >= a.height) continue;
            const float3 v = ldg3(a.color, (size_t)ty * a.width + tx);
            if (!finite3(v)) continue;
            c[k] = v; ++n;
            sum = make_float3(__fadd_rn(sum.x, v.x), __fadd_rn(sum.y, v.y), __fadd_rn(sum.z, v.z));
        }
    }
    const float fn = (float)n;
    const float3 mu = make_float3(__fdiv_rn(sum.x, fn), __fdiv_rn(sum.y, fn), __fdiv_rn(sum.z, fn));
    float3 ss = make_float3(0.0f, 0.0f, 0.0f);
    #pragma unroll
    for (int k = 0; k < 9; ++k) {
        if (isnan(c[k].x)) continue;
        const float3 d = make_float3(__fsub_rn(c[k].x, mu.x), __fsub_rn(c[k].y, mu.y), __fsub_rn(c[k].z, mu.z));
        ss = make_float3(__fmaf_rn(d.x, d.x, ss.x), __fmaf_rn(d.y, d.y, ss.y), __fmaf_rn(d.z, d.z, ss.z));
    }
    const float3 r = make_float3(__fmul_rn(a.clip_sigma, __fsqrt_rn(__fdiv_rn(ss.x, fn))), __fmul_rn(a.clip_sigma, __fsqrt_rn(__fdiv_rn(ss.y, fn))),
                                 __fmul_rn(a.clip_sigma, __fsqrt_rn(__fdiv_rn(ss.z, fn))));
    return make_float3(fminf(fmaxf(h.x, __fsub_rn(mu.x, r.x)), __fadd_rn(mu.x, r.x)), fminf(fmaxf(h.y, __fsub_rn(mu.y, r.y)), __fadd_rn(mu.y, r.y)),
                       fminf(fmaxf(h.z, __fsub_rn(mu.z, r.z)), __fadd_rn(mu.z, r.z)));
}

} // namespace

__global__ void __launch_bounds__(256) k_temporal(const __grid_constant__ TemporalArgs a)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= a.width || y >= a.height) return;
    const size_t p = (size_t)y * a.width + x;
    const float3 c = ldg3(a.color, p);
    float3 out = c;
    float len = 1.0f;
    float2 v;
    float3 h;
    float lh;
    Taps t;
    t.used = 0u;
    if (a.history && finite3(c) && pixel_motion(a, x, y, ldg3(a.vectors, p), &v) && fetch_history(a, x, y, v, &h, &lh, &t.used, &t.sw)) {
        if (isfinite(a.clip_sigma)) h = clip_history(a, x, y, h);
        len = fminf(lh + 1.0f, (float)a.max_history);
        out = make_float3(blend(h.x, c.x, len), blend(h.y, c.y, len), blend(h.z, c.z, len));
    }
    a.out[3 * p] = out.x; a.out[3 * p + 1] = out.y; a.out[3 * p + 2] = out.z;
    a.out_len[p] = len;
    if (a.out_display) a.out_display[p] = tonemap_display(out, a.exposure_scale).word;
    if (a.n_layers == 0) return;
    // the layers: every channel of every plane with the beauty's taps and L_new, unclipped; no history (t.used == 0): the value itself.
    // The footprint is recomputed from v rather than kept across the clip, whose 3x3 window needs the registers.
    const bool have = t.used != 0u;
    if (have) footprint(a, x, y, v, &t.x0, &t.y0, &t.fx, &t.fy);
    const size_t n = (size_t)a.width * a.height;
    for (int l = 0; l < a.n_layers; ++l) {
        const TemporalLayer& L = a.layers[l];
        const unsigned nc = L.channels;
        for (unsigned k = 0; k < L.count; ++k) {
            const size_t base = (size_t)k * n * nc;
            for (unsigned ch = 0; ch < nc; ++ch) {
                const size_t i = base + p * nc + ch;
                const float xv = __ldg(L.src + i);
                L.dst[i] = have ? blend(tap_mean(a, t, L.history + base, nc, ch), xv, len) : xv;
            }
        }
    }
}

cudaError_t launch_temporal(const TemporalArgs& a, cudaStream_t s)
{
    const dim3 block(32, 8), grid((a.width + 31) / 32, (a.height + 7) / 8);
    k_temporal<<<grid, block, 0, s>>>(a);
    return cudaGetLastError();
}

} // namespace vpt
