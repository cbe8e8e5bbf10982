// vpt_denoise.cu -- sm_90a kernels of vpt_denoise (include/vpt_b200.h): an edge-avoiding a-trous filter of a finished HDR frame,
// guided by the noise variance of each pixel's mean luminance and by the depth buffer.  tests/denoise_ref.py restates it in NumPy.
//
//   k_denoise_prep    : per pixel the luminance Y and the variance v (from vpt_render_adaptive's error map, or the 5x5 spatial variance
//                       of Y), into the planes {r, g, b, v} and {Y, z}
//   k_denoise_atrous  : one level of step 2^i: 3x3 Gaussian of v, 5x5 B3-spline taps weighted by luminance and depth similarity;
//                       reads plane pair i & 1 and writes the other, the last level writes the caller's outputs instead
//
// and of vpt_denoise_layers, which filters further layers with the beauty's weights (tests/denoise_layers_ref.py restates it):
//   k_denoise_layer_gather    : one layer's planes into float4 scratch planes, unused lanes 0
//   k_denoise_layers_atrous<G>: one level for G scratch planes, launched right after the beauty's level i and guided by the same plane
//                               pair i & 1 the beauty read (which beauty level i + 1 only overwrites later in stream order); the last
//                               level scatters into the callers' layers
//
// Deterministic: every pixel is one thread summing its taps in a fixed order, no atomics.  A level's planes (24 B per pixel) are read
// through the read-only path; at 1080p one level's pair is about the size of the L2.
#include "vpt_kernels.h"
#include "vpt_tonemap.cuh"

namespace vpt {

constexpr int kDnBlockX = 32, kDnBlockY = 8;

__device__ __forceinline__ bool finite_f(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }
__device__ __forceinline__ float luma(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

// Y of pixel q of the caller's colour; false for a pixel whose colour or luminance is not finite (copied, never a neighbour)
__device__ __forceinline__ bool color_luma(const float* __restrict__ color, size_t q, float& r, float& g, float& b, float& Y) {
    r = __ldg(color + 3 * q); g = __ldg(color + 3 * q + 1); b = __ldg(color + 3 * q + 2);
    Y = luma(r, g, b);
    return finite_f(r) && finite_f(g) && finite_f(b) && finite_f(Y);
}

__global__ void __launch_bounds__(kDnBlockX * kDnBlockY)
k_denoise_prep(const int w, const int h, const float* __restrict__ color, const float* __restrict__ depth, const float* __restrict__ rel_error,
               float4* __restrict__ cv, float2* __restrict__ yz)
{
    const int x = blockIdx.x * kDnBlockX + threadIdx.x, y = blockIdx.y * kDnBlockY + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t p = (size_t)y * w + x;
    float r, g, b, Y, v = 0.0f;
    const bool ok = color_luma(color, p, r, g, b, Y);
    if (ok && rel_error) {
        // err = sigma / max(mean, kAdaptMeanFloor) with the accumulated colour's Y for the mean; NaN or <= 0 -> 0, +inf stays +inf
        const float e = __ldg(rel_error + p);
        if (e > 0.0f) {
            const float s = e * fmaxf(Y, kAdaptMeanFloor);
            v = s * s;
        }
    } else if (ok) {
        // population variance of Y over the 5x5 window, clipped at the frame edge, finite pixels only; two passes
        float sum = 0.0f; int n = 0;
        for (int dy = -2; dy <= 2; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= h) continue;
            for (int dx = -2; dx <= 2; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= w) continue;
                float qr, qg, qb, qY;
                if (color_luma(color, (size_t)yy * w + xx, qr, qg, qb, qY)) { sum += qY; ++n; }
            }
        }
        const float mean = sum / (float)n;
        float ss = 0.0f;
        for (int dy = -2; dy <= 2; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= h) continue;
            for (int dx = -2; dx <= 2; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= w) continue;
                float qr, qg, qb, qY;
                if (color_luma(color, (size_t)yy * w + xx, qr, qg, qb, qY)) { const float d = qY - mean; ss += d * d; }
            }
        }
        v = ss / (float)n;
    }
    cv[p] = make_float4(r, g, b, v);
    yz[p] = make_float2(ok ? Y : __int_as_float(0x7fffffff), depth ? __ldg(depth + p) : 0.0f);   // a NaN Y marks a copied pixel
}

struct DenoiseLevel {
    int w, h, step, use_depth;
    float sigma_l, sigma_z, exposure_scale;
    const float4* cv_in; const float2* yz_in;
    float4* cv_out; float2* yz_out;          // inner levels
    float* out_f3; unsigned* out_display;    // last level (out_f3 != null)
};

// The weights and copy decision of one level for the layers: k_denoise_atrous's own, term for term, so that the layers take the very
// same taps and copy the very same pixels.  (k_denoise_atrous keeps its inline copy: calling these from it reorders fused multiply-adds
// in its inlined tonemap, which could move a display word.)  The layers-equal-beauty tests check both bit for bit.

// false for a pixel p = (x, y) that keeps its values bit for bit: its colour or luminance is not finite (yzp.x, the Y of yz_in[p], is
// NaN), or g, the 3x3 Gaussian of the level's v (cv_in[].w), is 0.  Otherwise true with inv_l = 1 / (sigma_l sqrt(g) + 1e-10).
__device__ __forceinline__ bool atrous_filters(const int w, const int h, const float sigma_l, const float4* cv_in, const int x, const int y,
                                               const float2 yzp, float& inv_l)
{
    const float kG3[3] = { 0.25f, 0.5f, 0.25f };               // Gaussian of v, per axis
    if (!finite_f(yzp.x)) return false;
    // g: 3x3 Gaussian of the current v, renormalised over the taps inside the frame
    float gs = 0.0f, gw = 0.0f;
    #pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= h) continue;
        #pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int xx = x + dx;
            if (xx < 0 || xx >= w) continue;
            const float k = kG3[dy + 1] * kG3[dx + 1];
            gs += k * __ldg(&cv_in[(size_t)yy * w + xx].w);
            gw += k;
        }
    }
    const float gv = gs / gw;
    if (!(gv > 0.0f)) return false;                            // g == 0: the pixel keeps its colour and variance bit for bit
    inv_l = 1.0f / (sigma_l * sqrtf(gv) + 1e-10f);
    return true;
}

// h w of tap (j, i) at q inside the frame for a filtered pixel p; false when the tap drops out.
__device__ __forceinline__ bool atrous_tap(const int use_depth, const float sigma_z, const float2* yz_in, const size_t p, const float2 yzp,
                                           const float inv_l, const int j, const int i, const size_t q, float& hw)
{
    const float kB3[5] = { 1.0f / 16.0f, 1.0f / 4.0f, 3.0f / 8.0f, 1.0f / 4.0f, 1.0f / 16.0f };   // B3-spline, per axis
    float wq = 1.0f;                                           // the centre tap weighs exactly 1
    if (q != p) {
        const float2 yzq = __ldg(yz_in + q);
        if (!finite_f(yzq.x)) return false;                    // non-finite neighbour: weight 0
        float e = fabsf(yzp.x - yzq.x) * inv_l;
        if (use_depth) e += fabsf(yzp.y - yzq.y) / (sigma_z * fmaxf(fabsf(yzp.y), fabsf(yzq.y)) + 1e-6f);
        wq = __expf(-e);
    }
    hw = kB3[j] * kB3[i] * wq;
    return hw > 0.0f;                                          // underflowed (or NaN from a NaN depth): the tap drops out
}

__global__ void __launch_bounds__(kDnBlockX * kDnBlockY)
k_denoise_atrous(const DenoiseLevel L)
{
    const int x = blockIdx.x * kDnBlockX + threadIdx.x, y = blockIdx.y * kDnBlockY + threadIdx.y;
    if (x >= L.w || y >= L.h) return;
    const float kB3[5] = { 1.0f / 16.0f, 1.0f / 4.0f, 3.0f / 8.0f, 1.0f / 4.0f, 1.0f / 16.0f };   // B3-spline, per axis
    const float kG3[3] = { 0.25f, 0.5f, 0.25f };                                                  // Gaussian of v, per axis
    const size_t p = (size_t)y * L.w + x;
    const float4 c = __ldg(L.cv_in + p);
    const float2 yzp = __ldg(L.yz_in + p);
    float4 o = c;
    float Yo = yzp.x;
    if (finite_f(yzp.x)) {
        // g: 3x3 Gaussian of the current v, renormalised over the taps inside the frame
        float gs = 0.0f, gw = 0.0f;
        #pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= L.h) continue;
            #pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= L.w) continue;
                const float k = kG3[dy + 1] * kG3[dx + 1];
                gs += k * __ldg(&L.cv_in[(size_t)yy * L.w + xx].w);
                gw += k;
            }
        }
        const float gv = gs / gw;
        if (gv > 0.0f) {                                       // g == 0: the pixel keeps its colour and variance bit for bit
            const float inv_l = 1.0f / (L.sigma_l * sqrtf(gv) + 1e-10f);
            float sw = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f, sv = 0.0f;
            #pragma unroll
            for (int j = 0; j < 5; ++j) {
                const int yy = y + (j - 2) * L.step;
                if (yy < 0 || yy >= L.h) continue;
                #pragma unroll
                for (int i = 0; i < 5; ++i) {
                    const int xx = x + (i - 2) * L.step;
                    if (xx < 0 || xx >= L.w) continue;
                    const size_t q = (size_t)yy * L.w + xx;
                    float wq = 1.0f;                           // the centre tap weighs exactly 1
                    if (q != p) {
                        const float2 yzq = __ldg(L.yz_in + q);
                        if (!finite_f(yzq.x)) continue;        // non-finite neighbour: weight 0
                        float e = fabsf(yzp.x - yzq.x) * inv_l;
                        if (L.use_depth) e += fabsf(yzp.y - yzq.y) / (L.sigma_z * fmaxf(fabsf(yzp.y), fabsf(yzq.y)) + 1e-6f);
                        wq = __expf(-e);
                    }
                    const float hw = kB3[j] * kB3[i] * wq;
                    if (!(hw > 0.0f)) continue;                // underflowed (or NaN from a NaN depth): the tap drops out
                    const float4 cq = __ldg(L.cv_in + q);
                    sw += hw; sr += hw * cq.x; sg += hw * cq.y; sb += hw * cq.z; sv += hw * hw * cq.w;
                }
            }
            const float inv = 1.0f / sw;
            o = make_float4(sr * inv, sg * inv, sb * inv, sv * inv * inv);
            Yo = luma(o.x, o.y, o.z);
        }
    }
    if (L.out_f3) {
        float* d = L.out_f3 + 3 * p;
        d[0] = o.x; d[1] = o.y; d[2] = o.z;
        if (L.out_display) L.out_display[p] = tonemap_display(make_float3(o.x, o.y, o.z), L.exposure_scale).word;
    } else {
        L.cv_out[p] = o;
        L.yz_out[p] = make_float2(Yo, yzp.y);
    }
}

// One layer of count planes of H*W pixels with `channels` floats each -> count float4 scratch planes, unused lanes 0.
__global__ void __launch_bounds__(256)
k_denoise_layer_gather(const float* __restrict__ src, const int channels, const size_t n, float4* __restrict__ planes)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* s = src + i * channels;
    planes[i] = make_float4(__ldg(s), channels > 1 ? __ldg(s + 1) : 0.0f, channels > 2 ? __ldg(s + 2) : 0.0f, channels > 3 ? __ldg(s + 3) : 0.0f);
}

constexpr int kDnLayerGroup = 8;                  // planes per launch of k_denoise_layers_atrous, at most

struct DenoiseLayerLevel {
    int w, h, step, use_depth;
    float sigma_l, sigma_z;
    const float4* cv_in; const float2* yz_in;     // the beauty's guide planes of this level
    const float4* in; float4* out;                // G planes of w * h pixels each, `out` null at the last level
    float* dst[kDnLayerGroup];                    // last level: plane k's pixels go to dst[k] with channels[k] floats each
    int channels[kDnLayerGroup];
};

// x' = sum(h w x_q) / sum(h w) for every lane of G planes, with the beauty's weights and copies.  k_denoise_atrous accumulates with FFMA
// and finishes with s * (1 / sw); so does this kernel, explicitly, so a plane equal to the beauty's colour comes out equal to it bit for bit.
template <int G>
__global__ void __launch_bounds__(kDnBlockX * kDnBlockY)
k_denoise_layers_atrous(const DenoiseLayerLevel L)
{
    const int x = blockIdx.x * kDnBlockX + threadIdx.x, y = blockIdx.y * kDnBlockY + threadIdx.y;
    if (x >= L.w || y >= L.h) return;
    const size_t px = (size_t)L.w * L.h, p = (size_t)y * L.w + x;
    const float2 yzp = __ldg(L.yz_in + p);
    float4 o[G];
    float inv_l;
    if (atrous_filters(L.w, L.h, L.sigma_l, L.cv_in, x, y, yzp, inv_l)) {
        float sw = 0.0f;
        float4 s[G];
        #pragma unroll
        for (int k = 0; k < G; ++k) s[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        #pragma unroll
        for (int j = 0; j < 5; ++j) {
            const int yy = y + (j - 2) * L.step;
            if (yy < 0 || yy >= L.h) continue;
            #pragma unroll
            for (int i = 0; i < 5; ++i) {
                const int xx = x + (i - 2) * L.step;
                if (xx < 0 || xx >= L.w) continue;
                const size_t q = (size_t)yy * L.w + xx;
                float hw;
                if (!atrous_tap(L.use_depth, L.sigma_z, L.yz_in, p, yzp, inv_l, j, i, q, hw)) continue;
                sw += hw;
                #pragma unroll
                for (int k = 0; k < G; ++k) {
                    const float4 v = __ldg(L.in + k * px + q);
                    s[k].x = __fmaf_rn(hw, v.x, s[k].x); s[k].y = __fmaf_rn(hw, v.y, s[k].y);
                    s[k].z = __fmaf_rn(hw, v.z, s[k].z); s[k].w = __fmaf_rn(hw, v.w, s[k].w);
                }
            }
        }
        const float inv = 1.0f / sw;
        #pragma unroll
        for (int k = 0; k < G; ++k) o[k] = make_float4(s[k].x * inv, s[k].y * inv, s[k].z * inv, s[k].w * inv);
    } else {
        #pragma unroll
        for (int k = 0; k < G; ++k) o[k] = __ldg(L.in + k * px + p);    // copied with the beauty, bit for bit
    }
    #pragma unroll
    for (int k = 0; k < G; ++k) {
        if (L.out) {
            L.out[k * px + p] = o[k];
        } else {
            float* d = L.dst[k] + (size_t)L.channels[k] * p;
            d[0] = o[k].x;
            if (L.channels[k] > 1) d[1] = o[k].y;
            if (L.channels[k] > 2) d[2] = o[k].z;
            if (L.channels[k] > 3) d[3] = o[k].w;
        }
    }
}

template <int G>
static cudaError_t launch_layers_level(const dim3 grid, const dim3 block, const DenoiseLayerLevel& L, cudaStream_t s)
{
    k_denoise_layers_atrous<G><<<grid, block, 0, s>>>(L);
    return cudaGetLastError();
}

cudaError_t launch_denoise(const DenoiseArgs& a, cudaStream_t s)
{
    const dim3 block(kDnBlockX, kDnBlockY);
    const dim3 grid((a.width + kDnBlockX - 1) / kDnBlockX, (a.height + kDnBlockY - 1) / kDnBlockY);
    const size_t px = (size_t)a.width * a.height;
    k_denoise_prep<<<grid, block, 0, s>>>(a.width, a.height, a.color, a.depth, a.rel_error, a.cv[0], a.yz[0]);
    cudaError_t e = cudaGetLastError();
    // every layer into the scratch planes before any level runs: the beauty's last level may write a layer's source (in place)
    size_t n_planes = 0;
    for (int l = 0; l < a.n_layers && e == cudaSuccess; ++l) {
        const size_t n = px * a.layers[l].count;
        k_denoise_layer_gather<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a.layers[l].src, a.layers[l].channels, n, a.lp[0] + n_planes * px);
        e = cudaGetLastError();
        n_planes += a.layers[l].count;
    }
    for (int i = 0; i < a.iterations && e == cudaSuccess; ++i) {
        const bool last = i + 1 == a.iterations;
        DenoiseLevel L;
        L.w = a.width; L.h = a.height; L.step = 1 << i; L.use_depth = a.depth != nullptr;
        L.sigma_l = a.sigma_l; L.sigma_z = a.sigma_z; L.exposure_scale = a.exposure_scale;
        L.cv_in = a.cv[i & 1]; L.yz_in = a.yz[i & 1];
        L.cv_out = last ? nullptr : a.cv[(i + 1) & 1]; L.yz_out = last ? nullptr : a.yz[(i + 1) & 1];
        L.out_f3 = last ? a.out_f3 : nullptr; L.out_display = last ? a.out_display : nullptr;
        k_denoise_atrous<<<grid, block, 0, s>>>(L);
        e = cudaGetLastError();
        // the layers of level i, guided by the plane pair the beauty just read; the largest group of 8, 4, 2 or 1 planes per launch
        int l = 0; unsigned k = 0;                                   // the layer and plane of scratch plane j, for the last level
        for (size_t j = 0; j < n_planes && e == cudaSuccess;) {
            const size_t left = n_planes - j;
            const int g = left >= 8 ? 8 : left >= 4 ? 4 : left >= 2 ? 2 : 1;
            DenoiseLayerLevel Q;
            Q.w = a.width; Q.h = a.height; Q.step = 1 << i; Q.use_depth = a.depth != nullptr;
            Q.sigma_l = a.sigma_l; Q.sigma_z = a.sigma_z;
            Q.cv_in = a.cv[i & 1]; Q.yz_in = a.yz[i & 1];
            Q.in = a.lp[i & 1] + j * px; Q.out = last ? nullptr : a.lp[(i + 1) & 1] + j * px;
            for (int m = 0; m < kDnLayerGroup; ++m) { Q.dst[m] = nullptr; Q.channels[m] = 0; }
            if (last) {
                for (int m = 0; m < g; ++m) {
                    while (k >= a.layers[l].count) { ++l; k = 0; }
                    Q.channels[m] = (int)a.layers[l].channels;
                    Q.dst[m] = a.layers[l].dst + (size_t)k * px * a.layers[l].channels;
                    ++k;
                }
            }
            e = g == 8 ? launch_layers_level<8>(grid, block, Q, s) : g == 4 ? launch_layers_level<4>(grid, block, Q, s)
              : g == 2 ? launch_layers_level<2>(grid, block, Q, s) : launch_layers_level<1>(grid, block, Q, s);
            j += g;
        }
    }
    return e;
}

} // namespace vpt
