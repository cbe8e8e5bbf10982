// vpt_tonemap.cuh -- the display tail of the reference kernel, shared by k_resolve (vpt_kernels.cu), level (A) (vpt_level_a.cu, both
// through vpt_frame.cuh) and the denoiser (vpt_denoise.cu), so a display word means the same thing whoever wrote it.  Self-contained
// (plain component arithmetic, no vpt_math.cuh) because the denoiser's object must not define vpt_math.cuh's out-of-line functions a
// second time in the library.
#pragma once
#include <cuda_runtime.h>

namespace vpt {

__device__ __forceinline__ float3 aces_fit(float3 v) {        // reference rtt_and_odt_fit, :2208-2213
    const float3 a = make_float3(v.x * (v.x + 0.0245786f) - 0.000090537f, v.y * (v.y + 0.0245786f) - 0.000090537f,
                                 v.z * (v.z + 0.0245786f) - 0.000090537f);
    const float3 b = make_float3(v.x * (0.983729f * v.x + 0.4329510f) + 0.238081f, v.y * (0.983729f * v.y + 0.4329510f) + 0.238081f,
                                 v.z * (0.983729f * v.z + 0.4329510f) + 0.238081f);
    return make_float3(a.x / b.x, a.y / b.y, a.z / b.z);
}

__device__ __forceinline__ float3 mat3_mul(const float m[9], float3 v) {
    return make_float3(m[0] * v.x + m[1] * v.y + m[2] * v.z, m[3] * v.x + m[4] * v.y + m[5] * v.z, m[6] * v.x + m[7] * v.y + m[8] * v.z);
}

// The reference's display tail (render_kernel.cu:2300-2312): ACES fit of the running mean, exposure, gamma 2.2 and the BGRA pack.
// `val` is the tonemapped colour the raw buffer keeps, `word` the display word.
struct Tonemapped { float3 val; unsigned int word; };
__device__ __forceinline__ Tonemapped tonemap_display(const float3 accum, const float exposure_scale) {
    const float aces_in[9]  = { 0.59719f, 0.35458f, 0.04823f, 0.07600f, 0.90834f, 0.01566f, 0.02840f, 0.13383f, 0.83777f };
    const float aces_out[9] = { 1.60475f, -0.53108f, -0.07367f, -0.10208f, 1.10813f, -0.00605f, -0.00327f, -0.07276f, 1.07602f };
    const float3 m = mat3_mul(aces_out, aces_fit(mat3_mul(aces_in, accum)));
    Tonemapped t;
    t.val = make_float3(m.x * exposure_scale, m.y * exposure_scale, m.z * exposure_scale);
    const unsigned int r = (unsigned int)(255.0f * fminf(powf(fmaxf(t.val.x, 0.0f), (float)(1.0 / 2.2)), 1.0f));
    const unsigned int gg = (unsigned int)(255.0f * fminf(powf(fmaxf(t.val.y, 0.0f), (float)(1.0 / 2.2)), 1.0f));
    const unsigned int b = (unsigned int)(255.0f * fminf(powf(fmaxf(t.val.z, 0.0f), (float)(1.0 / 2.2)), 1.0f));
    t.word = 0xff000000 | (r << 16) | (gg << 8) | b;
    return t;
}

} // namespace vpt
