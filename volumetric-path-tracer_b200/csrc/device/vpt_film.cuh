// vpt_film.cuh -- the film projection of a perspective camera, shared by the motion vectors (vpt_kernels.cu, DESIGN.md section 8o) and
// the temporal filter (vpt_temporal.cu, section 8p).  Self-contained (the single-rounding intrinsics spelled out, no vpt_math.cuh) for the
// reason vpt_tonemap.cuh is: the temporal filter's object must not include the trace machinery.  The operations are those of vpt_math.cuh's
// dot, cross, pmul, psub and pfma, in the same order, so the motion-vector kernels compile to the code they had before the move.
#pragma once
#include <cuda_runtime.h>
#include "../../../include/vpt_abi.h"

namespace vpt {

__device__ __forceinline__ float film_dot(const float3 a, const float3 b) { return __fmaf_rn(a.z, b.z, __fmaf_rn(a.x, b.x, __fmul_rn(a.y, b.y))); }
__device__ __forceinline__ float3 film_cross(const float3 a, const float3 b) {
    return make_float3(__fmaf_rn(a.y, b.z, -__fmul_rn(a.z, b.y)), __fmaf_rn(a.z, b.x, -__fmul_rn(a.x, b.z)), __fmaf_rn(a.x, b.y, -__fmul_rn(a.y, b.x)));
}

// The film projection pi_K of camera K: d = P - origin, e = lower_left_corner - origin, n = cross(horizontal, vertical), k = e.n / d.n,
// q = k d - e, and (s, t) with q = s horizontal + t vertical (the 2x2 normal equations; the dot-product form when horizontal . vertical is 0),
// in the units of camera_b0's (x + jx) / W, (y + jy) / H: (s W, t H).  FilmCam holds what depends on K alone.
struct FilmCam { float3 o, e, h, v; float en, hh, hv, vv, det; };
__device__ __forceinline__ FilmCam film_cam(const vpt_f3 origin, const vpt_f3 llc, const vpt_f3 horizontal, const vpt_f3 vertical)
{
    FilmCam K;
    K.o = make_float3(origin.x, origin.y, origin.z); K.h = make_float3(horizontal.x, horizontal.y, horizontal.z);
    K.v = make_float3(vertical.x, vertical.y, vertical.z);
    K.e = make_float3(__fsub_rn(llc.x, origin.x), __fsub_rn(llc.y, origin.y), __fsub_rn(llc.z, origin.z));
    K.en = film_dot(K.e, film_cross(K.h, K.v));
    K.hh = film_dot(K.h, K.h); K.hv = film_dot(K.h, K.v); K.vv = film_dot(K.v, K.v);
    K.det = __fmaf_rn(K.hh, K.vv, -__fmul_rn(K.hv, K.hv));
    return K;
}
// The projection of the direction d (a point at infinity along d, or d = P - origin for the point P) into *st: pi_K with d in place of
// P - origin.  False when d does not point in front of K (k <= 0, NaN) or the result is not finite.
__device__ __forceinline__ bool film_project_dir(const FilmCam& K, const float3 d, const vpt_u2 res, float2* st)
{
    const float k = __fdiv_rn(K.en, film_dot(d, film_cross(K.h, K.v)));
    const float3 q = make_float3(__fmaf_rn(k, d.x, -K.e.x), __fmaf_rn(k, d.y, -K.e.y), __fmaf_rn(k, d.z, -K.e.z));
    const float qh = film_dot(q, K.h), qv = film_dot(q, K.v);
    float s, t;
    if (K.hv == 0.0f) { s = __fdiv_rn(qh, K.hh); t = __fdiv_rn(qv, K.vv); }
    else {
        s = __fdiv_rn(__fmaf_rn(K.vv, qh, -__fmul_rn(K.hv, qv)), K.det);
        t = __fdiv_rn(__fmaf_rn(K.hh, qv, -__fmul_rn(K.hv, qh)), K.det);
    }
    st->x = __fmul_rn(s, (float)res.x); st->y = __fmul_rn(t, (float)res.y);
    return k > 0.0f && isfinite(st->x) && isfinite(st->y);
}
// pi_K(P) into *st; false when P is not in front of K (k <= 0, NaN) or the result is not finite
__device__ __forceinline__ bool film_project(const FilmCam& K, const float3 P, const vpt_u2 res, float2* st)
{
    return film_project_dir(K, make_float3(__fsub_rn(P.x, K.o.x), __fsub_rn(P.y, K.o.y), __fsub_rn(P.z, K.o.z)), res, st);
}

} // namespace vpt
