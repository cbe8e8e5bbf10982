// vpt_frame.cuh -- device helpers shared by the wavefront kernels (vpt_kernels.cu) and the level (A) entry (vpt_level_a.cu):
// the per-volume record arithmetic, the per-CTA staged scene, small frame utilities, and -- at the end -- the trace machinery
// (vpt_trace.cuh: PathState, walk_step, advance, ...).
#pragma once
#include <type_traits>
#include <cstring>
#include "vpt_walk.cuh"
#include "vpt_atmosphere.cuh"
#include "vpt_kernels.h"
#include "vpt_tonemap.cuh"

namespace vpt {

constexpr uint32_t kMissSentinel = 0xffffffffu;   // planeA.w bit pattern marking a miss sample (a NaN no arithmetic produces)

__device__ __forceinline__ const vpt_octnode* oct_ptr(vpt_devptr_t p) { return reinterpret_cast<const vpt_octnode*>(p); }

// one pass's advance of a blue-noise entry (reference :2320-2325): += golden ratio, mod 1, on all three channels
VPT_DEV void bn_step(float3& v)
{
    v.x += (1.0f + sqrtf(5.0f)) / 2.0f; v.y += (1.0f + sqrtf(5.0f)) / 2.0f; v.z += (1.0f + sqrtf(5.0f)) / 2.0f;
    v.x = fmodf(v.x, 1.0f); v.y = fmodf(v.y, 1.0f); v.z = fmodf(v.z, 1.0f);
}

// per-volume world->index affine, evaluated with the reference's own adjugate formula order
__device__ VolumeRec make_volume_rec(const vpt_gpu_vdb& g)
{
    // n_rc of the transposed matrix == xform[r-1][c-1] in memory order
    const float n11 = g.xform[0][0], n12 = g.xform[0][1], n13 = g.xform[0][2], n14 = g.xform[0][3];
    const float n21 = g.xform[1][0], n22 = g.xform[1][1], n23 = g.xform[1][2], n24 = g.xform[1][3];
    const float n31 = g.xform[2][0], n32 = g.xform[2][1], n33 = g.xform[2][2], n34 = g.xform[2][3];
    const float n41 = g.xform[3][0], n42 = g.xform[3][1], n43 = g.xform[3][2], n44 = g.xform[3][3];

    const float t11 = n23 * n34 * n42 - n24 * n33 * n42 + n24 * n32 * n43 - n22 * n34 * n43 - n23 * n32 * n44 + n22 * n33 * n44;
    const float t12 = n14 * n33 * n42 - n13 * n34 * n42 - n14 * n32 * n43 + n12 * n34 * n43 + n13 * n32 * n44 - n12 * n33 * n44;
    const float t13 = n13 * n24 * n42 - n14 * n23 * n42 + n14 * n22 * n43 - n12 * n24 * n43 - n13 * n22 * n44 + n12 * n23 * n44;
    const float t14 = n14 * n23 * n32 - n13 * n24 * n32 - n14 * n22 * n33 + n12 * n24 * n33 + n13 * n22 * n34 - n12 * n23 * n34;

    const float det = n11 * t11 + n21 * t12 + n31 * t13 + n41 * t14;
    const float idet = 1.0f / det;

    // second and third output rows of the inverse (unscaled adjugate entries)
    const float a01 = n24 * n33 * n41 - n23 * n34 * n41 - n24 * n31 * n43 + n21 * n34 * n43 + n23 * n31 * n44 - n21 * n33 * n44;
    const float a11 = n13 * n34 * n41 - n14 * n33 * n41 + n14 * n31 * n43 - n11 * n34 * n43 - n13 * n31 * n44 + n11 * n33 * n44;
    const float a21 = n14 * n23 * n41 - n13 * n24 * n41 - n14 * n21 * n43 + n11 * n24 * n43 + n13 * n21 * n44 - n11 * n23 * n44;
    const float a31 = n13 * n24 * n31 - n14 * n23 * n31 + n14 * n21 * n33 - n11 * n24 * n33 - n13 * n21 * n34 + n11 * n23 * n34;

    const float a02 = n22 * n34 * n41 - n24 * n32 * n41 + n24 * n31 * n42 - n21 * n34 * n42 - n22 * n31 * n44 + n21 * n32 * n44;
    const float a12 = n14 * n32 * n41 - n12 * n34 * n41 - n14 * n31 * n42 + n11 * n34 * n42 + n12 * n31 * n44 - n11 * n32 * n44;
    const float a22 = n12 * n24 * n41 - n14 * n22 * n41 + n14 * n21 * n42 - n11 * n24 * n42 - n12 * n21 * n44 + n11 * n22 * n44;
    const float a32 = n14 * n22 * n31 - n12 * n24 * n31 - n14 * n21 * n32 + n11 * n24 * n32 + n12 * n21 * n34 - n11 * n22 * n34;

    VolumeRec r;
    r.m[0][0] = t11 * idet; r.m[0][1] = t12 * idet; r.m[0][2] = t13 * idet; r.adj3[0] = t14;
    r.m[1][0] = a01 * idet; r.m[1][1] = a11 * idet; r.m[1][2] = a21 * idet; r.adj3[1] = a31;
    r.m[2][0] = a02 * idet; r.m[2][1] = a12 * idet; r.m[2][2] = a22 * idet; r.adj3[2] = a32;
    r.idet = idet;
    r.bmin[0] = g.vdb_info.bmin.x; r.bmin[1] = g.vdb_info.bmin.y; r.bmin[2] = g.vdb_info.bmin.z;
    r.rdim[0] = 1.0f / float(g.vdb_info.dim.x); r.rdim[1] = 1.0f / float(g.vdb_info.dim.y); r.rdim[2] = 1.0f / float(g.vdb_info.dim.z);
    r.flags = (g.vdb_info.has_color ? 1u : 0u) | (g.vdb_info.has_emission ? 2u : 0u);
    r.density_tex = g.vdb_info.density_texture; r.emission_tex = g.vdb_info.emission_texture; r.color_tex = g.vdb_info.color_texture;
    return r;
}

// =====================================================================================================
// shared helpers of the per-frame kernels
// =====================================================================================================
struct FrameShared {
    SceneTables sc;
    OctShared   oct;
    VolumeRec   vol0;      // volume 0 staged for single-volume scenes (the headline case)
};

// ea: also stage the render call's empty-ahead table (sc_dev is then the context's SceneAlloc); null for the kernels that do not read it
VPT_DEV void load_frame_shared(FrameShared& fs, const SceneTables* sc_dev, EmptyAhead* ea = nullptr) {
    if (threadIdx.x == 0 && threadIdx.y == 0) fs.sc = *sc_dev;
    __syncthreads();
    // stage_octree assumes a 1-D thread index
    const int t = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    const uint4* src = reinterpret_cast<const uint4*>(fs.sc.internal);
    uint4* d = reinterpret_cast<uint4*>(fs.oct.node);
    for (int i = t; i < kOctInternalNodes * 3; i += nt) d[i] = __ldg(src + i);
    {   // 96-byte record of volume 0
        const uint4* vs = reinterpret_cast<const uint4*>(fs.sc.volumes);
        uint4* vd = reinterpret_cast<uint4*>(&fs.vol0);
        for (int i = t; i < (int)(sizeof(VolumeRec) / 16); i += nt) vd[i] = __ldg(vs + i);
    }
    if (ea) {
        const uint4* es = reinterpret_cast<const uint4*>(&reinterpret_cast<const SceneAlloc*>(sc_dev)->ahead);
        uint4* ed = reinterpret_cast<uint4*>(ea);
        for (int i = t; i < (int)(sizeof(EmptyAhead) / 16); i += nt) ed[i] = __ldg(es + i);
    }
    __syncthreads();
}

VPT_DEV SphereRec load_sphere(const vpt_sphere* s) {
    SphereRec r;
    r.center = f3(s->center.x, s->center.y, s->center.z); r.radius = s->radius;
    r.color = f3(s->color.x, s->color.y, s->color.z); r.roughness = s->roughness;
    return r;
}

VPT_DEV float3 ld3(const vpt_f3& v) { return f3(v.x, v.y, v.z); }

// b0 = lower_left_corner + u * horizontal + v * vertical - origin of pixel (x, y) at jitter (jx, jy) (reference camera::get_ray,
// camera.h:131-136, with the lens offset left out): the pinhole ray's direction before normalize, and the thin-lens ray's before the
// offset.  The operation order is pinned: k_generate, k_miss_cull and k_resolve (which rebuilds the miss samples of culled pixels) must
// get the same bits.  Every operation is monotone in the jitter, so over the closed jitter square each component lies between its values
// at the four corner jitters (k_miss_cull).
VPT_DEV float3 camera_b0(const vpt_camera& cam, const vpt_u2 res, const int x, const int y, const float jx, const float jy)
{
    const float u = __fdividef(padd((float)x, jx), (float)res.x);
    const float v = __fdividef(padd((float)y, jy), (float)res.y);
    return f3(psub(pfma(cam.vertical.x, v, pfma(cam.horizontal.x, u, cam.lower_left_corner.x)), cam.origin.x),
              psub(pfma(cam.vertical.y, v, pfma(cam.horizontal.y, u, cam.lower_left_corner.y)), cam.origin.y),
              psub(pfma(cam.vertical.z, v, pfma(cam.horizontal.z, u, cam.lower_left_corner.z)), cam.origin.z));
}

// The equirectangular projection's angles of pixel (x, y) at jitter (jx, jy): phi = (s - 1/2) hfov, theta = (t - 1/2) vfov with
// s = (x + jx) / W, t = (y + jy) / H.  Every operation is monotone in x + jx (phi) and y + jy (theta), so over a closed jitter range
// each angle lies between its values at the range's ends (k_miss_cull_equirect); |phi| <= hfov / 2 <= pi keeps __sinf / __cosf in
// their accurate range.
VPT_DEV float2 pano_angles(const Projection& pj, const vpt_u2 res, const int x, const int y, const float jx, const float jy)
{
    const float s = __fdividef(padd((float)x, jx), (float)res.x);
    const float t = __fdividef(padd((float)y, jy), (float)res.y);
    return make_float2(pmul(psub(s, 0.5f), pj.hfov), pmul(psub(t, 0.5f), pj.vfov));
}

// b0 = cos theta (sin phi u - cos phi w) + sin theta v of the equirectangular projection (forward -w, right u, up v of the caller's
// camera; row 0 at the bottom, as the reference's `vertical`): the ray's direction before normalize, from the camera origin.  The
// operation order is pinned: k_generate_equirect, k_miss_cull_equirect, k_resolve_equirect (which rebuilds the miss samples of culled
// pixels) and vpt_debug_camera_rays must get the same bits.
VPT_DEV float3 pano_b0(const vpt_camera& cam, const Projection& pj, const vpt_u2 res, const int x, const int y, const float jx, const float jy)
{
    const float2 a = pano_angles(pj, res, x, y, jx, jy);
    const float sp = __sinf(a.x), cp = __cosf(a.x), st = __sinf(a.y), ct = __cosf(a.y);
    const float hx = pfma(sp, cam.u.x, -pmul(cp, cam.w.x)), hy = pfma(sp, cam.u.y, -pmul(cp, cam.w.y)), hz = pfma(sp, cam.u.z, -pmul(cp, cam.w.z));
    return f3(pfma(st, cam.v.x, pmul(ct, hx)), pfma(st, cam.v.y, pmul(ct, hy)), pfma(st, cam.v.z, pmul(ct, hz)));
}

// The camera of a sample whose shutter draw is xi in (0, 1] under camera motion `mo` (the pose at shutter close; `cam` is the pose at shutter
// open): every component of origin, lower_left_corner, horizontal, vertical, u and v is c == o ? o : fma(xi, c - o, o), with o the open and c
// the close pose's value.  A component that does not move keeps the open pose's bits (-0 included), so close == open is the static camera
// and a pure translation keeps the basis; xi = 1 reaches c only up to the rounding of c - o.  lens_radius, focus_dist and viz_dof stay the
// open camera's.  The operation order is pinned: k_generate_motion (and its adaptive / region forms) and vpt_debug_motion_cameras must get
// the same bits.
VPT_DEV float motion_lerp(const float o, const float c, const float xi) { return c == o ? o : pfma(xi, psub(c, o), o); }
VPT_DEV vpt_f3 motion_lerp3(const vpt_f3 o, const vpt_f3 c, const float xi)
{
    vpt_f3 r; r.x = motion_lerp(o.x, c.x, xi); r.y = motion_lerp(o.y, c.y, xi); r.z = motion_lerp(o.z, c.z, xi);
    return r;
}
VPT_DEV vpt_camera motion_camera(const vpt_camera& cam, const CameraMotion& mo, const float xi)
{
    vpt_camera m = cam;
    m.origin = motion_lerp3(cam.origin, mo.origin, xi);
    m.lower_left_corner = motion_lerp3(cam.lower_left_corner, mo.lower_left_corner, xi);
    m.horizontal = motion_lerp3(cam.horizontal, mo.horizontal, xi);
    m.vertical = motion_lerp3(cam.vertical, mo.vertical, xi);
    m.u = motion_lerp3(cam.u, mo.u, xi);
    m.v = motion_lerp3(cam.v, mo.v, xi);
    return m;
}

// The camera of pixel (x, y)'s sample at jitter (jx, jy) under the omni-directional stereo projection `od` (vpt_set_projection_ods):
//   eye e (-1 left, +1 right), row y_e within the eye and the eye's height H_e from the layout (over-under: rows [H/2, H) are the left eye);
//   (phi, theta) = pano_angles and b0 = pano_b0 at resolution (W, H_e), row y_e;
//   k = 1 for |theta| <= merge_from, 0 for |theta| >= merge_to, (merge_to - |theta|) * inv_span in between (the pole merge);
//   s = (e * ipd/2) * k, r = cos phi u + sin phi w (the viewer's right at azimuth phi; the __sinf / __cosf values pano_b0 takes);
//   origin' = fma(s, r, origin), lower_left_corner' = origin' + b0, horizontal = vertical = 0, everything else the caller's camera.
// generate_body traces that camera under the perspective rule, so every sample is the reference's camera::get_ray of it.  The operation
// order is pinned: k_generate_ods (and its adaptive / region forms) and k_ods_cameras must get the same bits.
struct OdsCamera { vpt_camera cam; float e, k; };
VPT_DEV OdsCamera ods_camera(const vpt_camera& cam, const OdsParams& od, const vpt_u2 res, const int x, const int y, const float jx, const float jy)
{
    vpt_u2 re = res;
    int ye = y;
    float e = od.layout == kOdsRight ? 1.0f : -1.0f;
    if (od.layout == kOdsOverUnder) {
        re.y = res.y >> 1;
        if (y >= (int)re.y) ye = y - (int)re.y;
        else e = 1.0f;
    }
    Projection pj; pj.kind = kProjOds; pj.hfov = od.hfov; pj.vfov = od.vfov;
    const float2 a = pano_angles(pj, re, x, ye, jx, jy);
    const float3 b0 = pano_b0(cam, pj, re, x, ye, jx, jy);
    const float at = fabsf(a.y);
    const float k = at <= od.merge_from ? 1.0f : at >= od.merge_to ? 0.0f : pmul(psub(od.merge_to, at), od.inv_span);
    const float s = pmul(e < 0.0f ? -od.half_ipd : od.half_ipd, k);
    const float sp = __sinf(a.x), cp = __cosf(a.x);
    OdsCamera o;
    o.cam = cam; o.e = e; o.k = k;
    o.cam.origin.x = pfma(s, pfma(cp, cam.u.x, pmul(sp, cam.w.x)), cam.origin.x);
    o.cam.origin.y = pfma(s, pfma(cp, cam.u.y, pmul(sp, cam.w.y)), cam.origin.y);
    o.cam.origin.z = pfma(s, pfma(cp, cam.u.z, pmul(sp, cam.w.z)), cam.origin.z);
    o.cam.lower_left_corner.x = padd(o.cam.origin.x, b0.x);
    o.cam.lower_left_corner.y = padd(o.cam.origin.y, b0.y);
    o.cam.lower_left_corner.z = padd(o.cam.origin.z, b0.z);
    o.cam.horizontal.x = o.cam.horizontal.y = o.cam.horizontal.z = 0.0f;
    o.cam.vertical.x = o.cam.vertical.y = o.cam.vertical.z = 0.0f;
    return o;
}

// the pinhole camera: what k_generate and k_miss_cull test before taking the pinhole branch (an origin component of exactly 0 could meet a
// signed zero of the lens offset, so those cameras take the literal order)
VPT_DEV bool pinhole_camera(const vpt_camera& cam)
{
    return (cam.lens_radius == 0.0f) && cam.origin.x != 0.0f && cam.origin.y != 0.0f && cam.origin.z != 0.0f;
}

// the pinhole ray of pixel (x, y) at jitter (jx, jy), as k_generate builds it
VPT_DEV float3 pinhole_dir(const vpt_camera& cam, const vpt_u2 res, const int x, const int y, const float jx, const float jy)
{
    return normalize(camera_b0(cam, res, x, y, jx, jy));
}

// global row of a local row under the interleaved-stripe partition (identity for one rank)
VPT_DEV int global_row(const FrameGeom& g, int lr) {
    const int s = (g.stripe_h & (g.stripe_h - 1)) == 0 ? (lr >> (__ffs(g.stripe_h) - 1)) : lr / g.stripe_h;   // power-of-two stripes: no division
    return (s * g.n_ranks + g.rank) * g.stripe_h + (lr - s * g.stripe_h);
}

// The pixel word a ray carries (queue record, parked record).  One rank: the pixel index itself.  Several ranks: (local row << 16) | x --
// the Philox stream is keyed by the GLOBAL pixel every time a ray is un-parked and the sample is written at the LOCAL pixel, and from
// this form both are a shift / multiply-add away (a runtime division on the un-park path cost 5 % of the trace kernel).
VPT_DEV uint32_t ray_pixel_word(const FrameGeom& g, int lr, int x) {
    return g.n_ranks > 1 ? ((uint32_t)lr << 16) | (uint32_t)x : (uint32_t)lr * (uint32_t)g.width + (uint32_t)x;
}
VPT_DEV uint32_t ray_global_pixel(const FrameGeom& g, uint32_t w) {
    if (g.n_ranks <= 1) return w;
    return (uint32_t)global_row(g, (int)(w >> 16)) * (uint32_t)g.width + (w & 0xffffu);
}
VPT_DEV uint32_t ray_local_pixel(const FrameGeom& g, uint32_t w) {
    if (g.n_ranks <= 1) return w;
    return (w >> 16) * (uint32_t)g.width + (w & 0xffffu);
}

// radical inverse of n in `BASE` (reference vanDerCorput, gpu_vdb/camera.h:49-62)
template <int BASE>
VPT_DEV float radical_inverse(int n) {
    float rand_int = 0, denom = 1, invBase = 1.f / BASE;
    while (n) {
        denom *= BASE;
        rand_int = padd(rand_int, __fdividef((float)(n % BASE), denom));
        n *= invBase;
    }
    return rand_int;
}

// the lens sampler only ever asks for the radical inverse of int(xi * 100)
template <int BASE>
VPT_DEV float van_der_corput(Rng& rng) { return radical_inverse<BASE>(int(rng.next() * 100)); }

// The HDRI environment term (reference :1838-1850), in two halves so that the light groups can add it to two values of L (the beauty's
// L and 0) from one fetch: hdri_product = (env(dir) * sky_color) * beta, hdri_finish = L + product / (4 pi) as one fma.
VPT_DEV float3 hdri_product(const cudaTextureObject_t env, const float3 sky_color, const float3 dir, const float3 beta)
{
    const float4 e = tex2D<float4>(env,
        pfma(atan2f(dir.z, dir.x), (float)(0.5 / 3.14159265358979323846), 0.5f),
        pmul(acosf(fmaxf(fminf(dir.y, 1.0f), -1.0f)), (float)(1.0 / 3.14159265358979323846)));
    return f3(pmul(pmul(e.x, sky_color.x), beta.x), pmul(pmul(e.y, sky_color.y), beta.y), pmul(pmul(e.z, sky_color.z), beta.z));
}
VPT_DEV float3 hdri_finish(const float3 t, const float3 L)
{
    const float c = 1.0f / (4.0f * VPT_PI_F);                   // isotropic() returns the folded constant
    return f3(pfma(t.x, c, L.x), pfma(t.y, c, L.y), pfma(t.z, c, L.z));
}

// Radiance of a finished sample under the HDRI environment: L + env(dir) * sky_color * beta / (4 pi).  A lean k_trace finishes its rays
// with it, k_resolve<0> its misses (L = 0, beta = 1) and the hits of wide records.  nvcc contracts this expression per call site, so the
// order is pinned to the one the end-of-path site compiles to: u = fma(atan2, 1/(2 pi), 0.5), v = acos * 1/pi, L + ((env * sky) * beta) /
// (4 pi) as one fma.  Every caller then gives the same bits.
VPT_DEV float3 hdri_radiance(const cudaTextureObject_t env, const float3 sky_color, const float3 dir, const float3 L, const float3 beta)
{
    return hdri_finish(hdri_product(env, sky_color, dir, beta), L);
}

#include "vpt_texfilter.cuh"
#include "vpt_trace.cuh"
#ifndef VPT_LEVEL_A_MODULE          // the level (A) cubin exports exactly one entry: no wavefront kernels in it
#include "vpt_trace_brick.cuh"
#endif

} // namespace vpt
