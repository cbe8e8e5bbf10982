// vpt_atmosphere.cuh -- run-time lookup of the precomputed Bruneton sky (environment_type == 0).
//
// Reference: `sample_atmosphere` and the lookup half of the Bruneton model, source/render_kernel.cu:368-895
// (the precompute half lives in source/atmosphere/ and is SURVEY row N2, not part of the render pass).  Only
// k_resolve uses this: one sky evaluation per sample, at (env_pos, final ray direction).
//
// The model works ~6.4e6 m from the planet centre in fp32, so several discriminants cancel to a few ULPs of
// their operands; the reference gets its particular values from C++'s promotion rules (a `1.0` literal makes
// the surrounding sub-expression double, a float product stays float).  To land on the same numbers this file
// keeps, expression by expression, the same operand types and association -- that is the "algorithm" here.
// The four look-up textures and the scalars arrive in the reference's own AtmosphereParameters layout
// (vpt_atmosphere, include/vpt_abi.h).
#pragma once
#include "vpt_math.cuh"
#include "../../../include/vpt_abi.h"

namespace vpt {

// texture extents, source/atmosphere/constants.h:50-62
constexpr int kSkyTransW = 256, kSkyTransH = 64;
constexpr int kSkyScatR = 32, kSkyScatMu = 128, kSkyScatMuS = 32, kSkyScatNu = 8;
constexpr int kSkyIrrW = 256, kSkyIrrH = 64;

// kInPath selects the operation order of the reference's IN-PATH call sites (estimate_sky, render_kernel.cu:1382 / :1429) instead of
// its end-of-path ones (:1752 / :1840).  ptxas for sm_90a contracts the ill-conditioned sums as follows (read off the SASS of the
// reference kernel built for sm_90a with its own flags, nvdisasm -gi):
//     c*c - (pdp - pdv*pdv)          in path: FMUL, FADD            tail: FFMA(c, c, .)
//     (rmu*rmu - r*r) + Rt*Rt        sky_radiance, both sites: FMUL, FMUL, FADD, then FADD + FMUL(Rt*Rt)
//                                    radiance_to_point, both sites: FFMA(rmu, rmu, -r*r), then FADD + FMUL(Rt*Rt)
//     sc*ph_r + mie*ph_m             radiance_to_point, every site: FMUL(sc, ph_r), then FFMA(mie, ph_m, .)
// With r ~ 6.36e6 m a product rounded to fp32 is off by up to 2e6 m^2, so the forms give visibly different look-up coordinates.
template <bool kInPath>
struct Sky {
    const vpt_atmosphere& a;
    float Rg, Rt;                      // bottom / top radius

    VPT_DEV explicit Sky(const vpt_atmosphere& atm) : a(atm), Rg(atm.bottom_radius), Rt(atm.top_radius) {}

    static VPT_DEV float clampf_(float v, float lo, float hi) { return fmaxf(lo, fminf(v, hi)); }
    static VPT_DEV float clamp_cos(float mu) { return clampf_(mu, -1.0f, 1.0f); }
    static VPT_DEV float safe_sqrt(float v) { return sqrtf(fmaxf(v, 0.0f)); }
    static VPT_DEV float3 tex_rgb(float4 t) { return f3(t.x, t.y, t.z); }
    // [0,1] -> texel-centre range of an n-texel axis (:417-420)
    static VPT_DEV float to_texcoord(float x, int n) { return 0.5 / float(n) + x * (1.0 - 1.0 / float(n)); }
    static VPT_DEV float smooth01(float lo, float hi, float x) {
        const float y = clampf_((x - lo) / (hi - lo), 0.0f, 1.0f);
        return (y * y * (3.0f - (2.0f * y)));
    }

    VPT_DEV float clamp_radius(float r) const { return clampf_(r, Rg, Rt); }

    // distance along (r, mu) to the top boundary (:391-395)
    VPT_DEV float dist_to_top(float r, float mu) const {
        const float disc = r * r * (mu * mu - 1.0) + Rt * Rt;
        return fmaxf(-r * mu + safe_sqrt(disc), 0.0f);
    }
    // does the ray (r, mu) reach the ground (:403-407)
    VPT_DEV bool hits_ground(float r, float mu) const {
        return mu < 0.0 && r * r * (mu * mu - 1.0) + Rg * Rg >= 0.0;
    }

    // ---- transmittance (:427-484) ----
    VPT_DEV float3 trans_to_top(float r, float mu) const {
        const float H = sqrtf(Rt * Rt - Rg * Rg);
        const float rho = safe_sqrt(r * r - Rg * Rg);
        const float d = dist_to_top(r, mu);
        const float d_min = Rt - r;
        const float d_max = rho + H;
        const float x_mu = (d - d_min) / (d_max - d_min);
        const float x_r = rho / H;
        return tex_rgb(tex2D<float4>((cudaTextureObject_t)a.transmittance_texture,
                                     to_texcoord(x_mu, kSkyTransW), to_texcoord(x_r, kSkyTransH)));
    }
    VPT_DEV float3 trans_between(float r, float mu, float d, bool ground) const {
        const float r_d = clamp_radius(sqrt(d * d + 2.0 * r * mu * d + r * r));
        const float mu_d = clamp_cos((r * mu + d) / r_d);
        float3 q;
        if (ground) q = trans_to_top(r_d, -mu_d) / trans_to_top(r, -mu);
        else        q = trans_to_top(r, mu) / trans_to_top(r_d, mu_d);
        return f3(fminf(q.x, 1.0f), fminf(q.y, 1.0f), fminf(q.z, 1.0f));
    }
    VPT_DEV float3 trans_to_sun(float r, float mu_s) const {
        const float sin_h = Rg / r;
        const float cos_h = -sqrtf(fmax(1.0 - sin_h * sin_h, 0.0));
        return trans_to_top(r, mu_s) * smooth01(-sin_h * a.sun_angular_radius, sin_h * a.sun_angular_radius, mu_s - cos_h);
    }

    // ---- phase functions (:496-506) ----
    static VPT_DEV float rayleigh_phase(float nu) {
        const float k = 3.0 / (16.0 * VPT_PI_F);
        return k * (1.0 + nu * nu);
    }
    static VPT_DEV float mie_phase(float g, float nu) {
        const float k = 3.0 / (8.0 * VPT_PI_F) * (1.0 - g * g) / (2.0 + g * g);
        return k * (1.0 + nu * nu) / pow(1.0 + g * g - 2.0 * g * nu, 1.5);
    }

    // ---- 4-D scattering table, (r, mu, mu_s, nu) -> two 3-D fetches blended along nu (:508-556, :672-694) ----
    VPT_DEV float3 scattering(float r, float mu, float mu_s, float nu, bool ground, float3& single_mie) const {
        const float H = sqrt(Rt * Rt - Rg * Rg);
        const float rho = safe_sqrt(r * r - Rg * Rg);
        const float u_r = to_texcoord(rho / H, kSkyScatR);

        const float r_mu = r * mu;
        const float disc = r_mu * r_mu - r * r + Rg * Rg;
        float u_mu;
        if (ground) {
            const float d = -r_mu - safe_sqrt(disc);
            const float d_min = r - Rg;
            const float d_max = rho;
            u_mu = 0.5 - 0.5 * to_texcoord(d_max == d_min ? 0.0 : (d - d_min) / (d_max - d_min), kSkyScatMu / 2);
        } else {
            const float d = -r_mu + safe_sqrt(disc + H * H);
            const float d_min = Rt - r;
            const float d_max = rho + H;
            u_mu = 0.5 + 0.5 * to_texcoord((d - d_min) / (d_max - d_min), kSkyScatMu / 2);
        }

        const float d = dist_to_top(Rg, mu_s);
        const float d_min = Rt - Rg;
        const float d_max = H;
        const float aa = (d - d_min) / (d_max - d_min);
        const float A = -2.0 * a.mu_s_min * Rg / (d_max - d_min);
        const float u_mu_s = to_texcoord(fmax(1.0 - aa / A, 0.0) / (1.0 + aa), kSkyScatMuS);
        const float u_nu = (nu + 1.0) / 2.0;

        const float tcx = u_nu * float(kSkyScatNu - 1);
        const float tx = floorf(tcx);
        const float w = tcx - tx;
        const float x0 = (tx + u_mu_s) / float(kSkyScatNu);
        const float x1 = (tx + 1.0 + u_mu_s) / float(kSkyScatNu);

        const cudaTextureObject_t ts = (cudaTextureObject_t)a.scattering_texture;
        const cudaTextureObject_t tm = (cudaTextureObject_t)a.single_mie_scattering_texture;
        const float w0 = 1.0 - w;
        const float4 s0 = tex3D<float4>(ts, x0, u_mu, u_r), s1 = tex3D<float4>(ts, x1, u_mu, u_r);
        const float4 m0 = tex3D<float4>(tm, x0, u_mu, u_r), m1 = tex3D<float4>(tm, x1, u_mu, u_r);
        single_mie = f3(m0.x * w0 + m1.x * w, m0.y * w0 + m1.y * w, m0.z * w0 + m1.z * w);
        return f3(s0.x * w0 + s1.x * w, s0.y * w0 + s1.y * w, s0.z * w0 + s1.z * w);
    }

    // ---- ground irradiance (:636-654) ----
    VPT_DEV float3 irradiance(float r, float mu_s) const {
        const float x_r = (r - Rg) / (Rt - Rg);
        const float x_mu_s = mu_s * 0.5 + 0.5;
        return tex_rgb(tex2D<float4>((cudaTextureObject_t)a.irradiance_texture,
                                     to_texcoord(x_mu_s, kSkyIrrW), to_texcoord(x_r, kSkyIrrH)));
    }

    VPT_DEV float3 apply_luminance(float3 v, const vpt_f3& k) const {
        if (a.use_luminance != 0) v *= f3(k.x, k.y, k.z);
        return v;
    }

    // radiance of the sky seen from `cam` (planet-centred) along `view`, no light shafts (:696-749 with shadow_length 0)
    VPT_DEV float3 sky_radiance(float3 cam, float3 view, float3 sun, float3& transmittance) const {
        float r = length(cam);
        float rmu = dot(cam, view);
        const float s2 = psub(pmul(rmu, rmu), pmul(r, r));                              // rmu^2 - r^2
        const float to_top = psub(-rmu, sqrtf(padd(s2, pmul(Rt, Rt))));
        if (to_top > 0.0f) {                     // viewer in space: move to the boundary
            cam = cam + view * to_top;
            r = Rt;
            rmu += to_top;
        } else if (r > Rt) {                     // looking past the atmosphere
            transmittance = f3(1.0f);
            return f3(0.0f);
        }
        const float mu = rmu / r;
        const float mu_s = dot(cam, sun) / r;
        const float nu = dot(view, sun);
        const bool ground = hits_ground(r, mu);

        transmittance = ground ? f3(0.0f) : trans_to_top(r, mu);
        float3 mie;
        const float3 sc = scattering(r, mu, mu_s, nu, ground, mie);
        const float3 rad = sc * rayleigh_phase(nu) + mie * mie_phase(a.mie_phase_function_g, nu);
        return apply_luminance(rad, a.sky_spectral_radiance_to_luminance);
    }

    // in-scattered radiance between `cam` and the surface point `pt`, no light shafts (:751-812)
    VPT_DEV float3 radiance_to_point(float3 cam, float3 pt, float3 sun, float3& transmittance) const {
        const float3 view = normalize(pt - cam);
        float r = length(cam);
        float rmu = dot(cam, view);
        const float s2 = pfma(rmu, rmu, -pmul(r, r));                                   // rmu^2 - r^2 (the product fused here is the other one)
        const float to_top = psub(-rmu, sqrtf(padd(s2, pmul(Rt, Rt))));
        if (to_top > 0.0f) {
            cam = cam + view * to_top;
            r = Rt;
            rmu += to_top;
        }
        const float mu = rmu / r;
        const float mu_s = dot(cam, sun) / r;
        const float nu = dot(view, sun);
        float d = length(pt - cam);
        const bool ground = hits_ground(r, mu);

        transmittance = trans_between(r, mu, d, ground);

        float3 mie;
        float3 sc = scattering(r, mu, mu_s, nu, ground, mie);

        d = fmaxf(d - 0.0f, 0.0f);
        const float r_p = clamp_radius(sqrt(d * d + 2.0 * r * mu * d + r * r));
        const float mu_p = (r * mu + d) / r_p;
        const float mu_s_p = (r * mu_s + d * nu) / r_p;
        float3 mie_p;
        const float3 sc_p = scattering(r_p, mu_p, mu_s_p, nu, ground, mie_p);

        sc = sc - transmittance * sc_p;
        mie = mie - transmittance * mie_p;
        mie = mie * smooth01(0.0f, 0.01f, mu_s);      // sun-below-horizon fade

        // the reference rounds the Rayleigh product and fuses the Mie one, at all four call sites: fma(mie, ph_m, sc * ph_r)
        const float pr = rayleigh_phase(nu), pm = mie_phase(a.mie_phase_function_g, nu);
        const float3 rad = f3(pfma(mie.x, pm, pmul(sc.x, pr)), pfma(mie.y, pm, pmul(sc.y, pr)), pfma(mie.z, pm, pmul(sc.z, pr)));
        return apply_luminance(rad, a.sky_spectral_radiance_to_luminance);
    }

    // sun + sky irradiance on a surface point (:814-830)
    VPT_DEV float3 sun_and_sky_irradiance(float3 pt, float3 normal, float3 sun, float3& sky_irr) const {
        const float r = length(pt);
        const float mu_s = dot(pt, sun) / r;
        sky_irr = irradiance(r, mu_s) * (float)(1.0 + dot(normal, pt) / r) * 0.5f;
        const vpt_f3& si = a.solar_irradiance;
        float3 sun_irr = f3(si.x, si.y, si.z) * trans_to_sun(r, mu_s) * (float)fmax((double)dot(normal, sun), 0.0);
        if (a.use_luminance != 0) {
            sky_irr = apply_luminance(sky_irr, a.sky_spectral_radiance_to_luminance);
            sun_irr = apply_luminance(sun_irr, a.sun_spectral_radiance_to_luminance);
        }
        return sun_irr;
    }

    VPT_DEV float3 solar_radiance() const {
        const vpt_f3& si = a.solar_irradiance;
        const float3 s = f3(si.x, si.y, si.z) / (VPT_PI_F * a.sun_angular_radius * a.sun_angular_radius);   // M_PI is a float in the reference (helper_math.h:47)
        return apply_luminance(s, a.sun_spectral_radiance_to_luminance);
    }
};

// Environment radiance of the precomputed sky for a ray leaving the scene (:839-886).  The scene sits on the
// planet's surface: planet centre = (0, -bottom_radius, 0) in world units (metres).
template <bool kInPath = false>
VPT_DEV float3 sample_atmosphere(const vpt_atmosphere& atm, float azimuth, float elevation, float3 ray_pos, float3 ray_dir)
{
    const Sky<kInPath> sky(atm);
    const float3 centre = f3(.0f, -atm.bottom_radius, .0f);
    const float3 sun = sun_direction(azimuth, elevation);

    const float3 p = ray_pos - centre;
    const float p_dot_v = dot(p, ray_dir);
    const float p_dot_p = dot(p, p);
    const float q = psub(pmul(p_dot_v, p_dot_v), p_dot_p);                              // -(squared distance of the line from the centre)
    const float to_ground = psub(-p_dot_v, sqrtf(kInPath ? padd(pmul(centre.y, centre.y), q) : pfma(centre.y, centre.y, q)));

    float ground_alpha = 0.0f;
    float3 ground = f3(0.0f);
    if (to_ground > 0.0f) {
        const float3 pt = ray_pos + ray_dir * to_ground;
        const float3 n = normalize(pt - centre);
        float3 sky_irr;
        const float3 sun_irr = sky.sun_and_sky_irradiance(pt - centre, n, sun, sky_irr);
        const vpt_f3& ga = atm.ground_albedo;
        ground = f3(ga.x, ga.y, ga.z) * (float)(1.0 / VPT_PI_F) * (sun_irr + sky_irr);
        float3 t;
        const float3 in_scatter = sky.radiance_to_point(ray_pos - centre, pt - centre, sun, t);
        ground = ground * t + in_scatter;
        ground_alpha = 1.0f;
    }

    float3 t_sky;
    float3 rad = sky.sky_radiance(ray_pos - centre, ray_dir, sun, t_sky);
    if (dot(ray_dir, sun) > cosf(atm.sun_angular_radius)) rad = rad + t_sky * sky.solar_radiance();

    float3 out = lerp3(rad, ground, ground_alpha);
    const float3 expo = atm.use_luminance == 0 ? f3(atm.exposure) : f3(atm.exposure) * (float)1e-5;
    const vpt_f3& wp = atm.white_point;
    const float3 e = (f3(0.f) - out) / f3(wp.x, wp.y, wp.z) * expo;
    const float gam = (float)(1.0 / 2.2);
    return f3(powf(1.0f - expf(e.x), gam), powf(1.0f - expf(e.y), gam), powf(1.0f - expf(e.z), gam));
}

} // namespace vpt
