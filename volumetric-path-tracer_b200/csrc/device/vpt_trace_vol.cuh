// vpt_trace_vol.cuh -- control flow of the volumetric path integrator (Kernel_params.integrator != 0) for k_trace<1>.
// (included from vpt_trace.cuh, inside `namespace vpt`, after PathState / walk helpers)
//
// Reference: vol_integrator render_kernel.cu:1712-1756, uniform_sample_one_light :1519-1554, estimate_sun :1478-1516,
// estimate_point_light :1445-1475, estimate_sky :1356-1443 (env-CDF sampling :167-269, pdf_li :1342-1354,
// sample_spherical :293-304), estimate_emission :1275-1339.
//
// Unlike the direct integrator this one keeps tracking from the scatter point, estimates ONE of three light classes at
// every scatter (x3), and always ends on the precomputed sky (k_resolve adds `beta * sample_atmosphere` for it, at
// env_pos when |beta| > 0.9999 and at the last path position otherwise -- the position is handed over in planeD).
// The same heavy operations as the direct integrator are used (tracking step, transmittance set-up); only the glue
// differs.  Draw order facts read off the compiled reference: the light estimate runs before the emission walk
// (operands of `beta * uniform_sample_one_light(..) + estimate_emission(..)`), and the by-value RNG copies handed to
// draw_sample_from_distribution / sample_spherical peek at the next two draws without consuming them (quirk Q3).
#pragma once

enum VolPhase : int {
    VP_START = 0, VP_ITER, VP_AFTER_DELTA, VP_LIGHT, VP_AFTER_TR, VP_POINT_NEXT, VP_SKY_BSDF, VP_LIGHT_DONE, VP_AFTER_EMIT, VP_END
};
enum VolTrKind : int { VTR_SUN = 0, VTR_POINT = 1, VTR_SKY_LIGHT = 2, VTR_SKY_BSDF = 3 };

constexpr float kInv4Pi = 1.0f / (4.0f * VPT_PI_F);                             // isotropic(), :270-275 (float M_PI)

VPT_DEV float power_heuristic1(float f, float g) { return (f * f) / (f * f + g * g); }   // light.h:65-69 with nf = ng = 1

// equirect HDRI radiance along wi (reference sample_env_tex, :897-907)
VPT_DEV float3 env_tex_radiance(const vpt_kernel_params& kp, float3 wi) {
    const float4 t = tex2D<float4>((cudaTextureObject_t)kp.env_tex,
                                   atan2f(wi.z, wi.x) * (float)(0.5 / VPT_PI_F) + 0.5f,
                                   acosf(fmaxf(fminf(wi.y, 1.0f), -1.0f)) * (float)(1.0 / VPT_PI_F));
    return f3(t.x, t.y, t.z);
}

// one out-of-line copy of the sky model for the in-kernel uses (three call sites, ~2000 instructions each otherwise)
__device__ __noinline__ float3 sky_radiance_noinline(const vpt_atmosphere& atm, float az, float el, float3 pos, float3 wi) {
    return sample_atmosphere<true>(atm, az, el, pos, wi);        // the reference's in-path operation order (vpt_atmosphere.cuh)
}

// direction from the tabulated sky distribution (reference draw_sample_from_distribution, :167-246); `peek` is a COPY of the
// path's generator.  All five tables are point-sampled, unnormalised textures addressed exactly as the reference does.
VPT_DEV float env_cdf_sample(const vpt_kernel_params& kp, Rng peek, float3& wo) {
    const float xi = peek.next();
    const float zeta = peek.next();
    const cudaTextureObject_t mcdf = (cudaTextureObject_t)kp.env_marginal_cdf_tex, mfun = (cudaTextureObject_t)kp.env_marginal_func_tex;
    const cudaTextureObject_t ccdf = (cudaTextureObject_t)kp.env_cdf_tex, cfun = (cudaTextureObject_t)kp.env_func_tex;
    const int res = kp.env_sample_tex_res;

    int first = 0, len = res;
    while (len > 0) {                                              // upper bound of xi in the marginal cdf
        const int half = len >> 1, middle = first + half;
        if (tex1D<float>(mcdf, (float)middle) <= xi) { first = middle + 1; len -= half + 1; }
        else len = half;
    }
    const int v = max(0, min(first - 1, res - 2));
    float dv = xi - tex1D<float>(mcdf, (float)v);
    const float d_cdf_marginal = tex1D<float>(mcdf, (float)(v + 1)) - tex1D<float>(mcdf, (float)v);
    if (d_cdf_marginal > .0f) dv /= d_cdf_marginal;
    const float marginal_pdf = tex1D<float>(mfun, v + dv) / kp.env_marginal_int;
    const float theta = ((float(v) + dv) / float(res)) * VPT_PI_F;          // the reference's M_PI is the float of helper_math.h:47

    first = 0; len = res;
    while (len > 0) {                                              // upper bound of zeta in row v of the conditional cdf
        const int half = len >> 1, middle = first + half;
        if (tex2D<float>(ccdf, (float)middle, (float)v) <= zeta) { first = middle + 1; len -= half + 1; }
        else len = half;
    }
    const int u = max(0, min(first - 1, res - 2));
    float du = zeta - tex2D<float>(ccdf, (float)u, (float)v);
    const float d_cdf_conditional = tex2D<float>(ccdf, (float)(u + 1), (float)v) - tex2D<float>(ccdf, (float)u, (float)v);
    if (d_cdf_conditional > 0) du /= d_cdf_conditional;
    const float conditional_pdf = tex2D<float>(cfun, u + du, (float)v) / tex1D<float>(mfun, (float)v);
    const float xphi = (float(u) + du) / float(res);
    const float phi = pfma(xphi, VPT_PI_F, pmul(xphi, VPT_PI_F));             // (x * pi) * 2 as the reference build evaluates it: x*pi + x*pi, fused

    const float cos_theta = cosf(theta), sin_theta = sinf(theta);
    const float sin_phi = sinf(phi), cos_phi = cosf(phi);
    // normalize(): at this call site the reference build sums the squares in x, y, z order (SASS: FMUL x*x; FFMA y; FFMA z),
    // unlike the y-first order of its other dot products
    const float wx = pmul(sin_theta, cos_phi), wy = pmul(sin_theta, sin_phi);
    const float inv = rsqrtf(pfma(cos_theta, cos_theta, pfma(wy, wy, pmul(wx, wx))));
    wo = f3(pmul(wx, inv), pmul(wy, inv), pmul(cos_theta, inv));
    return (marginal_pdf * conditional_pdf) / (2 * VPT_PI_F * VPT_PI_F * sin_theta);
}

// density of direction wi under the tabulated distribution (reference pdf_li + draw_pdf_from_distribution, :1342-1354, :250-262)
VPT_DEV float env_cdf_pdf(const vpt_kernel_params& kp, float3 wi) {
    const float theta = acosf(fmaxf(-1.0f, fminf(wi.y, 1.0f)));
    const float phi = atan2f(wi.z, wi.x);
    const float sin_theta = sinf(theta);
    if (sin_theta == .0f) return .0f;
    const float s = 2.0f * VPT_PI_F * VPT_PI_F * sin_theta;
    const float px = (phi * 1.0f / (2.0f * VPT_PI_F)) / s;                    // INV_2_PI / INV_PI are unparenthesised float macros (:85-87)
    const float py = (theta * 1.0f / VPT_PI_F) / s;
    const int res = kp.env_sample_tex_res;
    const int iu = max(0, min(int(px * res), res - 1));
    const int iv = max(0, min(int(py * res), res - 1));
    const float conditional = tex2D<float>((cudaTextureObject_t)kp.env_func_tex, (float)iu, (float)iv);
    const float marginal = tex1D<float>((cudaTextureObject_t)kp.env_marginal_func_tex, (float)iv);
    return conditional / marginal;
}

// uniform direction on the sphere from a COPY of the generator (reference sample_spherical, :293-304; op order and fusion from its SASS)
VPT_DEV float3 peek_spherical(Rng peek) {
    const float phi = pmul(peek.next(), 2.0f * VPT_PI_F);
    const float u = peek.next();
    const float cos_theta = psub(1.0f, padd(u, u));
    const float sin_theta = sqrtf(pfma(-cos_theta, cos_theta, 1.0f));          // fused in the reference SASS
    return f3(pmul(sin_theta, cosf(phi)), pmul(sin_theta, sinf(phi)), cos_theta);
}

VPT_DEV float3 vol_env_radiance(const FrameArgs& fa, const vpt_atmosphere& atm, float3 pos, float3 wi) {
    return fa.kp.environment_type == 0 ? sky_radiance_noinline(atm, fa.kp.azimuth, fa.kp.elevation, pos, wi) : env_tex_radiance(fa.kp, wi);
}

// kGroups: every L += also goes to the ray's light-group sums in lg->planes.  The class of a light estimate is the last transmittance
// walk's tr_kind: uniform_sample_one_light leaves aux at 0 when it ran no walk, and then the group gains an exact zero.
// mt: the mattes, as advance's
template <bool kGroups = false, class... Mt>
VPT_DEV void advance_vol(PathState& st, const FrameShared& fs, const FrameArgs& fa, const vpt_atmosphere& atm, const TraceConsts& tc, const SphereRec& sph,
                         const LightGroups* lg = nullptr, const Mt*... mt)
{
    const SceneTables& sc = fs.sc;
    const vpt_kernel_params& kp = fa.kp;

    for (;;) {
        switch (st.phase) {
        case VP_START: {
            // depth pass (:1859-1889): walks only when the box is the closest object; the sphere alone sets the depth
            if (st.obj_c == 2) {
                st.depth = length(st.org - (st.pos + st.dir * st.tmin_c));
                if constexpr (sizeof...(Mt) > 0) matte_ids(mt...)->id[group_slot(st, fa)] = kMatteSphereId;
            }
            if (st.obj_c != 1) st.first_walk = false;
            float t, tmax;
            if (!aabb_intersect(sc.root_pmin, sc.root_pmax, st.pos, st.dir, t, tmax)) { st.op = OP_FINISH; return; }   // :1731
            st.pos = madd3(st.pos, st.dir, padd(t, VPT_EPS));
            st.rd = 1; st.phase = VP_ITER;
            break;
        }
        case VP_ITER:
            if (st.rd > kp.ray_depth) { st.phase = VP_END; break; }
            st.mi = false;
            st.wpos = st.pos; st.wdir = st.dir;
            if (!aabb_contains(sc.root_pmin, sc.root_pmax, st.pos)) {
                // `sample` returns at once (no draw, ray unchanged), and so does every remaining iteration
                if (st.first_walk) { st.depth = .0f; st.first_walk = false; }
                st.phase = VP_END;
                break;
            }
            st.sphere_free = line_misses_sphere(sph, st.pos, st.dir);
            st.t = 0.0f; st.distance = .0f; st.mode = W_DELTA; st.op = OP_STEP; st.phase = VP_AFTER_DELTA;
            return;
        case VP_AFTER_DELTA:
            st.pos = st.wpos;
            if (st.exit_reason == EX_SCATTER) { scatter_event(st, fs, fa, tc); st.mi = true; }
            if (st.first_walk) {                                    // this walk is also the depth pass's (same start, same draws)
                st.depth = st.mi ? length(st.org - st.pos) : .0f;
                if constexpr (sizeof...(Mt) > 0) {
                    if (st.mi) matte_ids(mt...)->id[group_slot(st, fa)] = collision_instance(sc, __float_as_int(st.aux.x), st.pos, last_draw(st.rng), tc.inv_max);
                }
                if (st.alpha < 1.0f) st.alpha += st.alpha;
                st.first_walk = false;
            }
            if (is_black(st.beta)) { st.phase = VP_END; break; }
            if (st.mi) { st.phase = VP_LIGHT; break; }
            st.rd++; st.phase = VP_ITER;
            break;
        case VP_LIGHT: {                                            // uniform_sample_one_light
            const float light_num = st.rng.next() * 3.0f;
            st.aux = f3(.0f);
            st.phase = VP_LIGHT_DONE;
            if (light_num < 1) {
                if (kp.sun_mult > .0f) {
                    st.tr_kind = VTR_SUN; st.wpos = st.pos; st.wdir = tc.sun_dir;
                    st.op = OP_TRBEGIN; st.phase = VP_AFTER_TR;
                    return;
                }
            } else if (light_num >= 1 && light_num < 2) {
                if (fa.lights.num_lights > 0) { st.light_budget = 10; st.phase = VP_POINT_NEXT; }
            } else if (kp.sky_mult > .0f) {                         // estimate_sky, light-sampling half
                (void)st.rng.next(); (void)st.rng.next();           // az, el: drawn, never used
                float3 wi; float light_pdf;
                if (kp.environment_type == 0) light_pdf = env_cdf_sample(kp, st.rng, wi);
                else { wi = peek_spherical(st.rng); light_pdf = kInv4Pi; }
                const float3 Li = vol_env_radiance(fa, atm, st.pos, wi);
                st.phase = VP_SKY_BSDF;
                if (light_pdf > .0f && !is_black(Li)) {
                    const float phase_pdf = hg_phase(dot(st.dir, wi), kp.phase_g1);
                    if (phase_pdf > .0f) {
                        st.tmin_c = light_pdf;                      // parked across the transmittance walk
                        st.tr_kind = VTR_SKY_LIGHT; st.wpos = st.pos; st.wdir = wi;
                        st.op = OP_TRBEGIN; st.phase = VP_AFTER_TR;
                        return;
                    }
                }
            }
            break;
        }
        case VP_AFTER_TR: {
            const float tr = finish_ratio_walk(st);
            if (st.tr_kind == VTR_SUN) {                            // estimate_sun
                const float phase_pdf = hg_phase(dot(st.dir, tc.sun_dir), kp.phase_g1);
                st.aux = f3(tr) * phase_pdf * ld3(kp.sun_color) * kp.sun_mult;
                st.phase = VP_LIGHT_DONE;
            } else if (st.tr_kind == VTR_POINT) {                   // point_light::Le, light.h:104-121
                if (st.light_budget < (int)fa.lights.num_lights) {
                    const vpt_point_light& pl = reinterpret_cast<const vpt_point_light*>(fa.lights.light_ptr)[st.light_index];
                    const float3 lpos = ld3(pl.pos);
                    const float3 wi = normalize(lpos - st.pos);
                    const float phase_pdf = hg_phase(dot(st.dir, wi), kp.phase_g1);
                    const float sqr_dist = length(lpos * lpos - st.pos * st.pos);
                    const float falloff = 1 / sqr_dist;
                    st.aux += ld3(pl.color) * pl.power * f3(tr) * phase_pdf * falloff;
                }
                st.light_budget--;
                st.phase = VP_POINT_NEXT;
            } else if (st.tr_kind == VTR_SKY_LIGHT) {
                const float3 wi = st.wdir;
                float3 Li = vol_env_radiance(fa, atm, st.pos, wi);
                Li *= f3(tr);
                if (!is_black(Li)) {
                    const float light_pdf = st.tmin_c;
                    const float phase_pdf = hg_phase(dot(st.dir, wi), kp.phase_g1);
                    const float weight = power_heuristic1(light_pdf, phase_pdf);
                    st.aux += Li * phase_pdf * weight / light_pdf;
                }
                st.phase = VP_SKY_BSDF;
            } else {                                                // phase-sampling half, after its transmittance walk
                const float3 Li = vol_env_radiance(fa, atm, st.pos, st.wdir);
                if (!is_black(Li)) st.aux += Li * f3(tr) * st.tmin_c;
                st.aux *= kp.sky_mult;
                st.phase = VP_LIGHT_DONE;
            }
            break;
        }
        case VP_POINT_NEXT: {                                       // estimate_point_light
            if (st.light_budget < 0) { st.phase = VP_LIGHT_DONE; break; }
            const vpt_point_light* lp = reinterpret_cast<const vpt_point_light*>(fa.lights.light_ptr);
            st.light_index = int(floorf(st.rng.next() * fa.lights.num_lights));
            st.tr_kind = VTR_POINT; st.wpos = st.pos; st.wdir = normalize(ld3(lp[st.light_index].pos) - st.pos);
            st.op = OP_TRBEGIN; st.phase = VP_AFTER_TR;
            return;
        }
        case VP_SKY_BSDF: {                                         // estimate_sky, phase-sampling half (:1409-1436)
            float3 wi = st.dir;
            const float cos_theta = hg_sample(wi, st.rng, kp.phase_g1);
            const float phase_pdf = hg_phase(-cos_theta, kp.phase_g1);
            st.phase = VP_LIGHT_DONE;
            if (phase_pdf > .0f) {
                const float light_pdf = kp.environment_type == 0 ? env_cdf_pdf(kp, wi) : kInv4Pi;
                if (light_pdf != 0.0f) {
                    st.tmin_c = power_heuristic1(phase_pdf, light_pdf);
                    st.tr_kind = VTR_SKY_BSDF; st.wpos = st.pos; st.wdir = wi;
                    st.op = OP_TRBEGIN; st.phase = VP_AFTER_TR;
                    return;
                }
            }
            st.aux *= kp.sky_mult;
            break;
        }
        case VP_LIGHT_DONE:                                         // L += beta * (3 * estimate) [+ emission], then resample the direction
            if constexpr (kGroups) {
                const float3 t = st.aux * 3.0f;
                st.L = pfma3(st.beta, t, st.L);
                const int group = st.tr_kind == VTR_SUN ? LG_SUN : st.tr_kind == VTR_POINT ? LG_POINT : LG_ENVIRONMENT;
                group_fma(lg, group_slot(st, fa), group, st.beta, t);
            } else st.L += st.beta * (st.aux * 3.0f);
            if (kp.emission_scale != 0) {
                st.wpos = st.pos; st.wdir = st.dir; st.t = 0.0f; st.aux = f3(.0f);
                st.mode = W_EMIT; st.op = OP_STEP; st.phase = VP_AFTER_EMIT;
                return;
            }
            hg_sample(st.dir, st.rng, kp.phase_g1);
            st.rd++; st.phase = VP_ITER;
            break;
        case VP_AFTER_EMIT:
            st.L += st.aux;
            if constexpr (kGroups) group_add(lg, group_slot(st, fa), LG_EMISSION, st.aux);
            hg_sample(st.dir, st.rng, kp.phase_g1);
            st.rd++; st.phase = VP_ITER;
            break;
        case VP_END:
        default:
            st.dir = normalize(st.dir);                             // :1747, only on paths that entered the box
            st.op = OP_FINISH;
            return;
        }
    }
}
