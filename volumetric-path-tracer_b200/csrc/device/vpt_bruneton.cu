// vpt_bruneton.cu -- precomputation of the Bruneton sky tables (SURVEY 8(f) row N2): transmittance, direct / indirect ground
// irradiance, single scattering, scattering density, multiple scattering, four orders.
//
// Replaces the nine Driver-API kernels of source/atmosphere/atmosphere_kernels.cu:621-792 and the arithmetic they call
// (:67-618), driven as atmosphere::precompute does (source/atmosphere/atmosphere.cpp:888-1114).  The model is Bruneton & Neyret's
// published precomputed atmospheric scattering; what has to be matched is not the textbook model but THIS application's build
// of it, because the render path consumes its tables:
//   * tables live in linear float4 buffers during the precompute and are looked up by NEAREST texel (index = int(u * size)), not
//     filtered (:161-171, :359-376, :607-618);
//   * every order after the first reads the running `scattering` / `irradiance` tables where Bruneton reads the per-order deltas
//     (:383-386, :452), and the host passes a float4 where the kernels declare `int blend` (atmosphere.cpp:1056-1058 vs
//     atmosphere_kernels.cu:654,676: quirk Q17), so `blend` is the bit pattern of 0.0f = 0: orders 2..4 OVERWRITE the scattering
//     and irradiance tables instead of accumulating.  The final scattering table is the 4th order alone, the single-Mie table the
//     first order, the irradiance table the 4th order's indirect term;
//   * the scattering look-up indexes its buffers with UNCLAMPED texel coordinates (:375-395): a coordinate one below 0 or at the
//     table size addresses the neighbouring row / slice through the linear index, and this build does the same; the transmittance
//     look-up clamps its linear index to one texel past the end (:161-171).  Where such an index leaves the buffer the reference
//     reads whatever lies there; this build clamps the LINEAR index to the table.  Which texels read outside was measured
//     (tests/test_bruneton_stages_gpu.py, each reference stage run with the guards around its buffers holding 0 and then 3.0): in
//     multiple scattering, 2048 texels per order -- the first five mu rows (rays just below the horizon) of the 2nd-5th r layers
//     -- whose look-ups near r = Rg take a negative mu coordinate in the lowest r slice and read BEFORE the delta scattering-
//     density buffer; in single scattering, the transmittance reads one past that table's end (sun below the horizon).
// Arithmetic keeps the reference's operand types: its double literals promote the neighbouring float products (see
// vpt_atmosphere.cuh for why that matters 6.4e6 m from the planet centre), compiled with the same --use_fast_math.
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/vpt_abi.h"

namespace vpt {
namespace bru {

constexpr int kTW = 256, kTH = 64;                              // transmittance table
constexpr int kSR = 32, kSMu = 128, kSMuS = 32, kSNu = 8;       // scattering table: r, mu, mu_s, nu
constexpr int kSW = kSNu * kSMuS, kSH = kSMu, kSD = kSR;        // 256 x 128 x 32 texels
constexpr int kIW = 256, kIH = 64;                              // irradiance table
constexpr float kPi = 3.14159265358979323846f;

struct V3 { float x, y, z; };
__device__ inline V3 v3(float x, float y, float z) { V3 r = { x, y, z }; return r; }
__device__ inline V3 v3(float s) { return v3(s, s, s); }
__device__ inline V3 v3(vpt_f3 a) { return v3(a.x, a.y, a.z); }
__device__ inline V3 v3(float4 a) { return v3(a.x, a.y, a.z); }
__device__ inline V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ inline V3 operator*(V3 a, V3 b) { return v3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ inline V3 operator*(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
__device__ inline V3 operator/(V3 a, V3 b) { return v3(a.x / b.x, a.y / b.y, a.z / b.z); }
__device__ inline V3 operator/(V3 a, float s) { return v3(a.x / s, a.y / s, a.z / s); }
__device__ inline void operator+=(V3& a, V3 b) { a.x += b.x; a.y += b.y; a.z += b.z; }
__device__ inline float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ inline V3 min3(V3 a, V3 b) { return v3(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z)); }
__device__ inline V3 exp3(V3 a) { return v3(expf(a.x), expf(a.y), expf(a.z)); }
__device__ inline V3 neg3(V3 a) { return v3(-a.x, -a.y, -a.z); }
__device__ inline float4 f4(V3 a, float w) { return make_float4(a.x, a.y, a.z, w); }
__device__ inline float clampf(float v, float lo, float hi) { return fmaxf(lo, fminf(v, hi)); }
__device__ inline float smooth(float lo, float hi, float x) { const float y = clampf((x - lo) / (hi - lo), 0.0f, 1.0f); return (y * y * (3.0f - (2.0f * y))); }

struct Mat3 { float m[9]; };                                    // row-major: y_r = sum_c m[r*3+c] * x_c  (mat3::toMatrix + operator*, matrix_math.h:505-513, 686-692)
__device__ inline V3 mul(const Mat3& M, V3 v) {
    return v3(M.m[0] * v.x + M.m[1] * v.y + M.m[2] * v.z, M.m[3] * v.x + M.m[4] * v.y + M.m[5] * v.z, M.m[6] * v.x + M.m[7] * v.y + M.m[8] * v.z);
}

// the nine working tables, named as the reference's AtmosphereParameters members (definitions.h:82-90)
struct Tables {
    float4 *delta_irradiance, *delta_rayleigh, *delta_mie, *delta_density, *delta_multiple;
    float4 *transmittance, *irradiance, *scattering, *single_mie;
};

struct Model {
    const vpt_atmosphere& a;
    const Tables& t;
    float Rg, Rt;
    __device__ Model(const vpt_atmosphere& atm, const Tables& tb) : a(atm), t(tb), Rg(atm.bottom_radius), Rt(atm.top_radius) {}

    // ---- geometry (:67-99) ----
    static __device__ float clamp_cos(float mu) { return clampf(mu, float(-1.0), float(1.0)); }
    static __device__ float clamp_dist(float d) { return fmaxf(d, 0.0f); }
    __device__ float clamp_radius(float r) const { return clampf(r, Rg, Rt); }
    static __device__ float safe_sqrt(float v) { return sqrtf(fmaxf(v, 0.0f)); }
    __device__ float dist_to_top(float r, float mu) const { const float disc = r * r * (mu * mu - 1.0) + Rt * Rt; return clamp_dist(-r * mu + safe_sqrt(disc)); }
    __device__ float dist_to_bottom(float r, float mu) const { const float disc = r * r * (mu * mu - 1.0) + Rg * Rg; return clamp_dist(-r * mu - safe_sqrt(disc)); }
    __device__ bool hits_ground(float r, float mu) const { return mu < 0.0 && r * r * (mu * mu - 1.0) + Rg * Rg >= 0.0f; }
    __device__ float dist_to_nearest(float r, float mu, bool ground) const { return ground ? dist_to_bottom(r, mu) : dist_to_top(r, mu); }

    // ---- density profiles (:101-111) ----
    static __device__ float layer_density(const vpt_density_layer& l, float h) {
        const float d = l.exp_term * exp(l.exp_scale * h) + l.linear_term * h + l.const_term;
        return clampf(d, float(0.0), float(1.0));
    }
    static __device__ float profile_density(const vpt_density_profile& p, float h) { return h < p.layers[0].width ? layer_density(p.layers[0], h) : layer_density(p.layers[1], h); }

    // ---- transmittance (:113-197) ----
    __device__ float optical_length_to_top(const vpt_density_profile& p, float r, float mu) const {
        const int N = 500;
        const float dx = dist_to_top(r, mu) / float(N);
        float result = 0.0f;
        for (int i = 0; i <= N; ++i) {
            const float d_i = float(i) * dx;
            const float r_i = sqrt(d_i * d_i + 2.0 * r * mu * d_i + r * r);
            const float y_i = profile_density(p, r_i - Rg);
            const float w_i = i == 0 || i == N ? 0.5 : 1.0;
            result += y_i * w_i * dx;
        }
        return result;
    }
    __device__ V3 compute_transmittance_to_top(float r, float mu) const {
        return exp3(neg3(v3(a.rayleigh_scattering) * optical_length_to_top(a.rayleigh_density, r, mu) +
                         v3(a.mie_extinction) * optical_length_to_top(a.mie_density, r, mu) +
                         v3(a.absorption_extinction) * optical_length_to_top(a.absorption_density, r, mu)));
    }
    static __device__ float to_texcoord(float x, int n) { return 0.5 / float(n) + x * (1.0 - 1.0 / float(n)); }
    static __device__ float from_texcoord(float u, int n) { return (u - 0.5 / float(n)) / (1.0 - 1.0 / float(n)); }
    __device__ float2 transmittance_uv(float r, float mu) const {
        const float H = sqrtf(Rt * Rt - Rg * Rg);
        const float rho = safe_sqrt(r * r - Rg * Rg);
        const float d = dist_to_top(r, mu);
        const float d_min = Rt - r, d_max = rho + H;
        const float x_mu = (d - d_min) / (d_max - d_min);
        const float x_r = rho / H;
        return make_float2(to_texcoord(x_mu, kTW), to_texcoord(x_r, kTH));
    }
    __device__ void transmittance_r_mu(float2 uv, float& r, float& mu) const {
        const float x_mu = from_texcoord(uv.x, kTW), x_r = from_texcoord(uv.y, kTH);
        const float H = sqrt(Rt * Rt - Rg * Rg);
        const float rho = H * x_r;
        r = sqrt(rho * rho + Rg * Rg);
        const float d_min = Rt - r, d_max = rho + H;
        const float d = d_min + x_mu * (d_max - d_min);
        mu = d == 0.0f ? float(1.0) : (H * H - rho * rho - d * d) / (2.0 * r * d);
        mu = clamp_cos(mu);
    }
    // nearest-texel read of the transmittance table (:161-171; the reference clamps the LINEAR index to [0, W*H], one past the end)
    __device__ V3 transmittance_to_top(float r, float mu) const {
        const float2 uv = transmittance_uv(r, mu);
        const int x = int(floor(uv.x * kTW)), y = int(floor(uv.y * kTH));
        int idx = y * kTW + x;
        idx = min(max(idx, 0), kTW * kTH - 1);
        return v3(t.transmittance[idx]);
    }
    __device__ V3 transmittance(float r, float mu, float d, bool ground) const {
        const float r_d = clamp_radius(sqrt(d * d + 2.0 * r * mu * d + r * r));
        const float mu_d = clamp_cos((r * mu + d) / r_d);
        if (ground) return min3(transmittance_to_top(r_d, -mu_d) / transmittance_to_top(r, -mu), v3(1.0f));
        return min3(transmittance_to_top(r, mu) / transmittance_to_top(r_d, mu_d), v3(1.0f));
    }
    __device__ V3 transmittance_to_sun(float r, float mu_s) const {
        const float sin_h = Rg / r;
        const float cos_h = -sqrt(max(1.0 - sin_h * sin_h, 0.0));
        return transmittance_to_top(r, mu_s) * smooth(-sin_h * a.sun_angular_radius, sin_h * a.sun_angular_radius, mu_s - cos_h);
    }

    // ---- single scattering (:199-247) ----
    __device__ void single_scattering_integrand(float r, float mu, float mu_s, float nu, float d, bool ground, V3& ray, V3& mie) const {
        const float r_d = clamp_radius(sqrt(d * d + 2.0 * r * mu * d + r * r));
        const float mu_s_d = clamp_cos((r * mu_s + d * nu) / r_d);
        const V3 tr = transmittance(r, mu, d, ground) * transmittance_to_sun(r_d, mu_s_d);
        ray = tr * profile_density(a.rayleigh_density, r_d - Rg);
        mie = tr * profile_density(a.mie_density, r_d - Rg);
    }
    __device__ void single_scattering(float r, float mu, float mu_s, float nu, bool ground, V3& ray, V3& mie) const {
        const int N = 50;
        const float dx = dist_to_nearest(r, mu, ground) / float(N);
        V3 rs = v3(0.0f), ms = v3(0.0f);
        for (int i = 0; i <= N; ++i) {
            const float d_i = float(i) * dx;
            V3 ri, mi;
            single_scattering_integrand(r, mu, mu_s, nu, d_i, ground, ri, mi);
            const float w_i = (i == 0 || i == N) ? 0.5 : 1.0;
            rs += ri * w_i; ms += mi * w_i;
        }
        ray = rs * dx * v3(a.solar_irradiance) * v3(a.rayleigh_scattering);
        mie = ms * dx * v3(a.solar_irradiance) * v3(a.mie_scattering);
    }
    static __device__ float rayleigh_phase(float nu) { const float k = 3.0 / (16.0 * kPi); return k * (1.0 + nu * nu); }
    static __device__ float mie_phase(float g, float nu) { const float k = 3.0 / (8.0 * kPi) * (1.0 - g * g) / (2.0 + g * g); return k * (1.0 + nu * nu) / pow(1.0 + g * g - 2.0 * g * nu, 1.5); }

    // ---- 4-D scattering table parametrisation (:249-357) ----
    __device__ float4 scattering_uvwz(float r, float mu, float mu_s, float nu, bool ground) const {
        const float H = sqrt(Rt * Rt - Rg * Rg);
        const float rho = safe_sqrt(r * r - Rg * Rg);
        const float u_r = to_texcoord(rho / H, kSR);
        const float r_mu = r * mu;
        const float disc = r_mu * r_mu - r * r + Rg * Rg;
        float u_mu;
        if (ground) {
            const float d = -r_mu - safe_sqrt(disc);
            const float d_min = r - Rg, d_max = rho;
            u_mu = 0.5 - 0.5 * to_texcoord(d_max == d_min ? 0.0 : (d - d_min) / (d_max - d_min), kSMu / 2);
        } else {
            const float d = -r_mu + safe_sqrt(disc + H * H);
            const float d_min = Rt - r, d_max = rho + H;
            u_mu = 0.5 + 0.5 * to_texcoord((d - d_min) / (d_max - d_min), kSMu / 2);
        }
        const float d = dist_to_top(Rg, mu_s);
        const float d_min = Rt - Rg, d_max = H;
        const float aa = (d - d_min) / (d_max - d_min);
        const float A = -2.0 * a.mu_s_min * Rg / (d_max - d_min);
        const float u_mu_s = to_texcoord(max(1.0 - aa / A, 0.0) / (1.0 + aa), kSMuS);
        const float u_nu = (nu + 1.0) / 2.0;
        return make_float4(u_nu, u_mu_s, u_mu, u_r);
    }
    __device__ void scattering_params(float4 uvwz, float& r, float& mu, float& mu_s, float& nu, bool& ground) const {
        const float H = sqrt(Rt * Rt - Rg * Rg);
        const float rho = H * from_texcoord(uvwz.w, kSR);
        r = sqrt(rho * rho + Rg * Rg);
        if (uvwz.z < 0.5) {
            const float d_min = r - Rg, d_max = rho;
            const float d = d_min + (d_max - d_min) * from_texcoord(1.0 - 2.0 * uvwz.z, kSMu / 2);
            mu = d == 0.0f ? float(-1.0) : clamp_cos(-(rho * rho + d * d) / (2.0 * r * d));
            ground = true;
        } else {
            const float d_min = Rt - r, d_max = rho + H;
            const float d = d_min + (d_max - d_min) * from_texcoord(2.0 * uvwz.z - 1.0, kSMu / 2);
            mu = d == 0.0f ? float(1.0) : clamp_cos((H * H - rho * rho - d * d) / (2.0 * r * d));
            ground = false;
        }
        const float x_mu_s = from_texcoord(uvwz.y, kSMuS);
        const float d_min = Rt - Rg, d_max = H;
        const float A = -2.0 * a.mu_s_min * Rg / (d_max - d_min);
        const float aa = (A - x_mu_s * A) / (1.0 + x_mu_s * A);
        const float d = d_min + min(aa, A) * (d_max - d_min);
        mu_s = d == 0.0f ? float(1.0) : clamp_cos((H * H - d * d) / (2.0 * Rg * d));
        nu = clamp_cos(uvwz.x * 2.0 - 1.0);
    }
    __device__ void scattering_params_at(float fx, float fy, float fz, float& r, float& mu, float& mu_s, float& nu, bool& ground) const {
        const float frag_nu = floor(fx / float(kSMuS));
        const float frag_mu_s = fmodf(fx, float(kSMuS));
        const float4 uvwz = make_float4(frag_nu / float(kSNu - 1), frag_mu_s / float(kSMuS), fy / float(kSMu), fz / float(kSR));
        scattering_params(uvwz, r, mu, mu_s, nu, ground);
        const double s = sqrt((1.0 - mu * mu) * (1.0 - mu_s * mu_s));     // the bounds are formed in double and rounded once (:362)
        nu = clampf(nu, mu * mu_s - s, mu * mu_s + s);
    }
    // nearest-texel read of a scattering table at the two nu slices around the coordinate (:375-395).  The texel coordinates are
    // NOT clamped per axis: like the reference, a coordinate one below 0 or at the table size addresses the neighbouring row /
    // slice through the linear index; only a linear index outside the table (where the reference reads beyond its buffer) is
    // clamped to the table's first / last texel.
    __device__ V3 scattering_lookup(const float4* table, float r, float mu, float mu_s, float nu, bool ground) const {
        const float4 uvwz = scattering_uvwz(r, mu, mu_s, nu, ground);
        const float tex_coord_x = uvwz.x * float(kSNu - 1);
        const float tex_x = floor(tex_coord_x);
        const float lerp = tex_coord_x - tex_x;
        const float u0 = (tex_x + uvwz.y) / float(kSNu), u1 = (tex_x + 1.0 + uvwz.y) / float(kSNu);
        const int x0 = int(u0 * kSW), x1 = int(u1 * kSW), y = int(uvwz.z * kSH), z = int(uvwz.w * kSD);
        const int n = kSW * kSH * kSD;
        const int i0 = min(max(x0 + kSW * (y + kSH * z), 0), n - 1), i1 = min(max(x1 + kSW * (y + kSH * z), 0), n - 1);
        const float4 v0 = table[i0], v1 = table[i1];
        return v3(v0) * (1.0 - lerp) + v3(v1) * lerp;
    }
    __device__ V3 scattering_of_order(float r, float mu, float mu_s, float nu, bool ground, int order) const {
        if (order == 1) {
            const V3 ray = scattering_lookup(t.delta_rayleigh, r, mu, mu_s, nu, ground);
            const V3 mie = scattering_lookup(t.delta_mie, r, mu, mu_s, nu, ground);
            return ray * rayleigh_phase(nu) + mie * mie_phase(a.mie_phase_function_g, nu);
        }
        return scattering_lookup(t.scattering, r, mu, mu_s, nu, ground);          // the running table, not the per-order delta (:383-386)
    }

    // ---- irradiance (:560-618) ----
    __device__ float2 irradiance_uv(float r, float mu_s) const {
        const float x_r = (r - Rg) / (Rt - Rg);
        const float x_mu_s = mu_s * 0.5 + 0.5;
        return make_float2(to_texcoord(x_mu_s, kIW), to_texcoord(x_r, kIH));
    }
    __device__ void irradiance_r_mu_s(float2 uv, float& r, float& mu_s) const {
        const float x_mu_s = from_texcoord(uv.x, kIW), x_r = from_texcoord(uv.y, kIH);
        r = Rg + x_r * (Rt - Rg);
        mu_s = clamp_cos(2.0 * x_mu_s - 1.0);
    }
    __device__ V3 irradiance_lookup(float r, float mu_s) const {
        const float2 uv = irradiance_uv(r, mu_s);
        const int x = int(floor(uv.x * kIW)), y = int(floor(uv.y * kIH));
        int idx = y * kIW + x;
        idx = min(max(idx, 0), kIW * kIH - 1);
        return v3(t.irradiance[idx]);                                               // the running table (:452, :607-618)
    }
    __device__ V3 direct_irradiance(float r, float mu_s) const {
        const float alpha_s = a.sun_angular_radius;
        const float avg_cos = mu_s < -alpha_s ? 0.0 : (mu_s > alpha_s ? mu_s : (mu_s + alpha_s) * (mu_s + alpha_s) / (4.0 * alpha_s));
        return v3(a.solar_irradiance) * transmittance_to_top(r, mu_s) * avg_cos;
    }
    __device__ V3 indirect_irradiance(float r, float mu_s, int order) const {
        const int N = 32;
        const float dphi = kPi / float(N), dtheta = kPi / float(N);
        V3 result = v3(0.0f);
        const V3 omega_s = v3(sqrt(1.0 - mu_s * mu_s), 0.0, mu_s);
        for (int j = 0; j < N / 2; ++j) {
            const float theta = (float(j) + 0.5) * dtheta;
            for (int i = 0; i < 2 * N; ++i) {
                const float phi = (float(i) + 0.5) * dphi;
                const V3 omega = v3(cos(phi) * sin(theta), sin(phi) * sin(theta), cos(theta));
                const float domega = dtheta * dphi * sin(theta);
                const float nu = dot3(omega, omega_s);
                result += scattering_of_order(r, omega.z, mu_s, nu, false, order) * omega.z * domega;
            }
        }
        return result;
    }

    // ---- scattering density and multiple scattering (:390-520) ----
    __device__ V3 scattering_density(float r, float mu, float mu_s, float nu, int order) const {
        const V3 zenith = v3(0.0, 0.0, 1.0);
        const V3 omega = v3(sqrt(1.0f - mu * mu), 0.0, mu);
        const float sun_x = omega.x == 0.0 ? 0.0 : (nu - mu * mu_s) / omega.x;
        const float sun_y = sqrt(max(1.0 - sun_x * sun_x - mu_s * mu_s, 0.0));
        const V3 omega_s = v3(sun_x, sun_y, mu_s);
        const int N = 16;
        const float dphi = kPi / float(N), dtheta = kPi / float(N);
        V3 acc = v3(0.0f);
        for (int l = 0; l < N; ++l) {
            const float theta = (float(l) + 0.5) * dtheta;
            const float cos_theta = cos(theta), sin_theta = sin(theta);
            const bool ground = hits_ground(r, cos_theta);
            float dist_ground = 0.0f;
            V3 tr_ground = v3(0.0f), albedo = v3(0.0f);
            if (ground) {
                dist_ground = dist_to_bottom(r, cos_theta);
                tr_ground = transmittance(r, cos_theta, dist_ground, true);
                albedo = v3(a.ground_albedo);
            }
            for (int m = 0; m < 2 * N; ++m) {
                const float phi = (float(m) + 0.5) * dphi;
                const V3 omega_i = v3(cos(phi) * sin_theta, sin(phi) * sin_theta, cos_theta);
                const float domega_i = dtheta * dphi * sin(theta);
                const float nu1 = dot3(omega_s, omega_i);
                V3 incident = scattering_of_order(r, omega_i.z, mu_s, nu1, ground, order - 1);
                V3 gn = zenith * r + omega_i * dist_ground;
                const float inv = rsqrtf(dot3(gn, gn));
                gn = gn * inv;
                const V3 ground_irr = irradiance_lookup(Rg, dot3(gn, omega_s));
                incident += tr_ground * albedo * (1.0 / kPi) * ground_irr;
                const float nu2 = dot3(omega, omega_i);
                const float ray_d = profile_density(a.rayleigh_density, r - Rg), mie_d = profile_density(a.mie_density, r - Rg);
                acc += incident * (v3(a.rayleigh_scattering) * ray_d * rayleigh_phase(nu2) + v3(a.mie_scattering) * mie_d * mie_phase(a.mie_phase_function_g, nu2)) * domega_i;
            }
        }
        return acc;
    }
    __device__ V3 multiple_scattering(float r, float mu, float mu_s, float nu, bool ground) const {
        const int N = 50;
        const float dx = dist_to_nearest(r, mu, ground) / float(N);
        V3 sum = v3(0.0f);
        for (int i = 0; i <= N; ++i) {
            const float d_i = float(i) * dx;
            const float r_i = clamp_radius(sqrt(d_i * d_i + 2.0 * r * mu * d_i + r * r));
            const float mu_i = clamp_cos((r * mu + d_i) / r_i);
            const float mu_s_i = clamp_cos((r * mu_s + d_i * nu) / r_i);
            const V3 v = scattering_lookup(t.delta_density, r_i, mu_i, mu_s_i, nu, ground) * transmittance(r, mu, d_i, ground) * dx;
            const float w_i = (i == 0 || i == N) ? 0.5 : 1.0;
            sum += v * w_i;
        }
        return sum;
    }
};

// ---- kernels: one thread per texel, the writes and read-modify-writes of atmosphere_kernels.cu:621-752 ---------------------------------
__global__ void k_transmittance(const vpt_atmosphere atm, const Tables t)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= kTW || y >= kTH) return;
    const Model M(atm, t);
    float r, mu;
    M.transmittance_r_mu(make_float2((x + 0.5f) / float(kTW), (y + 0.5f) / float(kTH)), r, mu);
    t.transmittance[y * kTW + x] = f4(M.compute_transmittance_to_top(r, mu), 0.0f);
}

__global__ void k_direct_irradiance(const vpt_atmosphere atm, const Tables t, const int blend)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= kIW || y >= kIH) return;
    const int idx = y * kIW + x;
    const Model M(atm, t);
    if (!blend) t.irradiance[idx] = make_float4(.0f, .0f, .0f, .0f);
    const float4 prev = t.irradiance[idx];
    float r, mu_s;
    M.irradiance_r_mu_s(make_float2((x + 0.5f) / float(kIW), (y + 0.5f) / float(kIH)), r, mu_s);
    t.delta_irradiance[idx] = f4(M.direct_irradiance(r, mu_s), 0.0f);
    if (blend) { float4 v = t.irradiance[idx]; v.x += prev.x; v.y += prev.y; v.z += prev.z; v.w += prev.w; t.irradiance[idx] = v; }
}

__global__ void k_single_scattering(const vpt_atmosphere atm, const Tables t, const int blend_scattering, const int blend_mie, const Mat3 lfr)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, z = blockIdx.z * blockDim.z + threadIdx.z;
    if (x >= kSW || y >= kSH || z >= kSD) return;
    const int idx = x + kSW * (y + kSH * z);
    const Model M(atm, t);
    const float4 prev_s = t.scattering[idx], prev_m = t.single_mie[idx];
    float r, mu, mu_s, nu; bool ground;
    M.scattering_params_at(x + 0.5f, y + 0.5f, z + 0.5f, r, mu, mu_s, nu, ground);
    V3 ray, mie;
    M.single_scattering(r, mu, mu_s, nu, ground, ray, mie);
    t.delta_rayleigh[idx] = f4(ray, 1.0f);
    t.delta_mie[idx] = f4(mie, 1.0f);
    float4 s = f4(mul(lfr, ray), mul(lfr, mie).x), m = f4(mie, 1.0f);
    if (blend_scattering) { s.x += prev_s.x; s.y += prev_s.y; s.z += prev_s.z; s.w += prev_s.w; }
    if (blend_mie) { m.x += prev_m.x; m.y += prev_m.y; m.z += prev_m.z; m.w += prev_m.w; }
    t.scattering[idx] = s; t.single_mie[idx] = m;
}

__global__ void k_scattering_density(const vpt_atmosphere atm, const Tables t, const int order)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, z = blockIdx.z * blockDim.z + threadIdx.z;
    if (x >= kSW || y >= kSH || z >= kSD) return;
    const Model M(atm, t);
    float r, mu, mu_s, nu; bool ground;
    M.scattering_params_at(x + 0.5f, y + 0.5f, z + 0.5f, r, mu, mu_s, nu, ground);
    t.delta_density[x + kSW * (y + kSH * z)] = f4(M.scattering_density(r, mu, mu_s, nu, order), 1.0f);
}

__global__ void k_indirect_irradiance(const vpt_atmosphere atm, const Tables t, const int blend, const Mat3 lfr, const int order)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= kIW || y >= kIH) return;
    const int idx = y * kIW + x;
    const Model M(atm, t);
    float r, mu_s;
    M.irradiance_r_mu_s(make_float2((x + 0.5f) / float(kIW), (y + 0.5f) / float(kIH)), r, mu_s);
    const V3 delta = M.indirect_irradiance(r, mu_s, order - 1);
    const float4 prev = t.irradiance[idx];
    float4 v = f4(mul(lfr, delta), 0.0f);
    t.delta_irradiance[idx] = v;
    if (blend) { v.x += prev.x; v.y += prev.y; v.z += prev.z; v.w += prev.w; }
    t.irradiance[idx] = v;
}

__global__ void k_multiple_scattering(const vpt_atmosphere atm, const Tables t, const int blend, const Mat3 lfr)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, z = blockIdx.z * blockDim.z + threadIdx.z;
    if (x >= kSW || y >= kSH || z >= kSD) return;
    const int idx = x + kSW * (y + kSH * z);
    const Model M(atm, t);
    const float4 prev = t.scattering[idx];
    float r, mu, mu_s, nu; bool ground;
    M.scattering_params_at(x + 0.5f, y + 0.5f, z + 0.5f, r, mu, mu_s, nu, ground);
    const V3 delta = M.multiple_scattering(r, mu, mu_s, nu, ground);
    t.delta_multiple[idx] = f4(delta, 1.0f);
    float4 v = f4(mul(lfr, delta) / Model::rayleigh_phase(nu), .0f);
    if (blend) { v.x += prev.x; v.y += prev.y; v.z += prev.z; v.w += prev.w; }
    t.scattering[idx] = v;
}

} // namespace bru

// One launch of one of the six table kernels (stage = VPT_BRUNETON_*, vpt_b200.h) on the nine tables in the order of definitions.h:82-90.
// `blend` goes to every kernel that takes it (single scattering: both flags); `order` to the three kernels of the later orders.
cudaError_t bruneton_stage(int stage, const vpt_atmosphere& atm, float4* const tables[9], const float lfr9[9], int blend, int order, cudaStream_t s)
{
    bru::Tables t;
    t.delta_irradiance = tables[0]; t.delta_rayleigh = tables[1]; t.delta_mie = tables[2]; t.delta_density = tables[3]; t.delta_multiple = tables[4];
    t.transmittance = tables[5]; t.irradiance = tables[6]; t.scattering = tables[7]; t.single_mie = tables[8];
    bru::Mat3 M; for (int i = 0; i < 9; ++i) M.m[i] = lfr9[i];
    const dim3 b2(8, 8, 1), b3(8, 8, 8);
    const dim3 gt((bru::kTW + 7) / 8, (bru::kTH + 7) / 8, 1), gi((bru::kIW + 7) / 8, (bru::kIH + 7) / 8, 1);
    const dim3 gs((bru::kSW + 7) / 8, (bru::kSH + 7) / 8, (bru::kSD + 7) / 8);
    switch (stage) {
    case 0: bru::k_transmittance<<<gt, b2, 0, s>>>(atm, t); break;
    case 1: bru::k_direct_irradiance<<<gi, b2, 0, s>>>(atm, t, blend); break;
    case 2: bru::k_single_scattering<<<gs, b3, 0, s>>>(atm, t, blend, blend, M); break;
    case 3: bru::k_scattering_density<<<gs, b3, 0, s>>>(atm, t, order); break;
    case 4: bru::k_indirect_irradiance<<<gi, b2, 0, s>>>(atm, t, blend, M, order); break;
    case 5: bru::k_multiple_scattering<<<gs, b3, 0, s>>>(atm, t, blend, M); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// One precompute iteration = atmosphere::precompute (atmosphere.cpp:888-1114): transmittance, direct irradiance, single scattering,
// then for every further order {scattering density, indirect irradiance, multiple scattering}.  `blend` is the host's BLEND flag
// (accumulate over wavelength triples, luminance mode PRECOMPUTED); the later kernels of the reference receive 0 whatever it is
// (quirk Q17) and so do these.  `transmittance_only`: atmosphere::compute_transmittance.
cudaError_t bruneton_iteration(const vpt_atmosphere& atm, float4* const tables[9], const float lfr9[9], int blend, int orders, int transmittance_only, cudaStream_t s)
{
    cudaError_t e = bruneton_stage(0, atm, tables, lfr9, 0, 0, s);
    if (transmittance_only) return e;
    if (e == cudaSuccess) e = bruneton_stage(1, atm, tables, lfr9, blend, 0, s);
    if (e == cudaSuccess) e = bruneton_stage(2, atm, tables, lfr9, blend, 0, s);
    for (int order = 2; order <= orders && e == cudaSuccess; ++order)
        for (int stage = 3; stage <= 5 && e == cudaSuccess; ++stage) e = bruneton_stage(stage, atm, tables, lfr9, 0, order, s);
    return e;
}

// texel centres of a float4 texture (linear filtering returns the texel itself there): tests read LUTs back through this
__global__ void k_texture_readback(cudaTextureObject_t tex, int w, int h, int d, float4* out)
{
    const size_t n = (size_t)w * h * (d > 0 ? d : 1);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % w), y = (int)((i / w) % h), z = (int)(i / ((size_t)w * h));
        out[i] = d > 0 ? tex3D<float4>(tex, (x + 0.5f) / w, (y + 0.5f) / h, (z + 0.5f) / d) : tex2D<float4>(tex, (x + 0.5f) / w, (y + 0.5f) / h);
    }
}

// arbitrary sample points of a single-channel 3-D texture (filter diagnostics)
__global__ void k_texture_sample_f1(cudaTextureObject_t tex, const float* __restrict__ uvw, int n, float* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = tex3D<float>(tex, uvw[3 * i], uvw[3 * i + 1], uvw[3 * i + 2]);
}

cudaError_t launch_texture_sample_f1(unsigned long long tex, const float* d_uvw, int n, float* d_out, cudaStream_t s)
{
    k_texture_sample_f1<<<(n + 255) / 256, 256, 0, s>>>((cudaTextureObject_t)tex, d_uvw, n, d_out);
    return cudaGetLastError();
}

cudaError_t launch_texture_readback(unsigned long long tex, int w, int h, int d, float4* d_out, cudaStream_t s)
{
    k_texture_readback<<<592, 256, 0, s>>>((cudaTextureObject_t)tex, w, h, d, d_out);
    return cudaGetLastError();
}

} // namespace vpt
