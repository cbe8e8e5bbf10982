// vpt_atmosphere_host.cpp -- host side of the Bruneton sky precompute (SURVEY 8(f) row N2) behind the C ABI.
//
// Replaces atmosphere::init / precompute / update_model / copy_*_texture (source/atmosphere/atmosphere.cpp:1177-1291, 888-1114,
// 676-783, 503-674): builds the model's spectra, reduces them to the three-wavelength AtmosphereParameters block the render path
// reads by value, runs the table kernels (vpt_bruneton.cu) and wraps the four tables the render path samples as textures with the
// reference's descriptors.  Constants are Bruneton's published Earth model as the reference configures it (atmosphere.h:66-109).
// Quirks of the reference that change the numbers are kept and marked (Q): mie_extinction is interpolated from the Mie SCATTERING
// spectrum (atmosphere.cpp:726-728); ground albedo 0.01; orders 2..4 overwrite instead of accumulate (see vpt_bruneton.cu).
#include "vpt_host.h"

#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "cie1931.inc"

namespace vpt {
cudaError_t bruneton_iteration(const vpt_atmosphere& atm, float4* const tables[9], const float lfr9[9], int blend, int orders, int transmittance_only, cudaStream_t s);
cudaError_t bruneton_stage(int stage, const vpt_atmosphere& atm, float4* const tables[9], const float lfr9[9], int blend, int order, cudaStream_t s);
cudaError_t launch_texture_readback(unsigned long long tex, int w, int h, int d, float4* d_out, cudaStream_t s);
cudaError_t launch_texture_sample_f1(unsigned long long tex, const float* d_uvw, int n, float* d_out, cudaStream_t s);
}

namespace {

constexpr int kLambdaMin = 360, kLambdaMax = 830;
constexpr double kLambdaR = 680.0, kLambdaG = 550.0, kLambdaB = 440.0;
constexpr double kMaxLuminousEfficacy = 683.0;
// solar spectrum (W/m^2/nm) and ozone cross-section (m^2) at 360, 370, ... 830 nm: Bruneton's Earth model data (atmosphere.h:66-83)
const double kSolar[48] = {
    1.11776, 1.14259, 1.01249, 1.14716, 1.72765, 1.73054, 1.6887, 1.61253, 1.91198, 2.03474, 2.02042, 2.02212, 1.93377, 1.95809, 1.91686, 1.8298,
    1.8685, 1.8931, 1.85149, 1.8504, 1.8341, 1.8345, 1.8147, 1.78158, 1.7533, 1.6965, 1.68194, 1.64654, 1.6048, 1.52143, 1.55622, 1.5113,
    1.474, 1.4482, 1.41018, 1.36775, 1.34188, 1.31429, 1.28303, 1.26758, 1.2367, 1.2082, 1.18737, 1.14683, 1.12362, 1.1058, 1.07124, 1.04992 };
const double kOzone[48] = {
    1.18e-27, 2.182e-28, 2.818e-28, 6.636e-28, 1.527e-27, 2.763e-27, 5.52e-27, 8.451e-27, 1.582e-26, 2.316e-26, 3.669e-26, 4.924e-26,
    7.752e-26, 9.016e-26, 1.48e-25, 1.602e-25, 2.139e-25, 2.755e-25, 3.091e-25, 3.5e-25, 4.266e-25, 4.672e-25, 4.398e-25, 4.701e-25,
    5.019e-25, 4.305e-25, 3.74e-25, 3.215e-25, 2.662e-25, 2.238e-25, 1.852e-25, 1.473e-25, 1.209e-25, 9.423e-26, 7.455e-26, 6.566e-26,
    5.105e-26, 4.15e-26, 4.228e-26, 3.237e-26, 2.451e-26, 2.801e-26, 2.534e-26, 1.624e-26, 1.465e-26, 2.078e-26, 1.383e-26, 7.105e-27 };
const double kXyzToSrgb[9] = { +3.2406, -1.5372, -0.4986, -0.9689, +1.8758, +0.0415, +0.0557, -0.2040, +1.0570 };
constexpr double kDobsonUnit = 2.687e20, kMaxOzoneNumberDensity = 300.0 * kDobsonUnit / 15000.0;
constexpr double kConstantSolarIrradiance = 1.5, kRayleigh = 1.24062e-6, kRayleighScaleHeight = 8000.0, kMieScaleHeight = 1200.0;
constexpr double kMieAngstromAlpha = 0.0, kMieAngstromBeta = 5.328e-3, kMieSingleScatteringAlbedo = 0.9, kGroundAlbedo = 0.01;

struct Spectra { std::vector<double> wl, solar, rayleigh, mie_scattering, mie_extinction, absorption, albedo; };

// CIE colour-matching function `col` (0 x, 1 y, 2 z) at a wavelength, linear between the 5 nm samples, 0 outside (360, 830)
double cie(double wavelength, int col) {
    if (wavelength <= kLambdaMin || wavelength >= kLambdaMax) return 0.0;
    double u = (wavelength - kLambdaMin) / 5.0;
    const int row = (int)floor(u);
    u -= row;
    const double* t = col == 0 ? kCieXbar : col == 1 ? kCieYbar : kCieZbar;
    return t[row] * (1.0 - u) + t[row + 1] * u;
}

double interp(const std::vector<double>& wl, const std::vector<double>& f, double w) {
    if (w < wl[0]) return f[0];
    for (size_t i = 0; i + 1 < wl.size(); ++i)
        if (w < wl[i + 1]) { const double u = (w - wl[i]) / (wl[i + 1] - wl[i]); return f[i] * (1.0 - u) + f[i + 1] * u; }
    return f.back();
}

// factors turning the 3-wavelength spectral radiance into sRGB luminance (atmosphere.cpp:185-213)
void radiance_to_luminance_factors(const Spectra& s, double lambda_power, double k[3]) {
    k[0] = k[1] = k[2] = 0.0;
    const double sr = interp(s.wl, s.solar, kLambdaR), sg = interp(s.wl, s.solar, kLambdaG), sb = interp(s.wl, s.solar, kLambdaB);
    for (int lambda = kLambdaMin; lambda < kLambdaMax; ++lambda) {
        const double x = cie(lambda, 0), y = cie(lambda, 1), z = cie(lambda, 2);
        const double r = kXyzToSrgb[0] * x + kXyzToSrgb[1] * y + kXyzToSrgb[2] * z;
        const double g = kXyzToSrgb[3] * x + kXyzToSrgb[4] * y + kXyzToSrgb[5] * z;
        const double b = kXyzToSrgb[6] * x + kXyzToSrgb[7] * y + kXyzToSrgb[8] * z;
        const double irr = interp(s.wl, s.solar, lambda);
        k[0] += r * irr / sr * pow(lambda / kLambdaR, lambda_power);
        k[1] += g * irr / sg * pow(lambda / kLambdaG, lambda_power);
        k[2] += b * irr / sb * pow(lambda / kLambdaB, lambda_power);
    }
    for (int c = 0; c < 3; ++c) k[c] *= kMaxLuminousEfficacy;
}

void white_point(const Spectra& s, double wp[3]) {                      // convert_spectrum_to_linear_srgb + normalisation (:215-234, 680-693)
    double x = 0, y = 0, z = 0;
    for (int lambda = kLambdaMin; lambda < kLambdaMax; ++lambda) {
        const double v = interp(s.wl, s.solar, lambda);
        x += cie(lambda, 0) * v; y += cie(lambda, 1) * v; z += cie(lambda, 2) * v;
    }
    wp[0] = kMaxLuminousEfficacy * (kXyzToSrgb[0] * x + kXyzToSrgb[1] * y + kXyzToSrgb[2] * z);
    wp[1] = kMaxLuminousEfficacy * (kXyzToSrgb[3] * x + kXyzToSrgb[4] * y + kXyzToSrgb[5] * z);
    wp[2] = kMaxLuminousEfficacy * (kXyzToSrgb[6] * x + kXyzToSrgb[7] * y + kXyzToSrgb[8] * z);
    const double m = (wp[0] + wp[1] + wp[2]) / 3.0;
    wp[0] /= m; wp[1] /= m; wp[2] /= m;
}

double srgb_coeff(double lambda, int component) {                       // atmosphere::coeff, :137-146
    const double x = cie(lambda, 0), y = cie(lambda, 1), z = cie(lambda, 2);
    return kXyzToSrgb[component * 3 + 0] * x + kXyzToSrgb[component * 3 + 1] * y + kXyzToSrgb[component * 3 + 2] * z;
}

vpt_f3 f3d(double x, double y, double z) { vpt_f3 v = { (float)x, (float)y, (float)z }; return v; }

vpt_density_layer layer(double width, double exp_term, double exp_scale, double linear_term, double const_term) {
    vpt_density_layer l; memset(&l, 0, sizeof(l));
    l.width = (float)width; l.exp_term = (float)exp_term; l.exp_scale = (float)exp_scale; l.linear_term = (float)linear_term; l.const_term = (float)const_term;
    return l;
}

// atmosphere::update_model(lambdas), :696-783: the by-value block for one triple of wavelengths
void fill_model(vpt_atmosphere& P, const Spectra& s, const double lambdas[3], const double sky_k[3], const double sun_k[3], const vpt_atmosphere_options& o) {
    P.sky_spectral_radiance_to_luminance = f3d(sky_k[0], sky_k[1], sky_k[2]);
    P.sun_spectral_radiance_to_luminance = f3d(sun_k[0], sun_k[1], sun_k[2]);
    P.solar_irradiance = f3d(interp(s.wl, s.solar, lambdas[0]), interp(s.wl, s.solar, lambdas[1]), interp(s.wl, s.solar, lambdas[2]));
    P.sun_angular_radius = (float)(0.00935 / 2.0);
    P.bottom_radius = 6360000.0f; P.top_radius = 6420000.0f;           // length unit: metres
    memset(&P.rayleigh_density, 0, sizeof(P.rayleigh_density)); memset(&P.mie_density, 0, sizeof(P.mie_density)); memset(&P.absorption_density, 0, sizeof(P.absorption_density));
    P.rayleigh_density.layers[1] = layer(0.0, 1.0, -1.0 / kRayleighScaleHeight, 0.0, 0.0);
    P.rayleigh_scattering = f3d(interp(s.wl, s.rayleigh, lambdas[0]), interp(s.wl, s.rayleigh, lambdas[1]), interp(s.wl, s.rayleigh, lambdas[2]));
    P.mie_density.layers[1] = layer(0.0, 1.0, -1.0 / kMieScaleHeight, 0.0, 0.0);
    P.mie_scattering = f3d(interp(s.wl, s.mie_scattering, lambdas[0]), interp(s.wl, s.mie_scattering, lambdas[1]), interp(s.wl, s.mie_scattering, lambdas[2]));
    P.mie_extinction = P.mie_scattering;                                // (Q) the reference interpolates m_mie_scattering here, :726-728
    P.mie_phase_function_g = 0.8f;
    P.absorption_density.layers[0] = layer(25000.0, 0.0, 0.0, 1.0 / 15000.0, -2.0 / 3.0);
    P.absorption_density.layers[1] = layer(0.0, 0.0, 0.0, -1.0 / 15000.0, 8.0 / 3.0);
    P.absorption_extinction = f3d(interp(s.wl, s.absorption, lambdas[0]), interp(s.wl, s.absorption, lambdas[1]), interp(s.wl, s.absorption, lambdas[2]));
    P.ground_albedo = f3d(interp(s.wl, s.albedo, lambdas[0]), interp(s.wl, s.albedo, lambdas[1]), interp(s.wl, s.albedo, lambdas[2]));
    // pi is a FLOAT literal in the reference's translation unit (common/helper_math.h:47 redefines M_PI), widened to double for
    // the product: cos gives -0.50000006, not -0.5 (atmosphere.cpp:746-747)
    P.mu_s_min = (float)cos(120.0 / 180.0 * (double)3.14159265358979323846f);
    P.use_luminance = o.luminance_mode == 1 ? 1 : o.luminance_mode == 2 ? 2 : 0;
    double wp[3] = { 1.0, 1.0, 1.0 };
    if (o.do_white_balance) white_point(s, wp);
    P.white_point = f3d(wp[0], wp[1], wp[2]);
    P.exposure = o.exposure;
}

struct AtmosphereHandle {
    float4* slab = nullptr;                      // the nine working tables (freed after the textures exist)
    cudaArray_t arrays[4] = { nullptr, nullptr, nullptr, nullptr };
    cudaTextureObject_t tex[4] = { 0, 0, 0, 0 };
};

cudaError_t texture_from_device_2d(const float4* d, int w, int h, cudaArray_t* arr, cudaTextureObject_t* tex) {
    const cudaChannelFormatDesc desc = cudaCreateChannelDesc<float4>();
    cudaError_t e = cudaMallocArray(arr, &desc, w, h);
    if (e == cudaSuccess) e = cudaMemcpy2DToArray(*arr, 0, 0, d, (size_t)w * sizeof(float4), (size_t)w * sizeof(float4), h, cudaMemcpyDeviceToDevice);
    cudaResourceDesc res; memset(&res, 0, sizeof(res)); res.resType = cudaResourceTypeArray; res.res.array.array = *arr;
    cudaTextureDesc td; memset(&td, 0, sizeof(td));                    // atmosphere.cpp:523-530
    td.addressMode[0] = cudaAddressModeWrap; td.addressMode[1] = cudaAddressModeClamp; td.addressMode[2] = cudaAddressModeWrap;
    td.filterMode = cudaFilterModeLinear; td.readMode = cudaReadModeElementType; td.normalizedCoords = 1;
    if (e == cudaSuccess) e = cudaCreateTextureObject(tex, &res, &td, NULL);
    return e;
}

cudaError_t texture_from_device_3d(const float4* d, int w, int h, int dep, cudaArray_t* arr, cudaTextureObject_t* tex) {
    const cudaChannelFormatDesc desc = cudaCreateChannelDesc<float4>();
    const cudaExtent ext = make_cudaExtent((size_t)w, (size_t)h, (size_t)dep);
    cudaError_t e = cudaMalloc3DArray(arr, &desc, ext);
    cudaMemcpy3DParms cp; memset(&cp, 0, sizeof(cp));
    cp.srcPtr = make_cudaPitchedPtr((void*)d, (size_t)w * sizeof(float4), (size_t)w, (size_t)h);
    cp.dstArray = *arr; cp.extent = ext; cp.kind = cudaMemcpyDeviceToDevice;
    if (e == cudaSuccess) e = cudaMemcpy3D(&cp);
    cudaResourceDesc res; memset(&res, 0, sizeof(res)); res.resType = cudaResourceTypeArray; res.res.array.array = *arr;
    cudaTextureDesc td; memset(&td, 0, sizeof(td));                    // atmosphere.cpp:604-615
    td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
    td.filterMode = cudaFilterModeLinear; td.readMode = cudaReadModeElementType; td.normalizedCoords = 1;
    if (e == cudaSuccess) e = cudaCreateTextureObject(tex, &res, &td, NULL);
    return e;
}

} // namespace

extern "C" {

void vpt_atmosphere_options_defaults(vpt_atmosphere_options* o) {       // main.cpp:1433-1436
    if (!o) return;
    o->use_constant_solar_spectrum = 1; o->use_ozone = 1; o->luminance_mode = 0; o->do_white_balance = 1; o->exposure = 1.0f; o->num_scattering_orders = 4;
}

int vpt_atmosphere_precompute(const vpt_atmosphere_options* opt, vpt_atmosphere* out, void** handle_out) {
    if (!opt || !out || !handle_out) return vpt::fail_global(VPT_ERR_INVALID, "vpt_atmosphere_precompute: null argument");
    if (opt->num_scattering_orders < 1 || opt->num_scattering_orders > 16 || opt->luminance_mode < 0 || opt->luminance_mode > 2)
        return vpt::fail_global(VPT_ERR_INVALID, "vpt_atmosphere_precompute: bad options");
    *handle_out = nullptr;
    // spectra at 360, 370, ... 830 nm (atmosphere::init, :1199-1215)
    Spectra s;
    for (int l = kLambdaMin; l <= kLambdaMax; l += 10) {
        const double lambda = (double)l * 1e-3;                         // micrometres
        const double mie = kMieAngstromBeta / kMieScaleHeight * pow(lambda, -kMieAngstromAlpha);
        s.wl.push_back(l);
        s.solar.push_back(opt->use_constant_solar_spectrum ? kConstantSolarIrradiance : kSolar[(l - kLambdaMin) / 10]);
        s.rayleigh.push_back(kRayleigh * pow(lambda, -4));
        s.mie_scattering.push_back(mie * kMieSingleScatteringAlbedo);
        s.mie_extinction.push_back(mie);
        s.absorption.push_back(opt->use_ozone ? kMaxOzoneNumberDensity * kOzone[(l - kLambdaMin) / 10] : 0.0);
        s.albedo.push_back(kGroundAlbedo);
    }
    double sky_k[3], sun_k[3];
    if (opt->luminance_mode == 2) sky_k[0] = sky_k[1] = sky_k[2] = kMaxLuminousEfficacy;
    else radiance_to_luminance_factors(s, -3.0, sky_k);
    radiance_to_luminance_factors(s, 0.0, sun_k);

    const size_t small = (size_t)256 * 64, big = (size_t)256 * 128 * 32;
    const size_t counts[9] = { small, big, big, big, big, small, small, big, big };    // order of definitions.h:82-90
    size_t total = 0; for (size_t c : counts) total += c;
    AtmosphereHandle* h = new AtmosphereHandle();
    cudaError_t e = cudaMalloc(&h->slab, total * sizeof(float4));
    if (e == cudaSuccess) e = cudaMemset(h->slab, 0, total * sizeof(float4));
    float4* tables[9]; { size_t off = 0; for (int i = 0; i < 9; ++i) { tables[i] = h->slab + off; off += counts[i]; } }

    vpt_atmosphere P; memset(&P, 0, sizeof(P));
    const double default_lambdas[3] = { kLambdaR, kLambdaG, kLambdaB };
    const float identity[9] = { 1, 0, 0, 0, 1, 0, 0, 0, 1 };
    if (e == cudaSuccess) {
        if (opt->luminance_mode != 2) {
            fill_model(P, s, default_lambdas, sky_k, sun_k, *opt);
            e = vpt::bruneton_iteration(P, tables, identity, 0, opt->num_scattering_orders, 0, 0);
        } else {
            // 15 wavelengths in 5 triples, accumulated with the luminance-from-radiance matrices (:1236-1262), then the transmittance
            // table once more for the display wavelengths (:1268)
            const int n_iter = (15 + 2) / 3;
            const double dl = (kLambdaMax - kLambdaMin) / (3.0 * n_iter);
            for (int i = 0; i < n_iter && e == cudaSuccess; ++i) {
                const double lambdas[3] = { kLambdaMin + (3 * i + 0.5) * dl, kLambdaMin + (3 * i + 1.5) * dl, kLambdaMin + (3 * i + 2.5) * dl };
                float lfr[9];
                for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) lfr[r * 3 + c] = (float)(srgb_coeff(lambdas[c], r) * dl);
                fill_model(P, s, lambdas, sky_k, sun_k, *opt);
                e = vpt::bruneton_iteration(P, tables, lfr, i > 0 ? 1 : 0, opt->num_scattering_orders, 0, 0);
            }
            if (e == cudaSuccess) { fill_model(P, s, default_lambdas, sky_k, sun_k, *opt); e = vpt::bruneton_iteration(P, tables, identity, 0, opt->num_scattering_orders, 1, 0); }
        }
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    // tables -> textures (copy_*_texture, :503-674): transmittance, scattering, irradiance, single Mie
    if (e == cudaSuccess) e = texture_from_device_2d(tables[5], 256, 64, &h->arrays[0], &h->tex[0]);
    if (e == cudaSuccess) e = texture_from_device_3d(tables[7], 256, 128, 32, &h->arrays[1], &h->tex[1]);
    if (e == cudaSuccess) e = texture_from_device_2d(tables[6], 256, 64, &h->arrays[2], &h->tex[2]);
    if (e == cudaSuccess) e = texture_from_device_3d(tables[8], 256, 128, 32, &h->arrays[3], &h->tex[3]);
    cudaFree(h->slab); h->slab = nullptr;
    if (e != cudaSuccess) { vpt_atmosphere_destroy(h); return vpt::fail_global(VPT_ERR_CUDA, std::string("vpt_atmosphere_precompute: ") + cudaGetErrorString(e)); }
    P.transmittance_texture = (vpt_tex_t)h->tex[0]; P.scattering_texture = (vpt_tex_t)h->tex[1];
    P.irradiance_texture = (vpt_tex_t)h->tex[2]; P.single_mie_scattering_texture = (vpt_tex_t)h->tex[3];
    memcpy(out, &P, sizeof(P));
    *handle_out = h;
    return VPT_OK;
}

int vpt_atmosphere_destroy(void* handle) {
    AtmosphereHandle* h = reinterpret_cast<AtmosphereHandle*>(handle);
    if (!h) return VPT_OK;
    for (int i = 0; i < 4; ++i) { if (h->tex[i]) cudaDestroyTextureObject(h->tex[i]); if (h->arrays[i]) cudaFreeArray(h->arrays[i]); }
    cudaFree(h->slab);
    delete h;
    return VPT_OK;
}

int vpt_debug_bruneton_stage(int stage, const vpt_atmosphere* P, const vpt_devptr_t tables[9], const float lfr[9], int blend, int order) {
    if (!P || !tables || !lfr || stage < VPT_BRUNETON_TRANSMITTANCE || stage > VPT_BRUNETON_MULTIPLE_SCATTERING || blend < 0 || blend > 1 ||
        (stage >= VPT_BRUNETON_SCATTERING_DENSITY && (order < 2 || order > 16)))
        return vpt::fail_global(VPT_ERR_INVALID, "vpt_debug_bruneton_stage: bad arguments");
    float4* t[9];
    for (int i = 0; i < 9; ++i) {
        if (!tables[i] || tables[i] % 16) return vpt::fail_global(VPT_ERR_INVALID, "vpt_debug_bruneton_stage: null or misaligned table");
        t[i] = reinterpret_cast<float4*>(tables[i]);
    }
    cudaError_t e = vpt::bruneton_stage(stage, *P, t, lfr, blend, order, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return vpt::fail_global(VPT_ERR_CUDA, std::string("vpt_debug_bruneton_stage: ") + cudaGetErrorString(e));
    return VPT_OK;
}

int vpt_debug_texture_sample(vpt_tex_t tex, const float* uvw, int n, float* out) {
    if (!tex || !uvw || n < 1 || !out) return vpt::fail_global(VPT_ERR_INVALID, "vpt_debug_texture_sample: bad arguments");
    float *d_in = nullptr, *d_out = nullptr;
    cudaError_t e = cudaMalloc(&d_in, sizeof(float) * 3 * (size_t)n);
    if (e == cudaSuccess) e = cudaMalloc(&d_out, sizeof(float) * (size_t)n);
    if (e == cudaSuccess) e = cudaMemcpy(d_in, uvw, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = vpt::launch_texture_sample_f1(tex, d_in, n, d_out, 0);
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost);
    cudaFree(d_in); cudaFree(d_out);
    if (e != cudaSuccess) return vpt::fail_global(VPT_ERR_CUDA, std::string("vpt_debug_texture_sample: ") + cudaGetErrorString(e));
    return VPT_OK;
}

int vpt_texture_read_f4(vpt_tex_t tex, int w, int h, int d, float* host_out) {
    if (!tex || w < 1 || h < 1 || d < 0 || !host_out) return vpt::fail_global(VPT_ERR_INVALID, "vpt_texture_read_f4: bad arguments");
    const size_t n = (size_t)w * h * (d > 0 ? d : 1);
    float4* dev = nullptr;
    cudaError_t e = cudaMalloc(&dev, n * sizeof(float4));
    if (e == cudaSuccess) e = vpt::launch_texture_readback(tex, w, h, d, dev, 0);
    if (e == cudaSuccess) e = cudaMemcpy(host_out, dev, n * sizeof(float4), cudaMemcpyDeviceToHost);
    cudaFree(dev);
    if (e != cudaSuccess) return vpt::fail_global(VPT_ERR_CUDA, std::string("vpt_texture_read_f4: ") + cudaGetErrorString(e));
    return VPT_OK;
}

} // extern "C"
