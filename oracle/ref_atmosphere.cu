/* oracle/ref_atmosphere.cu -- TEST INFRASTRUCTURE (oracle side, never the product).
 *
 * Drives the reference's OWN Bruneton sky precompute so both render kernels (the unmodified reference
 * cubin and libvpt_b200) can be handed the same `AtmosphereParameters` -- scalars plus the four
 * look-up textures -- for environment_type == 0 parity tests.  The reference sources are compiled from
 * /root/reference at build time (oracle/Makefile: source/atmosphere/atmosphere.cpp and
 * atmosphere_kernels.cu); nothing is copied into the repo.
 *
 *   vptref_atmosphere_init : source/main.cpp:1468-1472 (`earth_atmosphere.init()`), with the GUI's default
 *                            switches of main.cpp:1433-1436 passed in by the caller.  The reference loads
 *                            "atmosphere_kernels.ptx" from the working directory (atmosphere.cpp:1190), so the
 *                            call runs with the cwd switched to `module_dir` (oracle/_ref/atmo).
 *   vptref_atmosphere_stage: ONE launch of one of the six `calculate_*` kernels of that cubin, with the launch shape and the
 *                            argument bytes of atmosphere::precompute (atmosphere.cpp:923-1083), on a caller-owned parameter
 *                            block whose nine buffer pointers the caller chose.  Lets a test drive the reference chain one
 *                            stage at a time and hand both implementations identical inputs.
 *
 * The reference's util/fileIO.cpp (OpenEXR/stb) and util/logger.cpp are not built; the five functions of
 * theirs that atmosphere.cpp links against are stubbed below: loaders report "no cached textures" (which makes
 * init() precompute, atmosphere.cpp:1182-1185), savers are no-ops.
 */
#include <cstdio>
#include <cstring>
#include <string>
#include <new>
#include <cstdlib>
#include <unistd.h>
#include <cuda.h>
#include <cuda_runtime.h>
#include "helper_math.h"
#include "atmosphere/atmosphere.h"

bool load_texture_exr(float4**, std::string, int&, int&, bool) { return false; }
bool load_texture_exr_gpu(float4**, std::string, int&, int&, bool) { return false; }
bool save_texture_exr(float4*, std::string, const int, const int, bool) { return true; }
bool save_texture_png(float4*, std::string, const int, const int) { return true; }
void log(const char*, unsigned int) {}
void log(std::string, unsigned int) {}

static atmosphere* g_atmo = nullptr;

extern "C" int vptref_atmosphere_init(const char* module_dir, int use_constant_solar_spectrum, int use_ozone,
                                      int luminance_mode, int do_white_balance, float exposure, void* out_params)
{
    static_assert(sizeof(AtmosphereParameters) == 464, "AtmosphereParameters layout");
    cudaFree(0);                                     // make the runtime's primary context current for cuModuleLoad
    char cwd[4096];
    if (!getcwd(cwd, sizeof cwd)) return -1;
    if (chdir(module_dir) != 0) { fprintf(stderr, "[vptref] atmosphere: cannot enter %s\n", module_dir); return -2; }
    // A fresh model per call (init() appends to its spectra); the old one is kept alive for its textures.  The reference's
    // object has static storage (main.cpp: `atmosphere earth_atmosphere;`) and relies on that zero-initialisation:
    // copy_*_texture() destroys "the previous texture" whenever the handle member is non-zero (atmosphere.cpp:506).
    // Give the object the same zeroed storage here, otherwise a stale heap word is destroyed as a texture handle.
    void* storage = calloc(1, sizeof(atmosphere));
    g_atmo = new (storage) atmosphere();
    {
        // The reference's precompute kernels index their scattering buffers with unclamped texel coordinates
        // (atmosphere_kernels.cu:378-392: u = 1 maps to texel `size`, one row / slice past the end, up to ~0.5 MB beyond
        // the allocation), which faults or not depending on what the driver mapped next to the buffer.  The buffer
        // pointers are public members, so the harness re-homes the nine buffers into one zeroed slab with 2 MB of
        // slack on both sides of each: the stray reads then land in mapped zeros, as they do in a lucky run.
        AtmosphereParameters& P = g_atmo->atmosphere_parameters;
        const size_t small = (size_t)TRANSMITTANCE_TEXTURE_WIDTH * TRANSMITTANCE_TEXTURE_HEIGHT * sizeof(float4);
        const size_t irr = (size_t)IRRADIANCE_TEXTURE_WIDTH * IRRADIANCE_TEXTURE_HEIGHT * sizeof(float4);
        const size_t big = (size_t)SCATTERING_TEXTURE_WIDTH * SCATTERING_TEXTURE_HEIGHT * SCATTERING_TEXTURE_DEPTH * sizeof(float4);
        float4** slot[9] = { &P.transmittance_buffer, &P.delta_irradience_buffer, &P.irradiance_buffer, &P.delta_rayleigh_scattering_buffer,
                             &P.delta_mie_scattering_buffer, &P.scattering_buffer, &P.optional_mie_single_scattering_buffer,
                             &P.delta_scattering_density_buffer, &P.delta_multiple_scattering_buffer };
        const size_t bytes[9] = { small, irr, irr, big, big, big, big, big, big };
        const size_t slack = (size_t)2 << 20;
        size_t total = slack;
        for (int i = 0; i < 9; ++i) total += bytes[i] + slack;
        char* slab = nullptr;
        if (cudaMalloc(&slab, total) != cudaSuccess || cudaMemset(slab, 0, total) != cudaSuccess) { chdir(cwd); return -5; }
        size_t off = slack;
        for (int i = 0; i < 9; ++i) { cudaFree(*slot[i]); *slot[i] = reinterpret_cast<float4*>(slab + off); off += bytes[i] + slack; }
    }
    g_atmo->m_use_constant_solar_spectrum = use_constant_solar_spectrum != 0;
    g_atmo->m_use_ozone = use_ozone != 0;
    g_atmo->m_use_luminance = luminance_mode == 1 ? APPROXIMATE : luminance_mode == 2 ? PRECOMPUTED : NONE;
    g_atmo->m_do_white_balance = do_white_balance != 0;
    g_atmo->m_exposure = exposure;
    g_atmo->texture_folder = "";                     // no cached EXRs: always precompute
    atmosphere_error_t err = g_atmo->init();
    if (chdir(cwd) != 0) return -3;
    if (err != ATMO_NO_ERR) return -10 - (int)err;
    if (cudaDeviceSynchronize() != cudaSuccess) return -4;
    g_atmo->update_model();                          // main.cpp:1733-1738 (exposure / white balance refresh)
    memcpy(out_params, &g_atmo->atmosphere_parameters, sizeof(AtmosphereParameters));
    return 0;
}

/* Stage numbers are those of vpt_debug_bruneton_stage (include/vpt_b200.h).  Arguments as atmosphere::precompute passes them:
 *   direct irradiance        int BLEND                                                  (:953)
 *   single scattering        float4 (0, 0, B, B), mat3                                  (:982-984)
 *   scattering density       float4 (0, 0, 0, 0), order                                 (:1027-1029)
 *   indirect irradiance,     float4 (0, 1, 0, 0) where the kernels declare `int blend`: the int they read is the bit pattern of
 *   multiple scattering      0.0f = 0 (quirk Q17, :1056-1082); mat3; order.  blend = 1 passes an int 1 instead (the reference never
 *                            does; the test drives both implementations' blend paths with it).
 * lfr9 is the luminance-from-radiance array row-major, as the host builds it (:1247-1252); the kernels receive it through
 * mat3::toMatrix, whose storage is the transpose (matrix_math.h:686-692).  Grid: size / 8 + 1 blocks of 8x8 (x 8), as :923-980.
 * The buffers of params464 must stay readable wherever the reference's look-ups stray (the caller surrounds them with guards). */
static CUmodule g_stage_mod = nullptr;
static CUfunction g_stage_fn[6] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };

extern "C" int vptref_atmosphere_stage(const char* module_dir, int stage, const void* params464, int blend, const float* lfr9, int order)
{
    static const char* names[6] = { "calculate_transmittance", "calculate_direct_irradiance", "calculate_single_scattering",
                                    "calculate_scattering_density", "calculate_indirect_irradiance", "calculate_multiple_scattering" };
    if (stage < 0 || stage > 5 || !params464 || !lfr9 || !module_dir) return -1;
    cudaFree(0);
    if (!g_stage_mod) {
        const std::string path = std::string(module_dir) + "/atmosphere_kernels.ptx";
        if (cuModuleLoad(&g_stage_mod, path.c_str()) != CUDA_SUCCESS) { g_stage_mod = nullptr; return -2; }
    }
    if (!g_stage_fn[stage] && cuModuleGetFunction(&g_stage_fn[stage], g_stage_mod, names[stage]) != CUDA_SUCCESS) return -3;
    alignas(16) unsigned char params[464];
    memcpy(params, params464, sizeof params);
    float mat[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) mat[c * 3 + r] = lfr9[r * 3 + c];
    const int blend_int = blend;
    const float4 blend_single = make_float4(0.0f, 0.0f, (float)blend, (float)blend);
    const float4 blend_zero = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const float4 blend_later = make_float4(0.0f, 1.0f, 0.0f, 0.0f);
    const void* blend_later_arg = blend ? (const void*)&blend_int : (const void*)&blend_later;
    int ord = order;
    void* args[4] = { params, nullptr, nullptr, nullptr };
    unsigned gx = SCATTERING_TEXTURE_WIDTH / 8 + 1, gy = SCATTERING_TEXTURE_HEIGHT / 8 + 1, gz = SCATTERING_TEXTURE_DEPTH / 8 + 1, bz = 8;
    if (stage == 0) { gx = TRANSMITTANCE_TEXTURE_WIDTH / 8 + 1; gy = TRANSMITTANCE_TEXTURE_HEIGHT / 8 + 1; gz = 1; bz = 1; }
    if (stage == 1 || stage == 4) { gx = IRRADIANCE_TEXTURE_WIDTH / 8 + 1; gy = IRRADIANCE_TEXTURE_HEIGHT / 8 + 1; gz = 1; bz = 1; }
    switch (stage) {
    case 1: args[1] = (void*)&blend_int; break;
    case 2: args[1] = (void*)&blend_single; args[2] = mat; break;
    case 3: args[1] = (void*)&blend_zero; args[2] = &ord; break;
    case 4: case 5: args[1] = (void*)blend_later_arg; args[2] = mat; args[3] = &ord; break;
    default: break;
    }
    if (cuLaunchKernel(g_stage_fn[stage], gx, gy, gz, 8, 8, bz, 0, NULL, args, NULL) != CUDA_SUCCESS) return -4;
    if (cudaDeviceSynchronize() != cudaSuccess) return -5;
    return 0;
}
