// vpt_context.cpp -- C-ABI implementation (include/vpt_b200.h): context, render-pass scheduling,
// scene-table cache, and the host-side scene helpers.
//
// Scheduling of one vpt_render_passes(n) call on the caller's stream (no host synchronisation):
//   [once per (volumes, octree) pair]  k_prepare_scene
//   for each chunk of <= passes_per_chunk sampled passes:
//        memset(queue counters) -> k_bn_prepare -> k_generate -> k_trace<integrator, lean> (persistent) -> k_resolve<env>
//   passes beyond max_interactions / render == false: k_resolve (re-tonemap) + k_bn_advance
// which leaves every buffer named by Kernel_params in the state n reference launches would.
// vpt_render_adaptive runs the same rounds over the tiles that still hold an active pixel (k_generate_adaptive, k_resolve_adaptive),
// with k_adapt and one stream synchronisation at every convergence test.
#include "vpt_host.h"
#include "vdb_reader.h"
#include "image_io.h"

#include <cuda_runtime.h>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <sstream>
#include <string>
#include <algorithm>
#include <vector>

static thread_local std::string g_last_error;
namespace vpt { int fail_global(int code, const std::string& msg) { g_last_error = msg; return code; } }

static int fail(vpt_context* ctx, int code, const std::string& msg) {
    g_last_error = msg;
    if (ctx) ctx->err = msg;
    return code;
}
namespace vpt { int fail_ctx(vpt_context* ctx, int code, const std::string& msg) { return fail(ctx, code, msg); } }
#define VPT_CUDA(ctx, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    return fail(ctx, VPT_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); } while (0)

namespace vpt { FrameGeom make_frame_geom(const vpt_context* c, unsigned w, unsigned h); }
static vpt::FrameGeom make_geom(const vpt_context* c, unsigned w, unsigned h) { return vpt::make_frame_geom(c, w, h); }
vpt::FrameGeom vpt::make_frame_geom(const vpt_context* c, unsigned w, unsigned h) {
    vpt::FrameGeom g;
    g.width = (int)w; g.height = (int)h; g.n_ranks = c->n_ranks; g.rank = c->rank;
    if (c->n_ranks == 1) { g.stripe_h = (int)h > 0 ? (int)h : 1; g.local_rows = (int)h; }
    else {
        g.stripe_h = c->stripe_rows;
        const int stripes = ((int)h + g.stripe_h - 1) / g.stripe_h;
        const int per_rank = (stripes + c->n_ranks - 1) / c->n_ranks;
        g.local_rows = per_rank * g.stripe_h;
    }
    g.n_local = g.local_rows * g.width;
    return g;
}

extern "C" {

const char* vpt_version(void) { return "vpt-b200 0.1 (sm_90a wavefront build)"; }

// sizeof of every boundary struct, in VPT_ARG order then the auxiliary ones (no CUDA call: usable on a CPU-only host)
int vpt_abi_sizes(size_t* out, int n) {
    const size_t s[] = { sizeof(vpt_camera), sizeof(vpt_light_list), sizeof(vpt_gpu_vdb), sizeof(vpt_sphere), sizeof(vpt_geometry_list),
                         sizeof(vpt_bvhnode), sizeof(vpt_octnode), sizeof(vpt_atmosphere), sizeof(vpt_kernel_params),
                         sizeof(vpt_point_light), sizeof(vpt_vdb_info), sizeof(vpt_aabb) };
    const int m = (int)(sizeof(s) / sizeof(s[0]));
    for (int i = 0; i < n && i < m; ++i) out[i] = s[i];
    return m;
}

const char* vpt_last_error(const vpt_context* ctx) { return ctx ? ctx->err.c_str() : g_last_error.c_str(); }

static void free_context(vpt_context* c) {
    if (!c) return;
    cudaFree(c->d_scene); cudaFree(c->d_internal); cudaFree(c->d_leaf_list); cudaFree(c->d_leaf_indices); cudaFree(c->d_vrec);
    cudaFree(c->d_stats);
    if (c->h_pinned) cudaFreeHost(c->h_pinned);
    vpt_comm_destroy(c);
    for (auto& e : c->events) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
    cudaFree(c->d_queue_id); cudaFree(c->d_queue_org); cudaFree(c->d_bn_table);
    cudaFree(c->d_counters); cudaFree(c->d_queue); cudaFree(c->d_planeA); cudaFree(c->d_planeB); cudaFree(c->d_planeC); cudaFree(c->d_planeD);
    cudaFree(c->d_plane_tr); cudaFree(c->d_lg_planes); cudaFree(c->d_miss_mask); cudaFree(c->d_matte_map); cudaFree(c->d_matte_ids);
    cudaFree(c->d_adapt_stat); cudaFree(c->d_adapt_stopped); cudaFree(c->d_adapt_tiles);
    cudaFree(c->d_dn_cv); cudaFree(c->d_dn_yz); cudaFree(c->d_dn_layer);
    delete c;
}

int vpt_create(vpt_context** out) {
    if (!out) return fail(nullptr, VPT_ERR_INVALID, "vpt_create: null output pointer");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_create: no CUDA device (") + cudaGetErrorString(e) + "); this library has no CPU path");
    vpt_context* c = new vpt_context();
    // every failure below releases what was allocated so far (the context never escapes half-built)
#define VPT_CREATE(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
        const std::string m_ = std::string("vpt_create: " #call ": ") + cudaGetErrorString(e_); free_context(c); return fail(nullptr, VPT_ERR_CUDA, m_); } } while (0)
    VPT_CREATE(cudaGetDevice(&c->device));
    cudaDeviceProp prop;
    VPT_CREATE(cudaGetDeviceProperties(&prop, c->device));
    if (prop.major != 9 || prop.minor != 0) { std::string m = "vpt_create: device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + ", kernels are built for sm_90a only"; free_context(c); return fail(nullptr, VPT_ERR_UNSUPPORTED, m); }
    c->num_sms = prop.multiProcessorCount;
    c->l2_bytes = (size_t)prop.l2CacheSize;
    VPT_CREATE(cudaMalloc(&c->d_scene, sizeof(vpt::SceneAlloc)));      // the tables, then the render call's empty-ahead table
    VPT_CREATE(cudaMalloc(&c->d_counters, sizeof(unsigned) * 4));
    VPT_CREATE(cudaMalloc(&c->d_stats, sizeof(unsigned long long) * 16));
    VPT_CREATE(cudaMemset(c->d_stats, 0, sizeof(unsigned long long) * 16));
    VPT_CREATE(cudaHostAlloc((void**)&c->h_pinned, sizeof(int) * 8, cudaHostAllocDefault));
    // per-DEVICE kernel attributes (dynamic shared memory opt-in) and the occupancy the persistent grid is sized with
    VPT_CREATE(vpt::trace_kernels_init(c->max_ctas));
#undef VPT_CREATE
    *out = c;
    return VPT_OK;
}

void vpt_destroy(vpt_context* c) { free_context(c); }

int vpt_set_option(vpt_context* c, const char* key, int value) {
    if (!c || !key) return fail(c, VPT_ERR_INVALID, "vpt_set_option: null argument");
    const std::string k(key);
    if (k == "passes_per_chunk") { if (value < 0 || value > 64) return fail(c, VPT_ERR_INVALID, "passes_per_chunk must be 0 (automatic) or 1..64"); c->chunk_auto = value == 0; if (value) c->passes_per_chunk = value; }
    else if (k == "max_scratch_mb") { if (value < 64) return fail(c, VPT_ERR_INVALID, "max_scratch_mb must be >= 64"); c->max_scratch_bytes = (size_t)value << 20; }
    else if (k == "gather_async") { c->gather_async = value ? 1 : 0; }
    else if (k == "l2_sector_fetch") { c->l2_sector_fetch = value ? 1 : 0; }
    else if (k == "trace_slots") { if (value != 0 && value != 2 && value != 3) return fail(c, VPT_ERR_INVALID, "trace_slots must be 0 (by grid size), 2 or 3"); c->trace_slots = value; }
    else if (k == "ctas_per_sm") { if (value < 0 || value > 8) return fail(c, VPT_ERR_INVALID, "ctas_per_sm must be 0..8"); c->ctas_per_sm = value; }
    else if (k == "sched_min_lanes") { if (value < 0 || value > 32) return fail(c, VPT_ERR_INVALID, "sched_min_lanes must be 0 (by kernel) or 1..32"); c->sched_min_lanes = value; }
    else if (k == "debug_flags") { c->debug_flags = value; }
    else if (k == "generic_kernel") { c->force_generic = value ? 1 : 0; }
    else if (k == "count_stats") { c->count_stats = value ? 1 : 0; }
    else if (k == "profile") { c->profile = value ? 1 : 0; }
    else if (k == "miss_cull") { c->miss_cull = value ? 1 : 0; }
    else if (k == "empty_ahead") { c->empty_ahead = value ? 1 : 0; }
    else return fail(c, VPT_ERR_INVALID, "unknown option " + k);
    return VPT_OK;
}

int vpt_set_partition(vpt_context* c, int rank, int n_ranks, int stripe_rows) {
    if (!c || n_ranks < 1 || rank < 0 || rank >= n_ranks || stripe_rows < 1) return fail(c, VPT_ERR_INVALID, "vpt_set_partition: bad arguments");
    c->rank = rank; c->n_ranks = n_ranks; c->stripe_rows = stripe_rows;
    return VPT_OK;
}

long long vpt_local_pixels(const vpt_context* c, unsigned width, unsigned height) {
    if (!c) return -1;
    return make_geom(c, width, height).n_local;
}

int vpt_set_aov_buffers(vpt_context* c, float* d_alpha, float* d_volume_f3) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_aov_buffers: null context");
    c->aov_alpha = d_alpha; c->aov_volume = d_volume_f3;
    c->aov_active = false;          // both null: off from now on; otherwise the buffers take over at the next call with iteration == 0
    return VPT_OK;
}

int vpt_set_light_group_buffers(vpt_context* c, float* d_sun_f3, float* d_point_f3, float* d_emission_f3, float* d_environment_f3) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_light_group_buffers: null context");
    c->lg_out[0] = d_sun_f3; c->lg_out[1] = d_point_f3; c->lg_out[2] = d_emission_f3; c->lg_out[3] = d_environment_f3;
    c->lg_active = false;           // all null: off from now on; otherwise the buffers take over at the next call with iteration == 0
    return VPT_OK;
}

static_assert(vpt::kDeepMaxSlices == VPT_DEEP_MAX_SLICES, "deep slice limit");

int vpt_set_deep_buffers(vpt_context* c, float* d_slices_f4, unsigned n_slices, const float* h_bounds) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_deep_buffers: null context");
    vpt::DeepSlices d;
    if (d_slices_f4) {
        if (n_slices < 1 || n_slices > VPT_DEEP_MAX_SLICES)
            return fail(c, VPT_ERR_INVALID, "vpt_set_deep_buffers: n_slices must be in 1.." + std::to_string(VPT_DEEP_MAX_SLICES) + ", got " + std::to_string(n_slices));
        if ((uintptr_t)d_slices_f4 % 16 != 0)
            return fail(c, VPT_ERR_INVALID, "vpt_set_deep_buffers: the slice buffer must be 16-byte aligned (the kernels move float4)");
        if (!h_bounds) return fail(c, VPT_ERR_INVALID, "vpt_set_deep_buffers: null bounds");
        for (unsigned k = 0; k <= n_slices; ++k) {
            const float z = h_bounds[k];
            const std::string at = "vpt_set_deep_buffers: bound " + std::to_string(k) + " (" + std::to_string(z) + ") ";
            if (std::isnan(z) || z < 0.0f) return fail(c, VPT_ERR_INVALID, at + "must be a number >= 0");
            if (std::isinf(z) && k < n_slices) return fail(c, VPT_ERR_INVALID, at + "is infinite: only the last bound may be +inf");
            if (k > 0 && !(z > h_bounds[k - 1])) return fail(c, VPT_ERR_INVALID, at + "must be greater than the bound before it");
            d.z[k] = z;
        }
        d.out = reinterpret_cast<float4*>(d_slices_f4);
        d.n = (int)n_slices;
    }
    c->deep_req = d;
    c->deep_active = false;         // null: off from now on; otherwise the slices take over at the next call with iteration == 0
    return VPT_OK;
}

static_assert(vpt::kMatteMax == VPT_MATTE_MAX, "matte limit");

int vpt_set_instance_mattes(vpt_context* c, float* d_mattes_f4, unsigned n_mattes, const int* h_matte_of_instance, unsigned n_instances,
                            int sphere_matte) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_instance_mattes: null context");
    vpt::Mattes m;
    std::vector<int8_t> map;
    if (d_mattes_f4) {
        if (n_mattes < 1 || n_mattes > VPT_MATTE_MAX)
            return fail(c, VPT_ERR_INVALID, "vpt_set_instance_mattes: n_mattes must be in 1.." + std::to_string(VPT_MATTE_MAX) + ", got " + std::to_string(n_mattes));
        if ((uintptr_t)d_mattes_f4 % 16 != 0)
            return fail(c, VPT_ERR_INVALID, "vpt_set_instance_mattes: the matte buffer must be 16-byte aligned (the kernels move float4)");
        if (!h_matte_of_instance && n_instances > 0) return fail(c, VPT_ERR_INVALID, "vpt_set_instance_mattes: null instance map");
        const auto in_range = [&](int k) { return k >= -1 && k < (int)n_mattes; };
        map.resize(n_instances);
        for (unsigned i = 0; i < n_instances; ++i) {
            const int k = h_matte_of_instance[i];
            if (!in_range(k))
                return fail(c, VPT_ERR_INVALID, "vpt_set_instance_mattes: instance " + std::to_string(i) + " maps to " + std::to_string(k) +
                                                ", outside -1.." + std::to_string((int)n_mattes - 1));
            map[i] = (int8_t)k;
        }
        if (!in_range(sphere_matte))
            return fail(c, VPT_ERR_INVALID, "vpt_set_instance_mattes: sphere_matte " + std::to_string(sphere_matte) + " is outside -1.." +
                                            std::to_string((int)n_mattes - 1));
        m.out = reinterpret_cast<float4*>(d_mattes_f4);
        m.n = (int)n_mattes;
        m.n_ids = n_instances;
        m.sphere = sphere_matte;
    }
    c->matte_req = m;
    c->matte_map_req.swap(map);
    c->matte_active = false;        // null: off from now on; otherwise the mattes take over at the next call with iteration == 0
    return VPT_OK;
}

int vpt_set_render_region(vpt_context* c, unsigned x0, unsigned y0, unsigned x1, unsigned y1) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_render_region: null context");
    c->region_req[0] = x0; c->region_req[1] = y0; c->region_req[2] = x1; c->region_req[3] = y1;   // checked and taken at the next iteration-0 call
    return VPT_OK;
}

static_assert(vpt::kProjPerspective == VPT_PROJECTION_PERSPECTIVE && vpt::kProjEquirect == VPT_PROJECTION_EQUIRECT &&
              vpt::kProjOds == VPT_PROJECTION_ODS, "projection kinds");
static_assert(vpt::kOdsLeft == VPT_ODS_LEFT && vpt::kOdsRight == VPT_ODS_RIGHT && vpt::kOdsOverUnder == VPT_ODS_OVER_UNDER, "ODS layouts");

// the field of view of a panorama (equirectangular, or each eye of an ODS frame), in float radians
static int panorama_fov(vpt_context* c, const char* fn, double hfov_deg, double vfov_deg, vpt::Projection* p) {
    if (!(hfov_deg > 0.0 && hfov_deg <= 360.0)) return fail(c, VPT_ERR_INVALID, std::string(fn) + ": hfov_deg must be in (0, 360], got " + std::to_string(hfov_deg));
    if (!(vfov_deg > 0.0 && vfov_deg <= 180.0)) return fail(c, VPT_ERR_INVALID, std::string(fn) + ": vfov_deg must be in (0, 180], got " + std::to_string(vfov_deg));
    p->hfov = (float)(hfov_deg * (3.14159265358979323846 / 180.0));
    p->vfov = (float)(vfov_deg * (3.14159265358979323846 / 180.0));
    return VPT_OK;
}

int vpt_set_projection(vpt_context* c, int kind, double hfov_deg, double vfov_deg) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_projection: null context");
    vpt::Projection p;
    if (kind == VPT_PROJECTION_EQUIRECT) {
        const int rc = panorama_fov(c, "vpt_set_projection", hfov_deg, vfov_deg, &p);
        if (rc != VPT_OK) return rc;
        p.kind = kind;
    } else if (kind == VPT_PROJECTION_ODS) {
        return fail(c, VPT_ERR_INVALID, "vpt_set_projection: VPT_PROJECTION_ODS needs its options: use vpt_set_projection_ods");
    } else if (kind != VPT_PROJECTION_PERSPECTIVE) {
        return fail(c, VPT_ERR_INVALID, "vpt_set_projection: unknown projection kind " + std::to_string(kind));
    }
    c->proj_req = p;                // taken at the next iteration-0 call
    return VPT_OK;
}

void vpt_ods_options_defaults(vpt_ods_options* opt) {
    if (!opt) return;
    opt->ipd = 0.064f; opt->layout = VPT_ODS_OVER_UNDER; opt->pole_merge_from_deg = 60.0f; opt->pole_merge_to_deg = 75.0f;
}

int vpt_set_projection_ods(vpt_context* c, double hfov_deg, double vfov_deg, const vpt_ods_options* opt) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_projection_ods: null context");
    vpt_ods_options o;
    vpt_ods_options_defaults(&o);
    if (opt) o = *opt;
    vpt::Projection p;
    const int rc = panorama_fov(c, "vpt_set_projection_ods", hfov_deg, vfov_deg, &p);
    if (rc != VPT_OK) return rc;
    if (!(std::isfinite(o.ipd) && o.ipd >= 0.0f)) return fail(c, VPT_ERR_INVALID, "vpt_set_projection_ods: ipd must be finite and >= 0, got " + std::to_string(o.ipd));
    if (o.layout != VPT_ODS_LEFT && o.layout != VPT_ODS_RIGHT && o.layout != VPT_ODS_OVER_UNDER)
        return fail(c, VPT_ERR_INVALID, "vpt_set_projection_ods: unknown layout " + std::to_string(o.layout));
    const double from = o.pole_merge_from_deg, to = o.pole_merge_to_deg;
    if (!(from >= 0.0 && from <= to && to <= 90.0))
        return fail(c, VPT_ERR_INVALID, "vpt_set_projection_ods: the pole merge needs 0 <= from <= to <= 90, got from " + std::to_string(from) + ", to " + std::to_string(to));
    p.kind = VPT_PROJECTION_ODS;
    vpt::OdsParams d;
    d.hfov = p.hfov; d.vfov = p.vfov;
    d.half_ipd = (float)((double)o.ipd / 2.0);
    d.layout = o.layout;
    d.merge_from = (float)(from * (3.14159265358979323846 / 180.0));
    d.merge_to = (float)(to * (3.14159265358979323846 / 180.0));
    d.inv_span = to > from ? (float)(1.0 / ((to - from) * (3.14159265358979323846 / 180.0))) : 0.0f;   // from == to: k is a step, inv_span unread
    c->proj_req = p; c->ods_req = d;          // taken at the next iteration-0 call
    return VPT_OK;
}

int vpt_set_camera_motion(vpt_context* c, const vpt_camera* shutter_close) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_camera_motion: null context");
    if (!shutter_close) { c->motion_req = false; return VPT_OK; }          // taken at the next iteration-0 call
    const struct { const char* name; vpt_f3 v; } fields[] = {
        { "origin", shutter_close->origin }, { "lower_left_corner", shutter_close->lower_left_corner }, { "horizontal", shutter_close->horizontal },
        { "vertical", shutter_close->vertical }, { "u", shutter_close->u }, { "v", shutter_close->v } };
    for (const auto& f : fields)
        if (!std::isfinite(f.v.x) || !std::isfinite(f.v.y) || !std::isfinite(f.v.z))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_camera_motion: shutter_close.") + f.name + " is not finite");
    vpt::CameraMotion m;
    m.origin = shutter_close->origin; m.lower_left_corner = shutter_close->lower_left_corner; m.horizontal = shutter_close->horizontal;
    m.vertical = shutter_close->vertical; m.u = shutter_close->u; m.v = shutter_close->v;
    c->motion_close_req = m; c->motion_req = true;
    return VPT_OK;
}

int vpt_set_motion_vectors(vpt_context* c, float* d_vectors_f3, const vpt_camera* target) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_motion_vectors: null context");
    vpt::MotionVectors m;
    if (d_vectors_f3) {
        if (!target) return fail(c, VPT_ERR_INVALID, "vpt_set_motion_vectors: null target camera");
        const struct { const char* name; vpt_f3 v; } fields[] = {
            { "origin", target->origin }, { "lower_left_corner", target->lower_left_corner }, { "horizontal", target->horizontal },
            { "vertical", target->vertical } };
        for (const auto& f : fields)
            if (!std::isfinite(f.v.x) || !std::isfinite(f.v.y) || !std::isfinite(f.v.z))
                return fail(c, VPT_ERR_INVALID, std::string("vpt_set_motion_vectors: target.") + f.name + " is not finite");
        m.out = reinterpret_cast<float3*>(d_vectors_f3);
        m.origin = target->origin; m.lower_left_corner = target->lower_left_corner; m.horizontal = target->horizontal; m.vertical = target->vertical;
    }
    c->mv_req = m;
    c->mv_active = false;           // null: off from now on; otherwise buffer and target take over at the next call with iteration == 0
    return VPT_OK;
}

int vpt_set_collision_aovs(vpt_context* c, float* d_position_f4, float* d_normal_f3, float* d_albedo_f3, float gradient_step) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_collision_aovs: null context");
    if (d_normal_f3 && !(std::isfinite(gradient_step) && gradient_step > 0.0f))
        return fail(c, VPT_ERR_INVALID, "vpt_set_collision_aovs: gradient_step must be finite and > 0 with a normal buffer (got " + std::to_string(gradient_step) + ")");
    vpt::CollisionAovs a;
    a.position = reinterpret_cast<float4*>(d_position_f4); a.normal = reinterpret_cast<float3*>(d_normal_f3); a.albedo = reinterpret_cast<float3*>(d_albedo_f3);
    a.step = gradient_step;
    c->ca_req = a;
    c->ca_active = false;           // all null: off from now on; otherwise the buffers take over at the next call with iteration == 0
    return VPT_OK;
}

static_assert(vpt::kCryptoMaxEntries == VPT_CRYPTO_MAX_ENTRIES, "Cryptomatte capacity");

int vpt_set_cryptomatte(vpt_context* c, uint32_t* d_state, unsigned capacity) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_cryptomatte: null context");
    vpt::Cryptomatte m;
    if (d_state) {
        if (capacity < 1 || capacity > VPT_CRYPTO_MAX_ENTRIES)
            return fail(c, VPT_ERR_INVALID, "vpt_set_cryptomatte: capacity must be in 1.." + std::to_string(VPT_CRYPTO_MAX_ENTRIES) + ", got " + std::to_string(capacity));
        if ((uintptr_t)d_state % 4 != 0) return fail(c, VPT_ERR_INVALID, "vpt_set_cryptomatte: the state buffer must be 4-byte aligned (the kernels move uint32)");
        m.state = d_state;
        m.cap = (int)capacity;
    }
    c->crypto_req = m;
    c->crypto_active = false;       // null: off from now on; otherwise the state takes over at the next call with iteration == 0
    return VPT_OK;
}

// MurmurHash3_x86_32 (Austin Appleby's public-domain hash) of the bytes with seed 0
uint32_t vpt_cryptomatte_hash(const char* name, size_t len, float* id_out) {
    const uint8_t* data = reinterpret_cast<const uint8_t*>(name);
    if (!data) len = 0;
    const uint32_t c1 = 0xcc9e2d51u, c2 = 0x1b873593u;
    auto rotl = [](uint32_t x, int r) { return (x << r) | (x >> (32 - r)); };
    uint32_t h = 0u;
    const size_t n4 = len / 4;
    for (size_t i = 0; i < n4; ++i) {
        uint32_t k = (uint32_t)data[4 * i] | (uint32_t)data[4 * i + 1] << 8 | (uint32_t)data[4 * i + 2] << 16 | (uint32_t)data[4 * i + 3] << 24;
        k *= c1; k = rotl(k, 15); k *= c2;
        h ^= k; h = rotl(h, 13); h = h * 5u + 0xe6546b64u;
    }
    const uint8_t* tail = data + 4 * n4;
    uint32_t k = 0u;
    switch (len & 3u) {
    case 3: k ^= (uint32_t)tail[2] << 16; [[fallthrough]];
    case 2: k ^= (uint32_t)tail[1] << 8; [[fallthrough]];
    case 1: k ^= tail[0]; k *= c1; k = rotl(k, 15); k *= c2; h ^= k;
    }
    h ^= (uint32_t)len;
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    if (id_out) {
        // the Cryptomatte float: no denormal, infinity or NaN (bit 23 flipped where the exponent is 0 or 255)
        const uint32_t e = (h >> 23) & 0xffu;
        const uint32_t bits = (e == 0u || e == 255u) ? h ^ (1u << 23) : h;
        memcpy(id_out, &bits, sizeof(bits));
    }
    return h;
}

int vpt_set_sample_offset(vpt_context* c, uint32_t offset) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_set_sample_offset: null context");
    c->sample_offset_req = offset;  // taken at the next iteration-0 call
    return VPT_OK;
}

int vpt_unpermute(vpt_context* c, const void* d_gathered, void* d_full, unsigned width, unsigned height, int elem_bytes, void* stream) {
    if (!c || !d_gathered || !d_full || elem_bytes <= 0 || (elem_bytes & 3)) return fail(c, VPT_ERR_INVALID, "vpt_unpermute: bad arguments");
    const vpt::FrameGeom g = make_geom(c, width, height);
    VPT_CUDA(c, vpt::launch_unpermute(d_gathered, d_full, g, elem_bytes, (cudaStream_t)stream));
    c->launches++;
    return VPT_OK;
}

int vpt_invalidate_scene(vpt_context* c) {
    if (!c) return VPT_ERR_INVALID;
    c->cached_volumes = 0; c->cached_root = 0; c->cached_generation = 0;
    return VPT_OK;
}

int vpt_get_stats(vpt_context* c, unsigned long long* launches, unsigned* last_queue_count) {
    if (!c) return VPT_ERR_INVALID;
    if (launches) *launches = c->launches;
    if (last_queue_count) VPT_CUDA(c, cudaMemcpy(last_queue_count, c->d_counters, sizeof(unsigned), cudaMemcpyDeviceToHost));
    return VPT_OK;
}

// Scratch of one round: the ray queue and plane A per sample, then either planes B, C (and D) per sample (wide records) or the tr plane
// per pixel (compact records).  A change of record layout reallocates, so the scratch never holds another layout's planes.  Light groups
// traced by a generic kernel also need their 12 float planes per sample, and the instance mattes their id plane, which are kept once grown.
static int ensure_frame_buffers(vpt_context* c, size_t n_samples, size_t n_pixels, bool wide, bool planeD, bool groups, bool mattes) {
    if (n_samples > c->cap_samples || wide != c->cap_wide || planeD != c->cap_planeD) {
        cudaFree(c->d_queue); cudaFree(c->d_planeA); cudaFree(c->d_planeB); cudaFree(c->d_planeC); cudaFree(c->d_planeD);
        cudaFree(c->d_queue_id); cudaFree(c->d_queue_org);
        c->d_queue = c->d_planeA = c->d_planeB = c->d_planeC = c->d_planeD = c->d_queue_org = nullptr; c->d_queue_id = nullptr;
        c->cap_samples = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_queue, n_samples * sizeof(float4)));
        VPT_CUDA(c, cudaMalloc(&c->d_queue_id, n_samples * sizeof(uint2)));
        VPT_CUDA(c, cudaMalloc(&c->d_queue_org, n_samples * sizeof(float4)));
        VPT_CUDA(c, cudaMalloc(&c->d_planeA, n_samples * sizeof(float4)));
        if (wide) {
            VPT_CUDA(c, cudaMalloc(&c->d_planeB, n_samples * sizeof(float4)));
            VPT_CUDA(c, cudaMalloc(&c->d_planeC, n_samples * sizeof(float4)));
        }
        if (planeD) VPT_CUDA(c, cudaMalloc(&c->d_planeD, n_samples * sizeof(float4)));
        c->cap_samples = n_samples; c->cap_wide = wide; c->cap_planeD = planeD;
    }
    if (groups && n_samples > c->cap_lg_samples) {
        cudaFree(c->d_lg_planes); c->d_lg_planes = nullptr; c->cap_lg_samples = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_lg_planes, n_samples * 12 * sizeof(float)));
        c->cap_lg_samples = n_samples;
    }
    if (mattes && n_samples > c->cap_matte_samples) {
        cudaFree(c->d_matte_ids); c->d_matte_ids = nullptr; c->cap_matte_samples = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_matte_ids, n_samples * sizeof(uint32_t)));
        c->cap_matte_samples = n_samples;
    }
    if (!wide && n_pixels > c->cap_tr) {
        cudaFree(c->d_plane_tr); c->d_plane_tr = nullptr; c->cap_tr = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_plane_tr, n_pixels * sizeof(float)));
        c->cap_tr = n_pixels;
    }
    return VPT_OK;
}

} // extern "C"

namespace {
// What one render call works with once the parameter block is unpacked: vpt_render_passes and vpt_render_adaptive share it (frame_setup).
struct FramePlan {
    vpt::FrameArgs fa;
    vpt_atmosphere atmo;                  // the caller's AtmosphereParameters
    vpt::TraceKernel trace = vpt::TK_GENERIC_3;
    vpt::ResolveKey resolve;
    int trace_ctas = 0, chunk = 1, bn_limit = 0;
    unsigned n_sampled = 0;               // how many of the requested passes sample (the rest only re-tonemap)
    vpt::AovBuffers aov;                  // the active compositing AOVs (both null: off)
    vpt::LightGroups lg;                  // the active light groups (every output null: off; planes null: a lean kernel traces the frame)
    vpt::DeepSlices deep;                 // the active deep slices (out null: off)
    vpt::Mattes mattes;                   // the active instance mattes (out null: off)
    vpt::MatteIds matte_ids;              // their id plane, for the trace kernel (the mattes' and the Cryptomatte's)
    vpt::Cryptomatte crypto;              // the active Cryptomatte (state null: off)
    vpt::MotionVectors mv;                // the active motion vectors (out null: off)
    vpt::CollisionAovs ca;                // the active collision AOVs (all three outputs null: off)
    bool collisions() const { return ca.position || ca.normal || ca.albedo; }
    bool region = false;                  // a render region is active: the region kernels over rg
    vpt::RenderRegion rg;
    vpt::Projection proj;                 // the frame's projection: the equirectangular kernels when equirect(proj)
    bool motion = false;                  // camera motion: the motion generate kernels with the shutter-close pose mo
    vpt::CameraMotion mo;
    const vpt::CameraMotion* motion_arg() const { return motion ? &mo : nullptr; }
    vpt::OdsParams ods;                   // the ODS projection when ods(proj): the ODS generate kernels
    const vpt::OdsParams* ods_arg() const { return vpt::ods(proj) ? &ods : nullptr; }
};

// Under option "profile": brackets the launches of fn with CUDA events of the given kind (0 generate, 1 trace, 2 resolve, 3 blue noise).
template <class F>
cudaError_t timed(vpt_context* c, cudaStream_t stream, int kind, F&& fn) {
    if (!c->profile) return fn();
    vpt_context::Ev ev; ev.kind = kind;
    cudaEventCreate(&ev.a); cudaEventCreate(&ev.b);
    cudaEventRecord(ev.a, stream);
    cudaError_t e = fn();
    cudaEventRecord(ev.b, stream);
    c->events.push_back(ev);
    return e;
}
} // namespace

static bool byte_ranges_overlap(const void* a, size_t na, const void* b, size_t nb) {
    if (!a || !b) return false;
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

// The AOV buffers may not share a byte with a Kernel_params output buffer or with each other (n = local pixels).
static int check_aov_buffers(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    const struct { const char* name; vpt_devptr_t p; size_t bytes; } outs[] = {
        { "accum_buffer", kp.accum_buffer, 12 * n }, { "depth_buffer", kp.depth_buffer, 4 * n }, { "cost_buffer", kp.cost_buffer, 12 * n },
        { "raw_buffer", kp.raw_buffer, 16 * n }, { "display_buffer", kp.display_buffer, 4 * n } };
    for (const auto& o : outs) {
        const void* p = (const void*)(uintptr_t)o.p;
        if (byte_ranges_overlap(c->aov_alpha, 4 * n, p, o.bytes))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_aov_buffers: the alpha buffer overlaps Kernel_params.") + o.name);
        if (byte_ranges_overlap(c->aov_volume, 12 * n, p, o.bytes))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_aov_buffers: the volume buffer overlaps Kernel_params.") + o.name);
    }
    if (byte_ranges_overlap(c->aov_alpha, 4 * n, c->aov_volume, 12 * n))
        return fail(c, VPT_ERR_INVALID, "vpt_set_aov_buffers: the alpha buffer and the volume buffer overlap");
    return VPT_OK;
}

// The light-group buffers may not share a byte with a Kernel_params output buffer, an AOV buffer or each other (n = local pixels).
static int check_light_group_buffers(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    static const char* const names[4] = { "sun", "point", "emission", "environment" };
    const struct { const char* name; const void* p; size_t bytes; } others[] = {
        { "Kernel_params.accum_buffer", (const void*)(uintptr_t)kp.accum_buffer, 12 * n }, { "Kernel_params.depth_buffer", (const void*)(uintptr_t)kp.depth_buffer, 4 * n },
        { "Kernel_params.cost_buffer", (const void*)(uintptr_t)kp.cost_buffer, 12 * n }, { "Kernel_params.raw_buffer", (const void*)(uintptr_t)kp.raw_buffer, 16 * n },
        { "Kernel_params.display_buffer", (const void*)(uintptr_t)kp.display_buffer, 4 * n },
        { "the alpha AOV buffer", c->aov_alpha, 4 * n }, { "the volume AOV buffer", c->aov_volume, 12 * n } };
    for (int k = 0; k < 4; ++k) {
        for (const auto& o : others)
            if (byte_ranges_overlap(c->lg_out[k], 12 * n, o.p, o.bytes))
                return fail(c, VPT_ERR_INVALID, std::string("vpt_set_light_group_buffers: the ") + names[k] + " buffer overlaps " + o.name);
        for (int j = 0; j < k; ++j)
            if (byte_ranges_overlap(c->lg_out[k], 12 * n, c->lg_out[j], 12 * n))
                return fail(c, VPT_ERR_INVALID, std::string("vpt_set_light_group_buffers: the ") + names[j] + " buffer and the " + names[k] + " buffer overlap");
    }
    return VPT_OK;
}

// The slice buffer may not share a byte with a Kernel_params output buffer, an AOV buffer or a light-group buffer (n = local pixels).
static int check_deep_buffers(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    const struct { const char* name; const void* p; size_t bytes; } others[] = {
        { "Kernel_params.accum_buffer", (const void*)(uintptr_t)kp.accum_buffer, 12 * n }, { "Kernel_params.depth_buffer", (const void*)(uintptr_t)kp.depth_buffer, 4 * n },
        { "Kernel_params.cost_buffer", (const void*)(uintptr_t)kp.cost_buffer, 12 * n }, { "Kernel_params.raw_buffer", (const void*)(uintptr_t)kp.raw_buffer, 16 * n },
        { "Kernel_params.display_buffer", (const void*)(uintptr_t)kp.display_buffer, 4 * n },
        { "the alpha AOV buffer", c->aov_alpha, 4 * n }, { "the volume AOV buffer", c->aov_volume, 12 * n },
        { "the sun light-group buffer", c->lg_out[0], 12 * n }, { "the point light-group buffer", c->lg_out[1], 12 * n },
        { "the emission light-group buffer", c->lg_out[2], 12 * n }, { "the environment light-group buffer", c->lg_out[3], 12 * n } };
    for (const auto& o : others)
        if (byte_ranges_overlap(c->deep_req.out, 16 * n * (size_t)c->deep_req.n, o.p, o.bytes))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_deep_buffers: the slice buffer overlaps ") + o.name);
    return VPT_OK;
}

// The matte buffer may not share a byte with a Kernel_params output buffer, an AOV, light-group or deep-slice buffer (n = local pixels).
static int check_matte_buffers(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    const struct { const char* name; const void* p; size_t bytes; } others[] = {
        { "Kernel_params.accum_buffer", (const void*)(uintptr_t)kp.accum_buffer, 12 * n }, { "Kernel_params.depth_buffer", (const void*)(uintptr_t)kp.depth_buffer, 4 * n },
        { "Kernel_params.cost_buffer", (const void*)(uintptr_t)kp.cost_buffer, 12 * n }, { "Kernel_params.raw_buffer", (const void*)(uintptr_t)kp.raw_buffer, 16 * n },
        { "Kernel_params.display_buffer", (const void*)(uintptr_t)kp.display_buffer, 4 * n },
        { "the alpha AOV buffer", c->aov_alpha, 4 * n }, { "the volume AOV buffer", c->aov_volume, 12 * n },
        { "the sun light-group buffer", c->lg_out[0], 12 * n }, { "the point light-group buffer", c->lg_out[1], 12 * n },
        { "the emission light-group buffer", c->lg_out[2], 12 * n }, { "the environment light-group buffer", c->lg_out[3], 12 * n },
        { "the deep slice buffer", c->deep_req.out, 16 * n * (size_t)c->deep_req.n } };
    for (const auto& o : others)
        if (byte_ranges_overlap(c->matte_req.out, 16 * n * (size_t)c->matte_req.n, o.p, o.bytes))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_instance_mattes: the matte buffer overlaps ") + o.name);
    return VPT_OK;
}

// The motion-vector buffer may not share a byte with a Kernel_params output buffer, an AOV, light-group, deep-slice or matte buffer
// (n = local pixels).
static int check_motion_vector_buffer(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    const struct { const char* name; const void* p; size_t bytes; } others[] = {
        { "Kernel_params.accum_buffer", (const void*)(uintptr_t)kp.accum_buffer, 12 * n }, { "Kernel_params.depth_buffer", (const void*)(uintptr_t)kp.depth_buffer, 4 * n },
        { "Kernel_params.cost_buffer", (const void*)(uintptr_t)kp.cost_buffer, 12 * n }, { "Kernel_params.raw_buffer", (const void*)(uintptr_t)kp.raw_buffer, 16 * n },
        { "Kernel_params.display_buffer", (const void*)(uintptr_t)kp.display_buffer, 4 * n },
        { "the alpha AOV buffer", c->aov_alpha, 4 * n }, { "the volume AOV buffer", c->aov_volume, 12 * n },
        { "the sun light-group buffer", c->lg_out[0], 12 * n }, { "the point light-group buffer", c->lg_out[1], 12 * n },
        { "the emission light-group buffer", c->lg_out[2], 12 * n }, { "the environment light-group buffer", c->lg_out[3], 12 * n },
        { "the deep slice buffer", c->deep_req.out, 16 * n * (size_t)c->deep_req.n },
        { "the matte buffer", c->matte_req.out, 16 * n * (size_t)c->matte_req.n } };
    for (const auto& o : others)
        if (byte_ranges_overlap(c->mv_req.out, 12 * n, o.p, o.bytes))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_motion_vectors: the motion-vector buffer overlaps ") + o.name);
    return VPT_OK;
}

// The collision-AOV buffers may not share a byte with a Kernel_params output buffer, an AOV, light-group, deep-slice, matte or motion-vector
// buffer, or with each other (n = local pixels).
// The Cryptomatte state may not share a byte with a Kernel_params output buffer or any layer buffer (n = local pixels).
static int check_cryptomatte_buffer(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    const vpt::CollisionAovs& ca = c->ca_req;
    const struct { const char* name; const void* p; size_t bytes; } others[] = {
        { "Kernel_params.accum_buffer", (const void*)(uintptr_t)kp.accum_buffer, 12 * n }, { "Kernel_params.depth_buffer", (const void*)(uintptr_t)kp.depth_buffer, 4 * n },
        { "Kernel_params.cost_buffer", (const void*)(uintptr_t)kp.cost_buffer, 12 * n }, { "Kernel_params.raw_buffer", (const void*)(uintptr_t)kp.raw_buffer, 16 * n },
        { "Kernel_params.display_buffer", (const void*)(uintptr_t)kp.display_buffer, 4 * n },
        { "the alpha AOV buffer", c->aov_alpha, 4 * n }, { "the volume AOV buffer", c->aov_volume, 12 * n },
        { "the sun light-group buffer", c->lg_out[0], 12 * n }, { "the point light-group buffer", c->lg_out[1], 12 * n },
        { "the emission light-group buffer", c->lg_out[2], 12 * n }, { "the environment light-group buffer", c->lg_out[3], 12 * n },
        { "the deep slice buffer", c->deep_req.out, 16 * n * (size_t)c->deep_req.n },
        { "the matte buffer", c->matte_req.out, 16 * n * (size_t)c->matte_req.n },
        { "the motion-vector buffer", c->mv_req.out, 12 * n },
        { "the collision position buffer", ca.position, 16 * n }, { "the collision normal buffer", ca.normal, 12 * n },
        { "the collision albedo buffer", ca.albedo, 12 * n } };
    const size_t bytes = 4 * n * (2 + 2 * (size_t)c->crypto_req.cap);
    for (const auto& o : others)
        if (byte_ranges_overlap(c->crypto_req.state, bytes, o.p, o.bytes))
            return fail(c, VPT_ERR_INVALID, std::string("vpt_set_cryptomatte: the state buffer overlaps ") + o.name);
    return VPT_OK;
}

static int check_collision_aov_buffers(vpt_context* c, const vpt_kernel_params& kp, size_t n) {
    const vpt::CollisionAovs& ca = c->ca_req;
    const struct { const char* name; const void* p; size_t bytes; } others[] = {
        { "Kernel_params.accum_buffer", (const void*)(uintptr_t)kp.accum_buffer, 12 * n }, { "Kernel_params.depth_buffer", (const void*)(uintptr_t)kp.depth_buffer, 4 * n },
        { "Kernel_params.cost_buffer", (const void*)(uintptr_t)kp.cost_buffer, 12 * n }, { "Kernel_params.raw_buffer", (const void*)(uintptr_t)kp.raw_buffer, 16 * n },
        { "Kernel_params.display_buffer", (const void*)(uintptr_t)kp.display_buffer, 4 * n },
        { "the alpha AOV buffer", c->aov_alpha, 4 * n }, { "the volume AOV buffer", c->aov_volume, 12 * n },
        { "the sun light-group buffer", c->lg_out[0], 12 * n }, { "the point light-group buffer", c->lg_out[1], 12 * n },
        { "the emission light-group buffer", c->lg_out[2], 12 * n }, { "the environment light-group buffer", c->lg_out[3], 12 * n },
        { "the deep slice buffer", c->deep_req.out, 16 * n * (size_t)c->deep_req.n },
        { "the matte buffer", c->matte_req.out, 16 * n * (size_t)c->matte_req.n },
        { "the motion-vector buffer", c->mv_req.out, 12 * n } };
    const struct { const char* name; const void* p; size_t bytes; } mine[3] = {
        { "position", ca.position, 16 * n }, { "normal", ca.normal, 12 * n }, { "albedo", ca.albedo, 12 * n } };
    for (int k = 0; k < 3; ++k) {
        for (const auto& o : others)
            if (byte_ranges_overlap(mine[k].p, mine[k].bytes, o.p, o.bytes))
                return fail(c, VPT_ERR_INVALID, std::string("vpt_set_collision_aovs: the ") + mine[k].name + " buffer overlaps " + o.name);
        for (int j = 0; j < k; ++j)
            if (byte_ranges_overlap(mine[k].p, mine[k].bytes, mine[j].p, mine[j].bytes))
                return fail(c, VPT_ERR_INVALID, std::string("vpt_set_collision_aovs: the ") + mine[j].name + " buffer and the " + mine[k].name + " buffer overlap");
    }
    return VPT_OK;
}

// The preamble of a render call of n_passes passes: validation, scene-table refresh, trace-kernel choice, chunk size and scratch buffers.
static int frame_setup(vpt_context* c, void* const params[VPT_NUM_ARGS], unsigned n_passes, cudaStream_t stream, FramePlan& plan) {
    vpt::FrameArgs& fa = plan.fa;
    memcpy(&fa.cam, params[VPT_ARG_CAMERA], sizeof(vpt_camera));
    memcpy(&fa.lights, params[VPT_ARG_LIGHTS], sizeof(vpt_light_list));
    memcpy(&fa.kp, params[VPT_ARG_KERNEL_PARAMS], sizeof(vpt_kernel_params));
    vpt_devptr_t d_volumes, d_sphere, d_root;
    memcpy(&d_volumes, params[VPT_ARG_VOLUMES], 8);
    memcpy(&d_sphere, params[VPT_ARG_SPHERE], 8);
    memcpy(&d_root, params[VPT_ARG_OCTREE], 8);
    const vpt_kernel_params& kp = fa.kp;

    // environment_type == 0: the caller's AtmosphereParameters (scalars + the four precomputed look-up textures)
    vpt_atmosphere& atmo = plan.atmo;
    memcpy(&atmo, params[VPT_ARG_ATMOSPHERE], sizeof(vpt_atmosphere));
    if (c->n_ranks > 1 && (kp.resolution.x > 65535u || kp.resolution.y > 65535u)) return fail(c, VPT_ERR_UNSUPPORTED, "a partitioned frame is limited to 65535 x 65535 pixels");
    const bool vol_integ = (kp.integrator != 0);             // vol_integrator always ends on the precomputed sky (:1752)
    const bool sky_env = (kp.environment_type == 0) || vol_integ;
    const bool samples = kp.render && kp.iteration < kp.max_interactions;
    if (sky_env && samples &&
        (!atmo.transmittance_texture || !atmo.scattering_texture || !atmo.irradiance_texture || !atmo.single_mie_scattering_texture))
        return fail(c, VPT_ERR_INVALID, "environment_type == 0 / integrator != 0 need the four precomputed atmosphere textures in AtmosphereParameters");
    if (vol_integ && samples && kp.environment_type == 0 && kp.sky_mult > 0.0f &&
        (!kp.env_func_tex || !kp.env_cdf_tex || !kp.env_marginal_func_tex || !kp.env_marginal_cdf_tex || kp.env_sample_tex_res < 2))
        return fail(c, VPT_ERR_INVALID, "integrator != 0 with environment_type == 0 needs the env sampling tables (env_*_tex, env_sample_tex_res) in Kernel_params");
    if (vol_integ && samples && kp.environment_type != 0 && !kp.env_tex)
        return fail(c, VPT_ERR_INVALID, "environment_type != 0 needs Kernel_params.env_tex");
    if (!d_volumes || !d_sphere || !d_root) return fail(c, VPT_ERR_INVALID, "volumes / sphere / octree device pointer is null");
    if (!kp.accum_buffer || !kp.depth_buffer || !kp.cost_buffer || !kp.display_buffer || !kp.raw_buffer || !kp.blue_noise_buffer)
        return fail(c, VPT_ERR_INVALID, "Kernel_params output buffer pointer is null");
    if (kp.resolution.x == 0 || kp.resolution.y == 0) return fail(c, VPT_ERR_INVALID, "resolution is zero");
    // render region: the one set last takes over at a call with iteration == 0, checked against this call's resolution first
    const unsigned* reg = kp.iteration == 0 ? c->region_req : c->region_cur;
    const bool region = (reg[0] | reg[1] | reg[2] | reg[3]) != 0;
    if (region) {
        const std::string r = "render region (" + std::to_string(reg[0]) + ", " + std::to_string(reg[1]) + ", " + std::to_string(reg[2]) + ", " +
                              std::to_string(reg[3]) + "): ";
        if (reg[0] >= reg[2]) return fail(c, VPT_ERR_INVALID, r + "x0 must be < x1");
        if (reg[1] >= reg[3]) return fail(c, VPT_ERR_INVALID, r + "y0 must be < y1");
        if (reg[2] > kp.resolution.x) return fail(c, VPT_ERR_INVALID, r + "x1 exceeds Kernel_params.resolution.x = " + std::to_string(kp.resolution.x));
        if (reg[3] > kp.resolution.y) return fail(c, VPT_ERR_INVALID, r + "y1 exceeds Kernel_params.resolution.y = " + std::to_string(kp.resolution.y));
    }
    // projection: the one set last takes over at a call with iteration == 0
    const vpt::Projection& proj = kp.iteration == 0 ? c->proj_req : c->proj_cur;
    if (vpt::equirect(proj) && fa.cam.lens_radius != 0.0f)
        return fail(c, VPT_ERR_UNSUPPORTED, "the equirectangular projection has no lens: camera.lens_radius must be 0 (got " + std::to_string(fa.cam.lens_radius) + ")");
    // camera motion: the shutter-close pose set last takes over at a call with iteration == 0
    const bool motion = kp.iteration == 0 ? c->motion_req : c->motion_cur;
    if (motion && vpt::equirect(proj))
        return fail(c, VPT_ERR_UNSUPPORTED, "camera motion (vpt_set_camera_motion) is not supported with the equirectangular projection");
    const vpt::OdsParams& ods = kp.iteration == 0 ? c->ods_req : c->ods_cur;
    if (vpt::ods(proj)) {
        if (fa.cam.lens_radius != 0.0f)
            return fail(c, VPT_ERR_UNSUPPORTED, "the ODS projection has no lens: camera.lens_radius must be 0 (got " + std::to_string(fa.cam.lens_radius) + ")");
        if (motion) return fail(c, VPT_ERR_UNSUPPORTED, "camera motion (vpt_set_camera_motion) is not supported with the ODS projection");
        if (ods.layout == vpt::kOdsOverUnder && (kp.resolution.y & 1u))
            return fail(c, VPT_ERR_UNSUPPORTED, "the over-under ODS layout needs an even height, got " + std::to_string(kp.resolution.y));
    }
    // motion vectors: the buffer and target set last take over at a call with iteration == 0 (the rule of the AOVs)
    const bool vectors = c->mv_active || (kp.iteration == 0 && c->mv_req.out);
    if (vectors && (vpt::equirect(proj) || vpt::ods(proj)))
        return fail(c, VPT_ERR_UNSUPPORTED, "motion vectors (vpt_set_motion_vectors) are not supported with the equirectangular or ODS projection");
    // collision AOVs: the same rule
    const bool collisions = c->ca_active || (kp.iteration == 0 && (c->ca_req.position || c->ca_req.normal || c->ca_req.albedo));
    if (collisions && (vpt::equirect(proj) || vpt::ods(proj)))
        return fail(c, VPT_ERR_UNSUPPORTED, "collision AOVs (vpt_set_collision_aovs) are not supported with the equirectangular or ODS projection");

    if (c->brick_pool || c->cell_table) {
        // brick / cell mode read volume 0 from their own copy of the grid: only the lean case of the direct integrator is built for them,
        // and that copy must have the dimensions of volume 0's density grid -- the samplers index it with the scene's coordinates
        vpt::SceneEntry ent;
        const bool ok = vpt::scene_registry_find(d_root, &ent) && ent.n == 1 && !(ent.any_flags & 1u) && !(kp.emission_scale > 0.0f) &&
                        fa.lights.num_lights == 0 && kp.integrator == 0 && !c->force_generic;
        if (!ok) return fail(c, VPT_ERR_UNSUPPORTED, "brick / cell mode needs a vpt_octree_build scene of ONE volume without colour grid, the direct integrator, no emission and no point lights");
        if (c->brick_pool && c->cell_table) return fail(c, VPT_ERR_INVALID, "brick mode and cell mode are both set");
        const int* have = c->brick_pool ? c->brick_dims : c->cell_dims;
        if (have[0] != ent.dim0[0] || have[1] != ent.dim0[1] || have[2] != ent.dim0[2]) {
            auto dims = [](const int* d) { return std::to_string(d[0]) + "x" + std::to_string(d[1]) + "x" + std::to_string(d[2]); };
            return fail(c, VPT_ERR_INVALID, std::string(c->brick_pool ? "the brick pool (vpt_set_brick_volume)" : "the cell table (vpt_set_cell_volume)") +
                                            " was set with dimensions " + dims(have) + ", volume 0's density grid is " + dims(ent.dim0));
        }
    }

    // ---- scene tables ---------------------------------------------------------------------------------------
    // Octrees built by vpt_octree_build are registered with their flat tables and instance count: nothing is read
    // back and nothing blocks.  A foreign (reference-built, pointer-linked) octree is flattened on the device and
    // its instance count read back (4 bytes, one stream synchronisation) when the pointers change or a frame starts.
    {
        vpt::SceneEntry ent;
        const bool registered = vpt::scene_registry_find(d_root, &ent);
        if (registered && ent.device != c->device) return fail(c, VPT_ERR_INVALID, "octree was built on another device");
        const bool key_changed = c->cached_volumes != d_volumes || c->cached_root != d_root || c->cached_generation != (registered ? ent.generation : 0ull);
        // iteration == 0 starts a new frame: every scene edit of the reference application resets it (main.cpp:1667-1780), so
        // refreshing the cheap tables there also covers buffers that were rewritten or reallocated at the same address
        if (key_changed || kp.iteration == 0) {
            if (registered) {
                if ((size_t)ent.n > c->cap_vrec) {
                    cudaFree(c->d_vrec); c->d_vrec = nullptr; c->cap_vrec = 0;
                    VPT_CUDA(c, cudaMalloc(&c->d_vrec, sizeof(vpt::VolumeRec) * (size_t)ent.n));
                    c->cap_vrec = (size_t)ent.n;
                }
                vpt::SceneTables hdr;
                for (int a = 0; a < 3; ++a) { hdr.root_pmin[a] = ent.root6[a]; hdr.root_pmax[a] = ent.root6[3 + a]; }
                hdr.max_extinction = ent.max_extinction; hdr.min_extinction = ent.min_extinction;
                hdr.num_volumes = ent.n; hdr.single_volume = ent.n == 1 ? 1 : 0;
                hdr.internal = ent.d_internal; hdr.leaf_list = ent.d_leaf_list; hdr.leaf_indices = ent.d_leaf_indices; hdr.volumes = c->d_vrec; hdr.leaf_nodes = nullptr;
                VPT_CUDA(c, vpt::launch_prepare_volumes(reinterpret_cast<const vpt_gpu_vdb*>(d_volumes), hdr, c->d_scene, c->d_vrec, stream));
                c->scene_single_volume = ent.n == 1;
                c->scene_instances = ent.n;
            } else {
                if (!c->d_internal) {
                    VPT_CUDA(c, cudaMalloc(&c->d_internal, sizeof(vpt::OctInternal) * vpt::kOctInternalNodes));
                    VPT_CUDA(c, cudaMalloc(&c->d_leaf_list, sizeof(uint2) * vpt::kOctLeaves));
                    VPT_CUDA(c, cudaMalloc(&c->d_leaf_indices, sizeof(int) * vpt::kOctLeaves * VPT_OCT_MAX_VOLUMES));
                }
                if (c->cap_vrec < VPT_OCT_MAX_VOLUMES) {
                    cudaFree(c->d_vrec); c->d_vrec = nullptr; c->cap_vrec = 0;
                    VPT_CUDA(c, cudaMalloc(&c->d_vrec, sizeof(vpt::VolumeRec) * VPT_OCT_MAX_VOLUMES));
                    c->cap_vrec = VPT_OCT_MAX_VOLUMES;
                }
                VPT_CUDA(c, vpt::launch_prepare_scene(reinterpret_cast<const vpt_gpu_vdb*>(d_volumes), reinterpret_cast<const vpt_octnode*>(d_root),
                                                      c->d_scene, c->d_internal, c->d_leaf_list, c->d_leaf_indices, c->d_vrec, VPT_OCT_MAX_VOLUMES, stream));
                static_assert(offsetof(vpt::SceneTables, single_volume) == offsetof(vpt::SceneTables, num_volumes) + sizeof(int), "instance count, then single_volume");
                VPT_CUDA(c, cudaMemcpyAsync(c->h_pinned, reinterpret_cast<const char*>(c->d_scene) + offsetof(vpt::SceneTables, num_volumes), 2 * sizeof(int),
                                            cudaMemcpyDeviceToHost, stream));
                VPT_CUDA(c, cudaStreamSynchronize(stream));
                c->scene_instances = c->h_pinned[0];
                c->scene_single_volume = c->h_pinned[1] != 0;
            }
            c->launches++;
            c->cached_volumes = d_volumes; c->cached_root = d_root; c->cached_generation = registered ? ent.generation : 0ull;
        }
        // the call's empty-ahead table (option "empty_ahead"), from the octree just refreshed: k_generate and the lean k_trace stage it
        VPT_CUDA(c, timed(c, stream, 0, [&] { return vpt::launch_empty_ahead(c->d_scene, c->empty_ahead, stream); }));
        c->launches++;
    }
    // "lean" = nothing but one volume, sun and environment in play (the headline configuration)
    const bool lean = c->scene_single_volume && !(kp.emission_scale > 0.0f) && fa.lights.num_lights == 0 && kp.integrator == 0 && !c->force_generic;

    fa.sphere = reinterpret_cast<const vpt_sphere*>(d_sphere);
    fa.scene = c->d_scene;
    fa.geom = make_geom(c, kp.resolution.x, kp.resolution.y);

    // how many of the requested passes actually sample (render_kernel.cu:2254)
    unsigned n_sampled = 0;
    if (kp.render && kp.iteration < kp.max_interactions) {
        const unsigned left = kp.max_interactions - kp.iteration;
        n_sampled = n_passes < left ? n_passes : left;
    }

    // passes fused per generate/trace/resolve round: 32 by default; a small local frame (multi-GPU shard, low resolution)
    // takes up to 64 so the fixed per-round cost and the persistent kernel's tail are paid half as often; always capped so
    // the per-round scratch (ray queue + sample planes: 56 B per sample with compact records, 88 B or 104 B with wide ones) stays under
    // max_scratch_bytes.  Compact records: an HDRI frame traced by a lean kernel, which then finishes each ray's environment term
    // itself.  A frame that ends on the precomputed sky needs wide records and env_pos (plane D: k_resolve<1/2> evaluate the sky from
    // them), and so does the generic kernel (the texture look-up in its service round cost it more than k_resolve<0> saved).
    // light groups, decided before the record layout: registered buffers take over at the first call of a frame (iteration == 0) and are
    // checked on every call.  They force wide records (a lean kernel's L is then the sun group, in plane B); a generic kernel keeps its
    // group sums in 12 more float planes per sample
    const bool groups = c->lg_active || (kp.iteration == 0 && (c->lg_out[0] || c->lg_out[1] || c->lg_out[2] || c->lg_out[3]));
    if (groups) {
        int rc = check_light_group_buffers(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
    }
    const bool group_planes = groups && !lean;
    // instance mattes, decided with the groups: registered mattes take over at the first call of a frame (iteration == 0) and are checked on
    // every call.  The trace kernel writes one id per sample (4 B more per sample)
    const bool mattes = c->matte_active || (kp.iteration == 0 && c->matte_req.out);
    if (mattes) {
        if (c->brick_pool || c->cell_table) return fail(c, VPT_ERR_UNSUPPORTED, "instance mattes (vpt_set_instance_mattes) are not supported in brick or cell mode");
        if (c->matte_req.n_ids != (uint32_t)c->scene_instances)
            return fail(c, VPT_ERR_INVALID, "vpt_set_instance_mattes: the map covers " + std::to_string(c->matte_req.n_ids) + " instances, the scene has " +
                                            std::to_string(c->scene_instances));
        int rc = check_matte_buffers(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
    }
    // the Cryptomatte: the same rule, and the same id plane (`ids`: the trace kernel writes it for either)
    const bool crypto = c->crypto_active || (kp.iteration == 0 && c->crypto_req.state);
    if (crypto) {
        if (c->brick_pool || c->cell_table) return fail(c, VPT_ERR_UNSUPPORTED, "the Cryptomatte (vpt_set_cryptomatte) is not supported in brick or cell mode");
        int rc = check_cryptomatte_buffer(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
    }
    const bool ids = mattes || crypto;
    const bool deep = c->deep_active || (kp.iteration == 0 && c->deep_req.out);
    // an active exchange whose block carries deep slices or mattes: this call's count must be the exported one, or k_binned_publish would
    // store another layout.  Checked before any state changes and before the call enqueues its first flag signal
    if (c->p2p_on) {
        const struct { bool on; unsigned have, exported; const char *what, *setter; } bins[2] = {
            { deep, (unsigned)c->deep_req.n, c->p2p_slices, "deep slices", "vpt_set_deep_buffers" },
            { mattes, (unsigned)c->matte_req.n, c->p2p_mattes, "mattes", "vpt_set_instance_mattes" } };
        for (const auto& b : bins)
            if (b.on && b.exported && b.have != b.exported)
                return fail(c, VPT_ERR_INVALID, std::string("the peer exchange block was exported with ") + std::to_string(b.exported) + " " + b.what +
                                                " (vpt_comm_p2p_export_binned), this call's " + b.what + " (" + b.setter + ") are " + std::to_string(b.have) +
                                                "; set " + std::to_string(b.exported) + ", or tear the exchange down (vpt_comm_destroy) and export again");
    }
    const bool planeD = sky_env;
    const bool wide = sky_env || !lean || groups;
    int chunk = c->passes_per_chunk;
    if (c->chunk_auto) chunk = (size_t)fa.geom.n_local <= ((size_t)1 << 20) ? 64 : 32;
    {
        const size_t per_sample = (wide ? 88 + (planeD ? 16 : 0) : 56) + (group_planes ? 48 : 0) + (ids ? 4 : 0);
        const size_t fit = c->max_scratch_bytes / (per_sample * (size_t)(fa.geom.n_local > 0 ? fa.geom.n_local : 1));
        if ((size_t)chunk > fit) chunk = fit < 1 ? 1 : (int)fit;
    }
    if (n_sampled) {
        const size_t per_chunk = (size_t)fa.geom.n_local * (size_t)(n_sampled < (unsigned)chunk ? n_sampled : (unsigned)chunk);
        int rc = ensure_frame_buffers(c, per_chunk, (size_t)fa.geom.n_local, wide, planeD, group_planes, ids);
        if (rc != VPT_OK) return rc;
    }
    if (c->cap_chunk < chunk) {
        cudaFree(c->d_bn_table); c->d_bn_table = nullptr;
        VPT_CUDA(c, cudaMalloc(&c->d_bn_table, sizeof(float2) * 65536 * (size_t)chunk));
        c->cap_chunk = chunk;
    }
    fa.queue_dir = c->d_queue; fa.queue_id = c->d_queue_id; fa.queue_aux = c->d_queue_org; fa.thin_lens = (fa.cam.lens_radius != 0.0f || motion || vpt::ods(proj)) ? 1 : 0;
    fa.bn_table = c->d_bn_table; fa.debug_flags = c->debug_flags;
    fa.queue_count = c->d_counters; fa.queue_head = c->d_counters + 1;
    fa.planeA = c->d_planeA;
    fa.planeB = wide ? c->d_planeB : nullptr; fa.planeC = wide ? c->d_planeC : nullptr; fa.planeD = planeD ? c->d_planeD : nullptr;
    fa.plane_tr = wide ? nullptr : c->d_plane_tr;
    // pixels no jitter can take to the root box or the sphere (pinhole and equirectangular HDRI frames that sample): k_miss_cull marks them once per call, and
    // k_generate / k_resolve skip their sample records.  Frames that end on the precomputed sky keep every record (see resolve_pixel), and
    // so do motion frames: the cull assumes one camera per strip, and k_resolve rebuilds a culled sample without the lens loop.  ODS frames
    // cull with k_miss_cull_ods, whose bound takes in every origin' of a strip.
    fa.miss_mask = nullptr;
    if (c->miss_cull && n_sampled && !sky_env && fa.cam.lens_radius == 0.0f && !motion && fa.geom.n_local > 0) {
        if ((size_t)fa.geom.n_local > c->cap_miss_mask) {
            cudaFree(c->d_miss_mask); c->d_miss_mask = nullptr; c->cap_miss_mask = 0;
            VPT_CUDA(c, cudaMalloc(&c->d_miss_mask, (size_t)fa.geom.n_local));
            c->cap_miss_mask = (size_t)fa.geom.n_local;
        }
        fa.miss_mask = c->d_miss_mask;
    }

    // rays per lane: 3 by default; 2 (more warps per SM) when warps in flight matter more than rays per warp -- a lean frame, whose
    // stepping loop is bound by the latency of its look-ups even when they hit L2, or a look-up that is a chain of cache misses: a density
    // grid that cannot live in L2 (every look-up a DRAM round trip) or long per-leaf instance lists (dependent loads) (DESIGN.md section 4).
    int slots = 3;
    if (c->cell_table) slots = 2;
    else if (!vol_integ && !c->brick_pool) {
        if (c->trace_slots) slots = c->trace_slots;
        else if (lean) slots = 2;
        else {
            vpt::SceneEntry ent;
            if (vpt::scene_registry_find(d_root, &ent) && (ent.max_grid_bytes > 2ull * c->l2_bytes || ent.n >= 64)) slots = 2;
        }
    }
    const vpt::TraceKernel trace = vpt::pick_trace_kernel(c->brick_pool != nullptr, c->cell_table != nullptr, vol_integ, lean, group_planes, slots, ids);
    fa.sched_min_lanes = c->sched_min_lanes > 0 ? c->sched_min_lanes : vpt::trace_sched_min_lanes(trace);
    int ctas_per_sm = c->ctas_per_sm > 0 ? c->ctas_per_sm : c->max_ctas[trace];
    if (ctas_per_sm < 1) ctas_per_sm = 1;

    fa.counters = c->count_stats ? c->d_stats : nullptr;
    fa.cell_table = c->cell_table; fa.cell_nx = c->cell_dims[0]; fa.cell_ny = c->cell_dims[1]; fa.cell_nz = c->cell_dims[2];
    const unsigned long long frame_px = (unsigned long long)kp.resolution.x * kp.resolution.y;
    plan.trace = trace; plan.trace_ctas = c->num_sms * ctas_per_sm;
    c->last_trace_rays = vpt::trace_rays_per_lane(trace);
    plan.chunk = chunk; plan.n_sampled = n_sampled;
    plan.bn_limit = frame_px < 65536ull ? (int)frame_px : 65536;

    // compositing AOVs: registered buffers take over at the first call of a frame (iteration == 0) and are checked on every call
    if (c->aov_active || (kp.iteration == 0 && (c->aov_alpha || c->aov_volume))) {
        int rc = check_aov_buffers(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
        c->aov_active = true;
        plan.aov.alpha = c->aov_alpha; plan.aov.volume = reinterpret_cast<float3*>(c->aov_volume);
    }
    if (groups) {
        c->lg_active = true;
        for (int k = 0; k < 4; ++k) plan.lg.out[k] = reinterpret_cast<float3*>(c->lg_out[k]);
        if (group_planes) { plan.lg.planes = c->d_lg_planes; plan.lg.stride = (unsigned long long)c->cap_lg_samples; }
    }
    plan.resolve.sky = sky_env ? (vol_integ ? 2 : 1) : 0;
    plan.resolve.aov = plan.aov.alpha || plan.aov.volume;
    plan.resolve.groups = plan.lg.out[0] || plan.lg.out[1] || plan.lg.out[2] || plan.lg.out[3];
    // deep slices: the buffer, its slice count and bounds take over at the first call of a frame (iteration == 0), checked on every call
    if (deep) {
        int rc = check_deep_buffers(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
        c->deep_active = true;
        plan.deep = c->deep_req;
    }
    plan.resolve.deep = plan.deep.out != nullptr;
    if (vectors) {
        int rc = check_motion_vector_buffer(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
        c->mv_active = true;
        plan.mv = c->mv_req;
    }
    if (collisions) {
        int rc = check_collision_aov_buffers(c, kp, (size_t)fa.geom.n_local);
        if (rc != VPT_OK) return rc;
        c->ca_active = true;
        plan.ca = c->ca_req;
        plan.ca.brick_pool = c->brick_pool;
        for (int a = 0; a < 3; ++a) plan.ca.brick_dims[a] = c->brick_dims[a];
    }
    // instance mattes: the map goes to the device when they take over
    if (mattes) {
        if (!c->matte_active) {
            const size_t n = c->matte_map_req.size();
            if (n > c->cap_matte_map) {
                cudaFree(c->d_matte_map); c->d_matte_map = nullptr; c->cap_matte_map = 0;
                VPT_CUDA(c, cudaMalloc(&c->d_matte_map, n));
                c->cap_matte_map = n;
            }
            if (n) VPT_CUDA(c, cudaMemcpyAsync(c->d_matte_map, c->matte_map_req.data(), n, cudaMemcpyHostToDevice, stream));
            c->matte_active = true;
        }
        plan.mattes = c->matte_req;
        plan.mattes.map = c->d_matte_map;
        plan.mattes.id = c->d_matte_ids;
    }
    if (crypto) {
        c->crypto_active = true;
        plan.crypto = c->crypto_req;
        plan.crypto.id = c->d_matte_ids;
    }
    if (ids) plan.matte_ids.id = c->d_matte_ids;
    plan.resolve.mattes = mattes;
    plan.proj = proj;
    plan.ods = ods;
    plan.motion = motion;
    plan.mo = kp.iteration == 0 ? c->motion_close_req : c->motion_close_cur;
    fa.sample_offset = kp.iteration == 0 ? c->sample_offset_req : c->sample_offset_cur;
    if (kp.iteration == 0) {
        memcpy(c->region_cur, c->region_req, sizeof(c->region_cur)); c->proj_cur = c->proj_req; c->ods_cur = c->ods_req;
        c->motion_cur = c->motion_req; c->motion_close_cur = c->motion_close_req;
        c->sample_offset_cur = c->sample_offset_req;
    }
    plan.region = region;
    if (region) plan.rg = vpt::region_geometry(fa.geom, (int)reg[0], (int)reg[1], (int)reg[2], (int)reg[3]);
    return VPT_OK;
}

// the rank-local sources of the exchange layers: depth and the frame's active AOVs and light groups (null: not active)
static vpt::LayerSources layer_sources(const FramePlan& plan) {
    vpt::LayerSources s;
    s.src[vpt::XL_DEPTH] = reinterpret_cast<const float*>(plan.fa.kp.depth_buffer);
    s.src[vpt::XL_ALPHA] = plan.aov.alpha;
    s.src[vpt::XL_VOLUME] = reinterpret_cast<const float*>(plan.aov.volume);
    for (int k = 0; k < vpt::kLightGroups; ++k) s.src[vpt::XL_SUN + k] = reinterpret_cast<const float*>(plan.lg.out[k]);
    return s;
}

// The arguments of k_generate* and k_trace*: they read Kernel_params.iteration only as the Philox stream key, so they get the stream
// iteration (vpt_set_sample_offset's offset added, 32-bit wrap) in its place and keep their code; every other kernel keeps the caller's.
static vpt::FrameArgs stream_args(const vpt::FrameArgs& fa) {
    vpt::FrameArgs s = fa;
    s.kp.iteration = fa.kp.iteration + fa.sample_offset;
    return s;
}

// the frame's trace kernel over whatever k_generate queued for a chunk of np passes
static cudaError_t launch_trace_of(vpt_context* c, const FramePlan& plan, unsigned np, cudaStream_t stream) {
    vpt::FrameArgs fa = stream_args(plan.fa);
    fa.n_passes = (int)np;
    return vpt::launch_trace(fa, plan.trace, plan.atmo, plan.lg, plan.matte_ids, c->brick_pool, c->brick_dims, plan.trace_ctas, stream);
}

extern "C" {

int vpt_render_passes(vpt_context* c, void* const params[VPT_NUM_ARGS], unsigned n_passes, void* stream_) {
    if (!c || !params) return fail(c, VPT_ERR_INVALID, "vpt_render_passes: null argument");
    for (int i = 0; i < VPT_NUM_ARGS; ++i) if (!params[i]) return fail(c, VPT_ERR_INVALID, "vpt_render_passes: params[" + std::to_string(i) + "] is null");
    if (n_passes == 0) return VPT_OK;
    cudaStream_t stream = (cudaStream_t)stream_;
    {
        // an adaptive frame is final: its pixels hold different sample counts, so no later pass can continue it
        vpt_kernel_params kp0;
        memcpy(&kp0, params[VPT_ARG_KERNEL_PARAMS], sizeof(vpt_kernel_params));
        if (c->adaptive_accum && kp0.accum_buffer == c->adaptive_accum) {
            if (kp0.iteration > 0)
                return fail(c, VPT_ERR_INVALID, "vpt_render_passes: accum_buffer holds a finished adaptive frame (vpt_render_adaptive), which cannot be "
                                                "continued; start a new frame with iteration == 0");
            c->adaptive_accum = 0;
        }
    }

    FramePlan plan;
    { int rc = frame_setup(c, params, n_passes, stream, plan); if (rc != VPT_OK) return rc; }
    vpt::FrameArgs& fa = plan.fa;
    const vpt_kernel_params& kp = fa.kp;
    const unsigned n_sampled = plan.n_sampled;
    const int chunk = plan.chunk, bn_limit = plan.bn_limit;
    if (c->p2p_on && ((int)kp.resolution.x != c->p2p_w || (int)kp.resolution.y != c->p2p_h))
        return fail(c, VPT_ERR_INVALID, "the peer exchange block was exported for another frame size (vpt_comm_p2p_export)");
    { int rc = vpt::comm_p2p_begin(c, stream); if (rc != VPT_OK) return rc; }      // multi-GPU peer exchange: this rank's frame may be overwritten from here on
    const uint32_t it0 = kp.iteration;
    // a render region runs the region kernels over R's tiles / pixels; the scratch layout, the trace kernel and the blue noise are the same
    const bool region = plan.region;
    const vpt::RenderRegion& rg = plan.rg;
    if (fa.miss_mask) {
        VPT_CUDA(c, timed(c, stream, 0, [&] { return region ? vpt::launch_miss_cull_region(fa, c->d_miss_mask, rg, plan.proj, stream, plan.ods_arg())
                                                            : vpt::launch_miss_cull(fa, c->d_miss_mask, plan.proj, stream, plan.ods_arg()); }));
        c->launches++;
    }
    unsigned done = 0;
    while (done < n_sampled) {
        const unsigned np = (n_sampled - done) < (unsigned)chunk ? (n_sampled - done) : (unsigned)chunk;
        fa.kp.iteration = it0 + done;
        VPT_CUDA(c, timed(c, stream, 3, [&] { return vpt::launch_bn_prepare((void*)kp.blue_noise_buffer, c->d_bn_table, (int)np, bn_limit, c->d_counters, stream); }));   // jitter table + advance + queue reset
        VPT_CUDA(c, timed(c, stream, 0, [&] { return region ? vpt::launch_generate_region(stream_args(fa), (int)np, rg, plan.proj, plan.motion_arg(), plan.ods_arg(), stream)
                                                            : vpt::launch_generate(stream_args(fa), (int)np, plan.proj, plan.motion_arg(), plan.ods_arg(), stream); }));
        VPT_CUDA(c, timed(c, stream, 1, [&] { return launch_trace_of(c, plan, np, stream); }));
        const bool last = (done + np == n_passes);
        if (c->gather_pending) { int rc = vpt::comm_before_accum_write(c, stream); if (rc != VPT_OK) return rc; }
        vpt::PeerFrames peers;
        if (last) { int rc = vpt::comm_p2p_peers(c, stream, &peers); if (rc != VPT_OK) return rc; }
        if (plan.mv.out) {
            VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_motion_vectors(fa, plan.mv, (int)np, 1, region ? &rg : nullptr, nullptr, plan.motion_arg(), stream); }));
            c->launches++;
        }
        if (plan.collisions()) {
            VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_collision_aovs(fa, plan.ca, (int)np, 1, region ? &rg : nullptr, nullptr, plan.motion_arg(), stream); }));
            c->launches++;
        }
        if (plan.crypto.state) {
            VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_cryptomatte(fa, plan.crypto, (int)np, 1, region ? &rg : nullptr, nullptr, stream); }));
            c->launches++;
        }
        VPT_CUDA(c, timed(c, stream, 2, [&] {
            return region ? vpt::launch_resolve_region(fa, plan.resolve, plan.atmo, (int)np, 1, last ? 1 : 0, last ? &peers : nullptr, plan.aov, plan.lg, plan.deep, plan.mattes, rg,
                                                       plan.proj, stream, plan.ods_arg())
                          : vpt::launch_resolve(fa, plan.resolve, plan.atmo, (int)np, 1, last ? 1 : 0, last ? &peers : nullptr, plan.aov, plan.lg, plan.deep, plan.mattes,
                                                plan.proj, stream, plan.ods_arg()); }));
        c->launches += 4 + (plan.resolve.deep ? 1 : 0) + (plan.resolve.mattes ? 1 : 0);   // deep slices and mattes: one more resolve kernel each
        done += np;
    }
    if (n_sampled < n_passes) {
        // passes that no longer sample: WHITE / re-tonemap semantics of the kernel tail
        fa.kp.iteration = it0 + n_sampled;
        if (c->gather_pending) { int rc = vpt::comm_before_accum_write(c, stream); if (rc != VPT_OK) return rc; }
        vpt::PeerFrames peers;
        { int rc = vpt::comm_p2p_peers(c, stream, &peers); if (rc != VPT_OK) return rc; }
        if (plan.mv.out) {
            VPT_CUDA(c, vpt::launch_motion_vectors(fa, plan.mv, (int)(n_passes - n_sampled), 0, region ? &rg : nullptr, nullptr, plan.motion_arg(), stream));
            c->launches++;
        }
        if (plan.collisions()) {
            VPT_CUDA(c, vpt::launch_collision_aovs(fa, plan.ca, (int)(n_passes - n_sampled), 0, region ? &rg : nullptr, nullptr, plan.motion_arg(), stream));
            c->launches++;
        }
        if (plan.crypto.state) {
            VPT_CUDA(c, vpt::launch_cryptomatte(fa, plan.crypto, (int)(n_passes - n_sampled), 0, region ? &rg : nullptr, nullptr, stream));
            c->launches++;
        }
        if (region) VPT_CUDA(c, vpt::launch_resolve_region(fa, plan.resolve, plan.atmo, (int)(n_passes - n_sampled), 0, 1, &peers, plan.aov, plan.lg, plan.deep, plan.mattes, rg,
                                                           plan.proj, stream, plan.ods_arg()));
        else VPT_CUDA(c, vpt::launch_resolve(fa, plan.resolve, plan.atmo, (int)(n_passes - n_sampled), 0, 1, &peers, plan.aov, plan.lg, plan.deep, plan.mattes, plan.proj, stream, plan.ods_arg()));
        VPT_CUDA(c, vpt::launch_bn_advance((void*)kp.blue_noise_buffer, (int)(n_passes - n_sampled), bn_limit, stream));
        c->launches += 2 + (plan.resolve.deep ? 1 : 0) + (plan.resolve.mattes ? 1 : 0);
    }
    // multi-GPU: the one exchange of the path.  Peer-memory mode: the last resolve above already stored every pixel into every rank's
    // frame, the exported layers follow; publish and wait for the peers.  NCCL mode: all-gather of the rank-local frame into the caller's
    // full-frame buffers.
    { int rc = vpt::comm_p2p_layers(c, fa.geom, region ? &rg : nullptr, layer_sources(plan), stream, plan.mv.out); if (rc != VPT_OK) return rc; }
    { int rc = vpt::comm_p2p_binned(c, fa.geom, region ? &rg : nullptr, plan.deep.out, plan.mattes.out, stream); if (rc != VPT_OK) return rc; }
    { int rc = vpt::comm_p2p_end(c, stream); if (rc != VPT_OK) return rc; }
    if (c->nccl_comm && (c->d_full_accum || c->d_full_display)) {
        int rc = vpt::comm_gather_frame(c, fa.geom, (const void*)kp.accum_buffer, (const void*)kp.display_buffer, stream);
        if (rc != VPT_OK) return rc;
    }
    return VPT_OK;
}

void vpt_adaptive_options_defaults(vpt_adaptive_options* opt) {
    if (!opt) return;
    opt->min_passes = 16; opt->check_interval = 16; opt->threshold = 0.01f;
}

// Adaptive frame.  Chunks end at every test point (min_passes, then every check_interval passes); after the resolve of a test chunk
// k_adapt stops the converged pixels and lists the tiles still active, whose number the host reads back (one stream synchronisation per
// test) to size the next chunk's grids.  Per pixel the work is that of vpt_render_passes: same Philox streams, same blue-noise table of
// each pass, same running mean in pass order.  A partitioned context with an active peer-memory exchange renders its share of the same
// frame: halo, agreement on when to stop and the final publish go through the exchange blocks (DESIGN.md section 8a).
int vpt_render_adaptive(vpt_context* c, void* const params[VPT_NUM_ARGS], unsigned max_passes, const vpt_adaptive_options* opt,
                        unsigned* d_pass_count, float* d_rel_error, unsigned* passes_run, void* stream_) {
    if (!c || !params) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: null argument");
    for (int i = 0; i < VPT_NUM_ARGS; ++i) if (!params[i]) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: params[" + std::to_string(i) + "] is null");
    if (!d_pass_count) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: d_pass_count is required (one unsigned per pixel)");
    vpt_adaptive_options o;
    vpt_adaptive_options_defaults(&o);
    if (opt) o = *opt;
    if (o.min_passes < 2) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: min_passes must be >= 2 (the error estimate needs two samples)");
    if (o.check_interval < 1) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: check_interval must be >= 1");
    if (!(o.threshold >= 0.0f)) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: threshold must be >= 0");
    if (o.threshold > 0.0f && o.threshold < FLT_MIN)
        return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: threshold must be 0 or >= FLT_MIN (the device flushes a subnormal threshold to 0)");
    if (max_passes == 0) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: max_passes must be >= 1");
    // a partitioned frame needs the peer-memory exchange: the 3x3 test reads across stripe boundaries and the ranks must agree on when to stop
    if (c->nccl_comm || (c->p2p_block && !c->p2p_on) || (c->n_ranks > 1 && !c->p2p_on))
        return fail(c, VPT_ERR_UNSUPPORTED, "vpt_render_adaptive: a partitioned context is supported only with an active peer-memory exchange "
                                            "(vpt_comm_p2p_export + import); vpt_set_partition alone, a suspended exchange and NCCL are not");
    const bool sharded = c->p2p_on;
    if (sharded && (c->region_req[0] | c->region_req[1] | c->region_req[2] | c->region_req[3]))
        return fail(c, VPT_ERR_UNSUPPORTED, "vpt_render_adaptive: a render region is not supported on a sharded adaptive frame (the convergence "
                                            "test and the final publish cover the whole frame); clear it with vpt_set_render_region(ctx, 0, 0, 0, 0)");
    vpt_kernel_params kp0;
    memcpy(&kp0, params[VPT_ARG_KERNEL_PARAMS], sizeof(vpt_kernel_params));
    if (sharded && ((int)kp0.resolution.x != c->p2p_w || (int)kp0.resolution.y != c->p2p_h))
        return fail(c, VPT_ERR_INVALID, "the peer exchange block was exported for another frame size (vpt_comm_p2p_export)");
    if (kp0.iteration != 0) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: Kernel_params.iteration must be 0 (an adaptive frame is a new frame)");
    if (!kp0.render) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: Kernel_params.render is 0, nothing would be sampled");
    if (kp0.max_interactions < 2) return fail(c, VPT_ERR_INVALID, "vpt_render_adaptive: Kernel_params.max_interactions must be >= 2");
    const unsigned n_total = max_passes < kp0.max_interactions ? max_passes : kp0.max_interactions;
    cudaStream_t stream = (cudaStream_t)stream_;

    FramePlan plan;
    { int rc = frame_setup(c, params, n_total, stream, plan); if (rc != VPT_OK) return rc; }
    vpt::FrameArgs& fa = plan.fa;
    const vpt::FrameGeom& g = fa.geom;
    const int n_tiles = ((g.width + 31) / 32) * ((g.local_rows + 3) / 4);

    // per-pixel state and the two tile lists, grown on demand and kept for later frames
    if ((size_t)g.n_local > c->cap_adapt_px) {
        cudaFree(c->d_adapt_stat); cudaFree(c->d_adapt_stopped); c->d_adapt_stat = nullptr; c->d_adapt_stopped = nullptr; c->cap_adapt_px = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_adapt_stat, sizeof(float4) * (size_t)g.n_local));
        VPT_CUDA(c, cudaMalloc(&c->d_adapt_stopped, (size_t)g.n_local));
        c->cap_adapt_px = (size_t)g.n_local;
    }
    if ((size_t)n_tiles > c->cap_adapt_tiles) {
        cudaFree(c->d_adapt_tiles); c->d_adapt_tiles = nullptr; c->cap_adapt_tiles = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_adapt_tiles, sizeof(unsigned) * (2 * (size_t)n_tiles + 5)));     // two lists + the read-back words below
        c->cap_adapt_tiles = (size_t)n_tiles;
    }
    unsigned* lists[2] = { c->d_adapt_tiles, c->d_adapt_tiles + n_tiles };
    // read back after a test: [0] tiles still active here (k_adapt's count of the next list); sharded frames also [1] tiles still active on
    // all ranks, [2] / [3] the error word after the halo / count barrier, [4] the error word when the call began
    unsigned* d_next_count = c->d_adapt_tiles + 2 * (size_t)n_tiles;

    vpt::AdaptArgs ad;
    ad.tiles = lists[0]; ad.n_tiles = n_tiles; ad.stopped = c->d_adapt_stopped; ad.stat = c->d_adapt_stat;
    ad.pass_count = d_pass_count; ad.rel_error = d_rel_error;
    ad.next_tiles = lists[1]; ad.next_count = d_next_count; ad.threshold = o.threshold;

    c->adaptive_accum = kp0.accum_buffer;        // from here on the buffers hold an adaptive frame
    // a render region: the frame starts on R's tiles, with every pixel outside R stopped
    if (plan.region) ad.n_tiles = (int)vpt::region_tiles(plan.rg);
    VPT_CUDA(c, timed(c, stream, 2, [&] { return plan.region ? vpt::launch_adapt_init_region(g, c->d_adapt_stopped, lists[0], plan.rg, stream)
                                                             : vpt::launch_adapt_init(g, c->d_adapt_stopped, lists[0], n_tiles, stream); }));
    c->launches++;

    // Sharded frame (peer-memory exchange): at every test the stripe-edge errors travel through the err planes of the blocks (halo), and
    // the ranks agree on the number of tiles still active anywhere; the frame goes on while that is > 0, so every rank issues the same
    // passes.  Two barriers per test on the adapt flags; ordering argument in DESIGN.md section 8a.
    vpt::AdaptPeers peers;
    vpt::P2pAdaptLocal own;
    bool entered = false;                        // every peer has entered this call: stores into their blocks are allowed
    auto await_peers = [&]() -> int {
        if (entered) return VPT_OK;
        entered = true;
        vpt::PeerFrames unused;
        return vpt::comm_p2p_peers(c, stream, &unused);
    };
    if (sharded) {
        vpt::comm_p2p_adapt_views(c, &peers, &own);
        { int rc = vpt::comm_p2p_begin(c, stream); if (rc != VPT_OK) return rc; }
        VPT_CUDA(c, vpt::launch_adapt_tally(nullptr, 0, own.error_word, d_next_count, 4, stream));
        c->launches++;
    }
    if (fa.miss_mask) {
        VPT_CUDA(c, timed(c, stream, 0, [&] { return plan.region ? vpt::launch_miss_cull_region(fa, c->d_miss_mask, plan.rg, plan.proj, stream, plan.ods_arg())
                                                                 : vpt::launch_miss_cull(fa, c->d_miss_mask, plan.proj, stream, plan.ods_arg()); }));
        c->launches++;
    }
    const void* bn = (const void*)(uintptr_t)kp0.blue_noise_buffer;
    unsigned done = 0, next_test = o.min_passes;
    unsigned active_anywhere = (unsigned)ad.n_tiles;      // sharded: tiles still active on any rank (a rank may have none left of its own)
    int cur = 0;
    while (done < n_total && active_anywhere > 0) {
        // a chunk never crosses a test point
        const unsigned boundary = next_test < n_total ? next_test : n_total;
        const unsigned np = (boundary - done) < (unsigned)plan.chunk ? (boundary - done) : (unsigned)plan.chunk;
        fa.kp.iteration = done;
        VPT_CUDA(c, timed(c, stream, 3, [&] { return vpt::launch_bn_prepare((void*)bn, c->d_bn_table, (int)np, plan.bn_limit, c->d_counters, stream); }));
        c->launches++;
        if (ad.n_tiles > 0) {
            VPT_CUDA(c, timed(c, stream, 0, [&] { return vpt::launch_generate_adaptive(stream_args(fa), (int)np, ad, plan.proj, plan.motion_arg(), plan.ods_arg(), stream); }));
            VPT_CUDA(c, timed(c, stream, 1, [&] { return launch_trace_of(c, plan, np, stream); }));
            if (plan.mv.out) {
                VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_motion_vectors(fa, plan.mv, (int)np, 1, nullptr, &ad, plan.motion_arg(), stream); }));
                c->launches++;
            }
            if (plan.collisions()) {
                VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_collision_aovs(fa, plan.ca, (int)np, 1, nullptr, &ad, plan.motion_arg(), stream); }));
                c->launches++;
            }
            if (plan.crypto.state) {
                VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_cryptomatte(fa, plan.crypto, (int)np, 1, nullptr, &ad, stream); }));
                c->launches++;
            }
            VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_resolve_adaptive(fa, plan.resolve, plan.atmo, (int)np, ad, plan.aov, plan.lg, plan.deep, plan.mattes, plan.proj, stream, plan.ods_arg()); }));
            c->launches += 3 + (plan.resolve.deep ? 1 : 0) + (plan.resolve.mattes ? 1 : 0);
        }
        done += np;
        if (done == next_test && done < n_total) {
            VPT_CUDA(c, cudaMemsetAsync(d_next_count, 0, sizeof(unsigned), stream));
            if (sharded) {
                { int rc = await_peers(); if (rc != VPT_OK) return rc; }
                VPT_CUDA(c, timed(c, stream, 2, [&] { return vpt::launch_adapt_halo(g, ad, peers, stream); }));
                { int rc = vpt::comm_p2p_adapt_barrier(c, stream); if (rc != VPT_OK) return rc; }         // halo barrier
            }
            VPT_CUDA(c, timed(c, stream, 2, [&] { return plan.region ? vpt::launch_adapt_region(g, ad, plan.rg, stream) : vpt::launch_adapt(g, ad, own.halo, stream); }));
            c->launches++;
            if (sharded) {
                VPT_CUDA(c, vpt::launch_adapt_count_publish(peers, c->rank, d_next_count, own.error_word, d_next_count, stream));
                { int rc = vpt::comm_p2p_adapt_barrier(c, stream); if (rc != VPT_OK) return rc; }         // count barrier
                VPT_CUDA(c, vpt::launch_adapt_tally(own.tiles, c->p2p_n, own.error_word, d_next_count, 3, stream));
                VPT_CUDA(c, cudaMemcpyAsync(c->h_pinned, d_next_count, 5 * sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
                c->launches += 3;
            } else {
                VPT_CUDA(c, cudaMemcpyAsync(c->h_pinned, d_next_count, sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
            }
            VPT_CUDA(c, cudaStreamSynchronize(stream));
            const unsigned* h = reinterpret_cast<const unsigned*>(c->h_pinned);
            if (sharded && h[3] != h[4])                 // a flag wait gave up (a rank is gone or made other calls): stop, do not trust the counts
                return fail(c, VPT_ERR_CUDA, std::string("vpt_render_adaptive: a peer flag wait was abandoned at the ") +
                                             (h[2] != h[4] ? "halo barrier (or the wait for the peers to enter the call)" : "count barrier") +
                                             " of the convergence test after " + std::to_string(done) + " passes; the exchange is no longer in step");
            cur ^= 1;
            ad.tiles = lists[cur]; ad.next_tiles = lists[cur ^ 1]; ad.n_tiles = (int)h[0];
            active_anywhere = sharded ? h[1] : h[0];
            next_test = o.check_interval > 0xffffffffu - next_test ? 0xffffffffu : next_test + o.check_interval;
        }
    }
    if (sharded) {
        // every local pixel, finished, into every rank's full-frame planes; then publish and wait until every peer has done the same
        { int rc = await_peers(); if (rc != VPT_OK) return rc; }
        VPT_CUDA(c, vpt::launch_adapt_publish(g, fa.kp, ad, peers, stream));
        c->launches++;
        { int rc = vpt::comm_p2p_layers(c, g, nullptr, layer_sources(plan), stream, plan.mv.out); if (rc != VPT_OK) return rc; }
        { int rc = vpt::comm_p2p_binned(c, g, nullptr, plan.deep.out, plan.mattes.out, stream); if (rc != VPT_OK) return rc; }
        { int rc = vpt::comm_p2p_end(c, stream); if (rc != VPT_OK) return rc; }
    }
    if (passes_run) *passes_run = done;
    return VPT_OK;
}

// The stopping rule alone: vpt_render_adaptive's schedule of chunks and tests on one rank, with k_debug_adapt_pass in place of the
// sample, trace and resolve kernels.  The tile lists, k_adapt / k_adapt_region and the Welford arithmetic are the production ones.
int vpt_debug_adapt_rule(const float* d_samples, unsigned width, unsigned height, unsigned n_passes, const vpt_adaptive_options* opt,
                         const unsigned* region, unsigned* d_pass_count, float* d_rel_error, float* d_test_err, unsigned max_tests,
                         unsigned* passes_run, unsigned* n_tests) {
    const char* me = "vpt_debug_adapt_rule: ";
    if (!d_samples || !d_pass_count) return vpt::fail_global(VPT_ERR_INVALID, std::string(me) + "null samples or pass counts");
    if (width == 0 || height == 0 || n_passes == 0) return vpt::fail_global(VPT_ERR_INVALID, std::string(me) + "width, height and n_passes must be >= 1");
    if ((unsigned long long)width * height > (1ull << 30)) return vpt::fail_global(VPT_ERR_INVALID, std::string(me) + "frame too large");
    if (max_tests > 0 && !d_test_err) return vpt::fail_global(VPT_ERR_INVALID, std::string(me) + "max_tests > 0 needs d_test_err");
    vpt_adaptive_options o;
    vpt_adaptive_options_defaults(&o);
    if (opt) o = *opt;
    if (o.min_passes < 2 || o.check_interval < 1 || !(o.threshold >= 0.0f) || (o.threshold > 0.0f && o.threshold < FLT_MIN))
        return vpt::fail_global(VPT_ERR_INVALID, std::string(me) + "options refused as vpt_render_adaptive refuses them");
    vpt::FrameGeom g;                                      // a single-rank frame of width x height
    g.width = (int)width; g.height = (int)height; g.local_rows = (int)height; g.n_local = (int)(width * height);
    g.stripe_h = (int)height; g.n_ranks = 1; g.rank = 0;
    vpt::RenderRegion rg;
    if (region) {
        if (region[0] >= region[2] || region[1] >= region[3] || region[2] > width || region[3] > height)
            return vpt::fail_global(VPT_ERR_INVALID, std::string(me) + "the region must satisfy x0 < x1 <= width and y0 < y1 <= height");
        rg = vpt::region_geometry(g, (int)region[0], (int)region[1], (int)region[2], (int)region[3]);
    }
    const int n_tiles = ((g.width + 31) / 32) * ((g.local_rows + 3) / 4);
    float4* stat = nullptr; uint8_t* stopped = nullptr; unsigned* lists = nullptr;
    cudaError_t e = cudaMalloc(&stat, sizeof(float4) * (size_t)g.n_local);
    if (e == cudaSuccess) e = cudaMalloc(&stopped, (size_t)g.n_local);
    if (e == cudaSuccess) e = cudaMalloc(&lists, sizeof(unsigned) * (2 * (size_t)n_tiles + 1));
    // NaN state (all bits set): a pixel that never samples -- outside the region -- holds its neighbours running if a test reads it
    if (e == cudaSuccess) e = cudaMemset(stat, 0xff, sizeof(float4) * (size_t)g.n_local);
    unsigned* list[2] = { lists, lists + n_tiles };
    int cur = 0;
    vpt::AdaptArgs ad;
    ad.tiles = list[0]; ad.n_tiles = region ? (int)vpt::region_tiles(rg) : n_tiles; ad.stopped = stopped; ad.stat = stat;
    ad.pass_count = d_pass_count; ad.rel_error = d_rel_error;
    ad.next_tiles = list[1]; ad.next_count = lists + 2 * (size_t)n_tiles; ad.threshold = o.threshold;
    if (e == cudaSuccess) e = region ? vpt::launch_adapt_init_region(g, stopped, lists, rg, 0) : vpt::launch_adapt_init(g, stopped, lists, n_tiles, 0);
    const float3* samples = reinterpret_cast<const float3*>(d_samples);
    unsigned done = 0, next_test = o.min_passes, tests = 0;
    while (e == cudaSuccess && done < n_passes && ad.n_tiles > 0) {
        const unsigned np = (next_test < n_passes ? next_test : n_passes) - done;
        e = vpt::launch_debug_adapt_pass(g, ad, samples, (int)done, (int)np, 0);
        done += np;
        if (e != cudaSuccess || done != next_test || done >= n_passes) continue;
        e = cudaMemset(ad.next_count, 0, sizeof(unsigned));
        if (e == cudaSuccess && tests < max_tests)          // every pixel's err as the test reads it: the .w plane of the state
            e = cudaMemcpy2D(d_test_err + (size_t)tests * g.n_local, sizeof(float), reinterpret_cast<const char*>(stat) + 3 * sizeof(float),
                             sizeof(float4), sizeof(float), (size_t)g.n_local, cudaMemcpyDeviceToDevice);
        if (e == cudaSuccess) e = region ? vpt::launch_adapt_region(g, ad, rg, 0) : vpt::launch_adapt(g, ad, nullptr, 0);
        unsigned active = 0;
        if (e == cudaSuccess) e = cudaMemcpy(&active, ad.next_count, sizeof(unsigned), cudaMemcpyDeviceToHost);
        cur ^= 1;
        ad.tiles = list[cur]; ad.next_tiles = list[cur ^ 1];
        ad.n_tiles = (int)active;
        ++tests;
        next_test = o.check_interval > 0xffffffffu - next_test ? 0xffffffffu : next_test + o.check_interval;
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaFree(stat); cudaFree(stopped); cudaFree(lists);
    if (e != cudaSuccess) return vpt::fail_global(VPT_ERR_CUDA, std::string(me) + cudaGetErrorString(e));
    if (passes_run) *passes_run = done;
    if (n_tests) *n_tests = tests;
    return VPT_OK;
}

int vpt_cryptomatte_rank(vpt_context* c, unsigned width, unsigned rows, const uint32_t* d_state, unsigned capacity, const float* d_id_of_instance,
                         unsigned n_instances, float sphere_id, unsigned n_ranks, float* d_out_f4, float* d_out_overflow, void* stream) {
    if (!c) return fail(nullptr, VPT_ERR_INVALID, "vpt_cryptomatte_rank: null context");
    if (!d_state || !d_out_f4) return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: null state or output");
    if (n_instances > 0 && !d_id_of_instance) return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: null id table with n_instances > 0");
    if (capacity < 1 || capacity > VPT_CRYPTO_MAX_ENTRIES)
        return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: capacity must be in 1.." + std::to_string(VPT_CRYPTO_MAX_ENTRIES) + ", got " + std::to_string(capacity));
    if (n_ranks < 2 || n_ranks > 32 || (n_ranks & 1u))
        return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: n_ranks must be even and in 2..32, got " + std::to_string(n_ranks));
    if (width == 0 || rows == 0) return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: width and rows must be >= 1");
    const unsigned long long n_px = (unsigned long long)width * rows;
    if (n_px > (1ull << 31)) return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: width * rows exceeds 2^31 pixels");
    if ((uintptr_t)d_state % 4 != 0 || (uintptr_t)d_out_f4 % 16 != 0 || (uintptr_t)d_id_of_instance % 4 != 0 || (uintptr_t)d_out_overflow % 4 != 0)
        return fail(c, VPT_ERR_INVALID, "vpt_cryptomatte_rank: the state, id table and overflow must be 4-byte aligned, the output 16-byte aligned");
    const size_t n = (size_t)n_px;
    const struct { const char* name; const void* p; size_t bytes; } bufs[] = {
        { "the state", d_state, 4 * n * (2 + 2 * (size_t)capacity) }, { "the id table", d_id_of_instance, 4 * (size_t)n_instances },
        { "the output", d_out_f4, 16 * n * (size_t)(n_ranks / 2) }, { "the overflow output", d_out_overflow, 4 * n } };
    for (int k = 2; k < 4; ++k)
        for (int j = 0; j < k; ++j)
            if (byte_ranges_overlap(bufs[k].p, bufs[k].bytes, bufs[j].p, bufs[j].bytes))
                return fail(c, VPT_ERR_INVALID, std::string("vpt_cryptomatte_rank: ") + bufs[k].name + " overlaps " + bufs[j].name);
    vpt::CryptoRank a;
    a.state = d_state; a.cap = (int)capacity; a.n_px = (long long)n_px; a.id_of_instance = d_id_of_instance; a.n_instances = n_instances;
    a.sphere_id = sphere_id; a.n_ranks = (int)n_ranks; a.out = reinterpret_cast<float2*>(d_out_f4); a.out_overflow = d_out_overflow;
    VPT_CUDA(c, vpt::launch_cryptomatte_rank(a, (cudaStream_t)stream));
    c->launches++;
    return VPT_OK;
}

void vpt_denoise_options_defaults(vpt_denoise_options* opt) {
    if (!opt) return;
    opt->iterations = 5; opt->sigma_luminance = 4.0f; opt->sigma_depth = 0.2f;
}

// The checks of vpt_denoise's arguments, for vpt_denoise and vpt_denoise_layers (`fn` names the caller in the messages): VPT_OK with the
// options in *o, or the refusal.
static int denoise_check(vpt_context* c, const char* fn, unsigned width, unsigned height, const float* d_color, const float* d_depth,
                         const float* d_rel_error, const vpt_denoise_options* opt, float* d_out, unsigned* d_out_display, vpt_denoise_options* o) {
    const std::string f(fn);
    if (!c || !d_color || !d_out) return fail(c, VPT_ERR_INVALID, f + ": null context, colour or output");
    if (width == 0 || height == 0) return fail(c, VPT_ERR_INVALID, f + ": width and height must be >= 1");
    if (width > 65535 || height > 65535) return fail(c, VPT_ERR_INVALID, f + ": width and height must be <= 65535");
    vpt_denoise_options_defaults(o);
    if (opt) *o = *opt;
    if (o->iterations < 1 || o->iterations > 10) return fail(c, VPT_ERR_INVALID, f + ": iterations must be 1..10");
    if (!(std::isfinite(o->sigma_luminance) && o->sigma_luminance > 0.0f))
        return fail(c, VPT_ERR_INVALID, f + ": sigma_luminance must be finite and > 0");
    if (!(std::isfinite(o->sigma_depth) && o->sigma_depth > 0.0f)) return fail(c, VPT_ERR_INVALID, f + ": sigma_depth must be finite and > 0");
    const size_t px = (size_t)width * height;
    const size_t b3 = 3 * sizeof(float) * px, b1 = sizeof(float) * px;
    if (d_out != d_color && byte_ranges_overlap(d_out, b3, d_color, b3))
        return fail(c, VPT_ERR_INVALID, f + ": d_out_f3 partially overlaps d_color_f3 (it may only be the very same buffer)");
    if (byte_ranges_overlap(d_out, b3, d_depth, b1) || byte_ranges_overlap(d_out, b3, d_rel_error, b1))
        return fail(c, VPT_ERR_INVALID, f + ": d_out_f3 overlaps d_depth or d_rel_error");
    if (byte_ranges_overlap(d_out_display, b1, d_color, b3) || byte_ranges_overlap(d_out_display, b1, d_depth, b1) ||
        byte_ranges_overlap(d_out_display, b1, d_rel_error, b1))
        return fail(c, VPT_ERR_INVALID, f + ": d_out_display overlaps an input");
    if (byte_ranges_overlap(d_out_display, b1, d_out, b3)) return fail(c, VPT_ERR_INVALID, f + ": d_out_display overlaps d_out_f3");
    return VPT_OK;
}

// The beauty's scratch planes (48 B per pixel) for px pixels, allocated on first use, grown when a larger frame comes.
static int denoise_scratch(vpt_context* c, size_t px) {
    if (px > c->cap_dn_px) {
        cudaFree(c->d_dn_cv); cudaFree(c->d_dn_yz); c->d_dn_cv = nullptr; c->d_dn_yz = nullptr; c->cap_dn_px = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_dn_cv, 2 * px * sizeof(float4)));
        VPT_CUDA(c, cudaMalloc(&c->d_dn_yz, 2 * px * sizeof(float2)));
        c->cap_dn_px = px;
    }
    return VPT_OK;
}

static vpt::DenoiseArgs denoise_args(vpt_context* c, unsigned width, unsigned height, const float* d_color, const float* d_depth,
                                     const float* d_rel_error, const vpt_denoise_options& o, float exposure_scale, float* d_out,
                                     unsigned* d_out_display) {
    const size_t px = (size_t)width * height;
    vpt::DenoiseArgs a;
    a.width = (int)width; a.height = (int)height; a.iterations = (int)o.iterations;
    a.sigma_l = o.sigma_luminance; a.sigma_z = o.sigma_depth; a.exposure_scale = exposure_scale;
    a.color = d_color; a.depth = d_depth; a.rel_error = d_rel_error; a.out_f3 = d_out; a.out_display = d_out_display;
    a.cv[0] = c->d_dn_cv; a.cv[1] = c->d_dn_cv + px; a.yz[0] = c->d_dn_yz; a.yz[1] = c->d_dn_yz + px;
    return a;
}

// Denoiser: prep + one a-trous launch per level on `stream` (csrc/device/vpt_denoise.cu), no synchronisation.  The scratch planes are the
// context's; the last level reads only them, which is what makes d_out_f3 == d_color_f3 safe.
int vpt_denoise(vpt_context* c, unsigned width, unsigned height, const float* d_color, const float* d_depth, const float* d_rel_error,
                const vpt_denoise_options* opt, float exposure_scale, float* d_out, unsigned* d_out_display, void* stream) {
    vpt_denoise_options o;
    { int rc = denoise_check(c, "vpt_denoise", width, height, d_color, d_depth, d_rel_error, opt, d_out, d_out_display, &o); if (rc != VPT_OK) return rc; }
    { int rc = denoise_scratch(c, (size_t)width * height); if (rc != VPT_OK) return rc; }
    const vpt::DenoiseArgs a = denoise_args(c, width, height, d_color, d_depth, d_rel_error, o, exposure_scale, d_out, d_out_display);
    VPT_CUDA(c, vpt::launch_denoise(a, (cudaStream_t)stream));
    c->launches += 1 + o.iterations;
    return VPT_OK;
}

// vpt_denoise plus layers filtered with the beauty's weights: the layers are gathered into the context's layer planes (two sets of
// 16 B per plane and pixel) before the first level, so the last level may write a layer's source or the beauty's colour.
int vpt_denoise_layers(vpt_context* c, unsigned width, unsigned height, const float* d_color, const float* d_depth, const float* d_rel_error,
                       const vpt_denoise_options* opt, float exposure_scale, float* d_out, unsigned* d_out_display,
                       const vpt_denoise_layer* layers, unsigned n_layers, void* stream) {
    vpt_denoise_options o;
    { int rc = denoise_check(c, "vpt_denoise_layers", width, height, d_color, d_depth, d_rel_error, opt, d_out, d_out_display, &o); if (rc != VPT_OK) return rc; }
    if (n_layers > 0 && !layers) return fail(c, VPT_ERR_INVALID, "vpt_denoise_layers: n_layers > 0 with a null layers array");
    const size_t px = (size_t)width * height;
    const size_t b3 = 3 * sizeof(float) * px, b1 = sizeof(float) * px;
    std::vector<vpt::DenoiseLayer> dl(n_layers);
    size_t n_planes = 0;
    for (unsigned l = 0; l < n_layers; ++l) {
        const vpt_denoise_layer& L = layers[l];
        const std::string at = "vpt_denoise_layers: layer " + std::to_string(l);
        if (!L.src || !L.dst) return fail(c, VPT_ERR_INVALID, at + " has a null src or dst");
        if (L.channels < 1 || L.channels > 4) return fail(c, VPT_ERR_INVALID, at + ": channels must be 1..4");
        if (L.count == 0) return fail(c, VPT_ERR_INVALID, at + ": count must be >= 1");
        dl[l] = vpt::DenoiseLayer{ L.src, L.dst, L.channels, L.count };
        n_planes += L.count;
    }
    auto bytes = [&](unsigned l) { return (size_t)layers[l].count * layers[l].channels * sizeof(float) * px; };
    for (unsigned l = 0; l < n_layers; ++l) {
        const std::string at = "vpt_denoise_layers: layer " + std::to_string(l);
        const float* dst = layers[l].dst;
        const size_t n = bytes(l);
        if (dst != layers[l].src && byte_ranges_overlap(dst, n, layers[l].src, n))
            return fail(c, VPT_ERR_INVALID, at + ": dst partially overlaps its src (it may only be the very same buffer)");
        for (unsigned m = 0; m < n_layers; ++m) {
            if (m == l) continue;
            if (byte_ranges_overlap(dst, n, layers[m].src, bytes(m)) || byte_ranges_overlap(dst, n, layers[m].dst, bytes(m)))
                return fail(c, VPT_ERR_INVALID, at + ": dst overlaps the src or dst of layer " + std::to_string(m));
        }
        if (byte_ranges_overlap(dst, n, d_color, b3) || byte_ranges_overlap(dst, n, d_out, b3) || byte_ranges_overlap(dst, n, d_out_display, b1))
            return fail(c, VPT_ERR_INVALID, at + ": dst overlaps d_color_f3, d_out_f3 or d_out_display");
        if (byte_ranges_overlap(dst, n, d_depth, b1) || byte_ranges_overlap(dst, n, d_rel_error, b1))
            return fail(c, VPT_ERR_INVALID, at + ": dst overlaps d_depth or d_rel_error");
    }
    { int rc = denoise_scratch(c, px); if (rc != VPT_OK) return rc; }
    const size_t need = n_planes * px;
    if (need > c->cap_dn_layer) {
        cudaFree(c->d_dn_layer); c->d_dn_layer = nullptr; c->cap_dn_layer = 0;
        VPT_CUDA(c, cudaMalloc(&c->d_dn_layer, 2 * need * sizeof(float4)));
        c->cap_dn_layer = need;
    }
    vpt::DenoiseArgs a = denoise_args(c, width, height, d_color, d_depth, d_rel_error, o, exposure_scale, d_out, d_out_display);
    a.layers = dl.data(); a.n_layers = (int)n_layers;
    a.lp[0] = c->d_dn_layer; a.lp[1] = c->d_dn_layer + need;
    VPT_CUDA(c, vpt::launch_denoise(a, (cudaStream_t)stream));
    c->launches += 1 + o.iterations + n_layers + (unsigned long long)o.iterations * vpt::denoise_layer_groups(n_planes);
    return VPT_OK;
}

void vpt_temporal_options_defaults(vpt_temporal_options* opt) {
    if (!opt) return;
    opt->max_history = 16; opt->clip_sigma = INFINITY;   // DESIGN.md section 8p: the sweep
}

static_assert(vpt::kTemporalMaxLayers == VPT_TEMPORAL_MAX_LAYERS, "temporal layer limit");

// Temporal filter: one k_temporal launch on `stream` (csrc/device/vpt_temporal.cu), no synchronisation, no scratch, for vpt_temporal (no
// layers) and vpt_temporal_layers (`fn` names the caller in the messages).  The fetch reads neighbouring pixels of the histories and the
// clip those of the colour, so no output may share a byte with any input or with another output.
static int temporal(vpt_context* c, const char* fn, unsigned width, unsigned height, const float* d_color, const float* d_vectors,
                    const vpt_camera* current, const vpt_camera* previous, const float* d_history, const float* d_history_len,
                    const vpt_temporal_options* opt, float exposure_scale, float* d_out, float* d_out_len, unsigned* d_out_display,
                    const vpt_temporal_layer* layers, unsigned n_layers, void* stream) {
    const std::string f(fn);
    if (!c || !d_color || !d_vectors || !current || !previous || !d_out || !d_out_len)
        return fail(c, VPT_ERR_INVALID, f + ": null context, colour, vectors, camera or output");
    if (width == 0 || height == 0) return fail(c, VPT_ERR_INVALID, f + ": width and height must be >= 1");
    if (width > 65535 || height > 65535) return fail(c, VPT_ERR_INVALID, f + ": width and height must be <= 65535");
    if (!d_history != !d_history_len) return fail(c, VPT_ERR_INVALID, f + ": d_history_f3 and d_history_len must both be set or both be NULL");
    vpt_temporal_options o;
    vpt_temporal_options_defaults(&o);
    if (opt) o = *opt;
    if (o.max_history < 1 || o.max_history > (1u << 24)) return fail(c, VPT_ERR_INVALID, f + ": max_history must be 1..2^24");
    if (!(o.clip_sigma > 0.0f)) return fail(c, VPT_ERR_INVALID, f + ": clip_sigma must be > 0 (+inf: no clip)");
    const struct { const char* cam; const vpt_camera* k; } cams[] = { { "current", current }, { "previous", previous } };
    for (const auto& k : cams) {
        const struct { const char* name; vpt_f3 v; } fields[] = {
            { "origin", k.k->origin }, { "lower_left_corner", k.k->lower_left_corner }, { "horizontal", k.k->horizontal }, { "vertical", k.k->vertical } };
        for (const auto& fl : fields)
            if (!std::isfinite(fl.v.x) || !std::isfinite(fl.v.y) || !std::isfinite(fl.v.z))
                return fail(c, VPT_ERR_INVALID, f + ": " + k.cam + "." + fl.name + " is not finite");
    }
    if (n_layers > 0 && !layers) return fail(c, VPT_ERR_INVALID, f + ": n_layers > 0 with a null layers array");
    if (n_layers > VPT_TEMPORAL_MAX_LAYERS)
        return fail(c, VPT_ERR_INVALID, f + ": at most " + std::to_string(VPT_TEMPORAL_MAX_LAYERS) + " layers");
    for (unsigned l = 0; l < n_layers; ++l) {
        const vpt_temporal_layer& L = layers[l];
        const std::string at = f + ": layer " + std::to_string(l);
        if (!L.src || !L.dst) return fail(c, VPT_ERR_INVALID, at + " has a null src or dst");
        if (!L.history != !d_history) return fail(c, VPT_ERR_INVALID, at + ": history must be set exactly when d_history_f3 is");
        if (L.channels < 1 || L.channels > 4) return fail(c, VPT_ERR_INVALID, at + ": channels must be 1..4");
        if (L.count == 0) return fail(c, VPT_ERR_INVALID, at + ": count must be >= 1");
    }
    const size_t px = (size_t)width * height;
    const size_t b3 = 3 * sizeof(float) * px, b1 = sizeof(float) * px;
    struct Range { std::string name; const void* p; size_t bytes; };
    std::vector<Range> ins = { { "d_color_f3", d_color, b3 }, { "d_vectors_f3", d_vectors, b3 }, { "d_history_f3", d_history, b3 },
                               { "d_history_len", d_history_len, b1 } };
    std::vector<Range> outs = { { "d_out_f3", d_out, b3 }, { "d_out_len", d_out_len, b1 }, { "d_out_display", d_out_display, b1 } };
    for (unsigned l = 0; l < n_layers; ++l) {
        const size_t n = (size_t)layers[l].count * layers[l].channels * sizeof(float) * px;
        const std::string at = "layer " + std::to_string(l);
        ins.push_back({ at + " src", layers[l].src, n });
        ins.push_back({ at + " history", layers[l].history, n });
        outs.push_back({ at + " dst", layers[l].dst, n });
    }
    for (const auto& w : outs) {
        for (const auto& r : ins)
            if (byte_ranges_overlap(w.p, w.bytes, r.p, r.bytes)) return fail(c, VPT_ERR_INVALID, f + ": " + w.name + " overlaps " + r.name);
        for (const auto& w2 : outs)
            if (&w2 != &w && byte_ranges_overlap(w.p, w.bytes, w2.p, w2.bytes))
                return fail(c, VPT_ERR_INVALID, f + ": " + w.name + " overlaps " + w2.name);
    }
    vpt::TemporalArgs a;
    a.width = (int)width; a.height = (int)height; a.max_history = o.max_history; a.clip_sigma = o.clip_sigma; a.exposure_scale = exposure_scale;
    a.a_origin = current->origin; a.a_llc = current->lower_left_corner; a.a_horizontal = current->horizontal; a.a_vertical = current->vertical;
    a.b_origin = previous->origin; a.b_llc = previous->lower_left_corner; a.b_horizontal = previous->horizontal; a.b_vertical = previous->vertical;
    a.color = d_color; a.vectors = d_vectors; a.history = d_history; a.history_len = d_history_len;
    a.out = d_out; a.out_len = d_out_len; a.out_display = d_out_display;
    a.n_layers = (int)n_layers;
    for (unsigned l = 0; l < n_layers; ++l)
        a.layers[l] = vpt::TemporalLayer{ layers[l].src, layers[l].history, layers[l].dst, layers[l].channels, layers[l].count };
    VPT_CUDA(c, vpt::launch_temporal(a, (cudaStream_t)stream));
    c->launches++;
    return VPT_OK;
}

int vpt_temporal(vpt_context* c, unsigned width, unsigned height, const float* d_color, const float* d_vectors, const vpt_camera* current,
                 const vpt_camera* previous, const float* d_history, const float* d_history_len, const vpt_temporal_options* opt,
                 float exposure_scale, float* d_out, float* d_out_len, unsigned* d_out_display, void* stream) {
    return temporal(c, "vpt_temporal", width, height, d_color, d_vectors, current, previous, d_history, d_history_len, opt, exposure_scale,
                    d_out, d_out_len, d_out_display, nullptr, 0, stream);
}

int vpt_temporal_layers(vpt_context* c, unsigned width, unsigned height, const float* d_color, const float* d_vectors,
                        const vpt_camera* current, const vpt_camera* previous, const float* d_history, const float* d_history_len,
                        const vpt_temporal_options* opt, float exposure_scale, float* d_out, float* d_out_len, unsigned* d_out_display,
                        const vpt_temporal_layer* layers, unsigned n_layers, void* stream) {
    return temporal(c, "vpt_temporal_layers", width, height, d_color, d_vectors, current, previous, d_history, d_history_len, opt,
                    exposure_scale, d_out, d_out_len, d_out_display, layers, n_layers, stream);
}

// Statistics accumulated since the last call (needs option "count_stats"): out[0..4] = volume lookups, lane-steps,
// warp step iterations, lane transitions, warp transition rounds; out[5] = rays taken from the queue; out[6] = bricks
// fetched (k_trace_brick only).  Synchronises the device.
int vpt_get_counters(vpt_context* c, unsigned long long out[8], int reset) {
    if (!c || !out) return VPT_ERR_INVALID;
    VPT_CUDA(c, cudaDeviceSynchronize());
    VPT_CUDA(c, cudaMemcpy(out, c->d_stats, sizeof(unsigned long long) * 8, cudaMemcpyDeviceToHost));
    out[7] = (unsigned long long)c->last_trace_rays;              // no kernel counts into slot 7
    if (reset) VPT_CUDA(c, cudaMemset(c->d_stats, 0, sizeof(unsigned long long) * 16));
    return VPT_OK;
}

// The hop statistics accumulated since the last reset (option "count_stats"; vpt_get_counters with reset clears them too): out[0..2] =
// k_trace hops over empty nodes in delta / ratio / emission walks, out[3] = k_trace walks ended by "empty ahead", out[4..6] = k_generate
// pre-step rays / their hops / pre-step rays ended by "empty ahead"; out[7] = 0.  Synchronises the device.
int vpt_get_hop_counters(vpt_context* c, unsigned long long out[8], int reset) {
    if (!c || !out) return VPT_ERR_INVALID;
    VPT_CUDA(c, cudaDeviceSynchronize());
    VPT_CUDA(c, cudaMemcpy(out, c->d_stats + 8, sizeof(unsigned long long) * 8, cudaMemcpyDeviceToHost));
    if (reset) VPT_CUDA(c, cudaMemset(c->d_stats + 8, 0, sizeof(unsigned long long) * 8));
    return VPT_OK;
}

int vpt_debug_empty_ahead(vpt_context* c, unsigned char out[VPT_EMPTY_AHEAD_BYTES]) {
    static_assert(sizeof(vpt::EmptyAhead) == VPT_EMPTY_AHEAD_BYTES, "vpt_b200.h states the table's size");
    if (!c || !out) return VPT_ERR_INVALID;
    VPT_CUDA(c, cudaDeviceSynchronize());
    VPT_CUDA(c, cudaMemcpy(out, &reinterpret_cast<const vpt::SceneAlloc*>(c->d_scene)->ahead, VPT_EMPTY_AHEAD_BYTES, cudaMemcpyDeviceToHost));
    return VPT_OK;
}

// Per-kernel device time accumulated since the last call (needs option "profile"):
// ms[0..3] = generate, trace, resolve, bn_advance; n[0..3] = launches of each.  Synchronises the device.
int vpt_get_kernel_times(vpt_context* c, float ms[4], int n[4]) {
    if (!c || !ms || !n) return VPT_ERR_INVALID;
    VPT_CUDA(c, cudaDeviceSynchronize());
    for (int i = 0; i < 4; ++i) { ms[i] = 0.f; n[i] = 0; }
    for (auto& e : c->events) {
        float t = 0.f; cudaEventElapsedTime(&t, e.a, e.b);
        if (e.kind >= 0 && e.kind < 4) { ms[e.kind] += t; n[e.kind]++; }
        cudaEventDestroy(e.a); cudaEventDestroy(e.b);
    }
    c->events.clear();
    return VPT_OK;
}

int vpt_render_pass(vpt_context* c, void* const params[VPT_NUM_ARGS], void* stream) {
    return vpt_render_passes(c, params, 1, stream);
}

// k_ods_cameras for the next render call (ods_req at iteration 0, else ods_cur) at the jitter the blue-noise buffer holds now, on the default
// stream; rays: camera_b0 of each pixel's camera (4 floats) instead of the camera (8 floats)
static int ods_cameras(vpt_context* c, const char* fn, const vpt_camera& cam, const vpt_kernel_params& kp, int rays, float* d_out) {
    const vpt::OdsParams& od = kp.iteration == 0 ? c->ods_req : c->ods_cur;
    if (od.layout == vpt::kOdsOverUnder && (kp.resolution.y & 1u))
        return fail(c, VPT_ERR_UNSUPPORTED, std::string(fn) + ": the over-under ODS layout needs an even height, got " + std::to_string(kp.resolution.y));
    VPT_CUDA(c, vpt::launch_ods_cameras(cam, od, kp.resolution, make_geom(c, kp.resolution.x, kp.resolution.y), (const void*)(uintptr_t)kp.blue_noise_buffer,
                                        rays, d_out, 0));
    return VPT_OK;
}

// b0 of every local pixel at the next render call's first pass: the projection that call takes (proj_req at iteration 0, else proj_cur)
// at the jitter the blue-noise buffer holds now, on the default stream.  Reads the camera, Kernel_params and the blue noise; writes d_out_f4 only.
int vpt_debug_camera_rays(vpt_context* c, void* const params[VPT_NUM_ARGS], float* d_out_f4) {
    if (!c || !params || !d_out_f4 || !params[VPT_ARG_CAMERA] || !params[VPT_ARG_KERNEL_PARAMS])
        return fail(c, VPT_ERR_INVALID, "vpt_debug_camera_rays: null argument");
    vpt_camera cam; vpt_kernel_params kp;
    memcpy(&cam, params[VPT_ARG_CAMERA], sizeof(cam));
    memcpy(&kp, params[VPT_ARG_KERNEL_PARAMS], sizeof(kp));
    if (!kp.blue_noise_buffer) return fail(c, VPT_ERR_INVALID, "vpt_debug_camera_rays: Kernel_params.blue_noise_buffer is null");
    if (kp.resolution.x == 0 || kp.resolution.y == 0) return fail(c, VPT_ERR_INVALID, "vpt_debug_camera_rays: resolution is zero");
    if (kp.iteration == 0 ? c->motion_req : c->motion_cur)
        return fail(c, VPT_ERR_UNSUPPORTED, "vpt_debug_camera_rays: the next call is a camera-motion frame, whose rays depend on each sample's "
                                            "shutter draw; use vpt_debug_motion_cameras");
    const vpt::Projection& pj = kp.iteration == 0 ? c->proj_req : c->proj_cur;
    if (vpt::ods(pj)) {                       // camera_b0 of each pixel's ODS camera
        const int rc = ods_cameras(c, "vpt_debug_camera_rays", cam, kp, 1, d_out_f4);
        if (rc == VPT_OK) c->launches++;
        return rc;
    }
    VPT_CUDA(c, vpt::launch_camera_rays(cam, kp.resolution, make_geom(c, kp.resolution.x, kp.resolution.y), pj, (const void*)(uintptr_t)kp.blue_noise_buffer,
                                        reinterpret_cast<float4*>(d_out_f4), 0));
    c->launches++;
    return VPT_OK;
}

// The ODS camera of every local pixel's first sample of the next render call (the projection it takes must be ODS).  Reads the camera,
// Kernel_params and the blue noise; writes d_out only.
int vpt_debug_ods_cameras(vpt_context* c, void* const params[VPT_NUM_ARGS], float* d_out) {
    if (!c || !params || !d_out || !params[VPT_ARG_CAMERA] || !params[VPT_ARG_KERNEL_PARAMS])
        return fail(c, VPT_ERR_INVALID, "vpt_debug_ods_cameras: null argument");
    vpt_camera cam; vpt_kernel_params kp;
    memcpy(&cam, params[VPT_ARG_CAMERA], sizeof(cam));
    memcpy(&kp, params[VPT_ARG_KERNEL_PARAMS], sizeof(kp));
    if (!kp.blue_noise_buffer) return fail(c, VPT_ERR_INVALID, "vpt_debug_ods_cameras: Kernel_params.blue_noise_buffer is null");
    if (kp.resolution.x == 0 || kp.resolution.y == 0) return fail(c, VPT_ERR_INVALID, "vpt_debug_ods_cameras: resolution is zero");
    if (!vpt::ods(kp.iteration == 0 ? c->proj_req : c->proj_cur))
        return fail(c, VPT_ERR_INVALID, "vpt_debug_ods_cameras: the next call has no ODS projection (vpt_set_projection_ods)");
    const int rc = ods_cameras(c, "vpt_debug_ods_cameras", cam, kp, 0, d_out);
    if (rc == VPT_OK) c->launches++;
    return rc;
}

// The camera of every local pixel's first sample of the next render call under camera motion (motion_req at iteration 0, else motion_cur,
// on the stream the sample offset selects):
// its shutter draw and motion_camera of it, on the default stream.  Reads the camera and Kernel_params; writes d_out only.
int vpt_debug_motion_cameras(vpt_context* c, void* const params[VPT_NUM_ARGS], float* d_out) {
    if (!c || !params || !d_out || !params[VPT_ARG_CAMERA] || !params[VPT_ARG_KERNEL_PARAMS])
        return fail(c, VPT_ERR_INVALID, "vpt_debug_motion_cameras: null argument");
    vpt_camera cam; vpt_kernel_params kp;
    memcpy(&cam, params[VPT_ARG_CAMERA], sizeof(cam));
    memcpy(&kp, params[VPT_ARG_KERNEL_PARAMS], sizeof(kp));
    if (kp.resolution.x == 0 || kp.resolution.y == 0) return fail(c, VPT_ERR_INVALID, "vpt_debug_motion_cameras: resolution is zero");
    const bool motion = kp.iteration == 0 ? c->motion_req : c->motion_cur;
    if (!motion) return fail(c, VPT_ERR_INVALID, "vpt_debug_motion_cameras: the next call has no camera motion (vpt_set_camera_motion)");
    const uint32_t stream = (kp.iteration == 0 ? c->sample_offset_req : c->sample_offset_cur) + kp.iteration;   // the sample offset's stream
    VPT_CUDA(c, vpt::launch_motion_cameras(cam, kp.iteration == 0 ? c->motion_close_req : c->motion_close_cur,
                                           make_geom(c, kp.resolution.x, kp.resolution.y), stream, d_out, 0));
    c->launches++;
    return VPT_OK;
}

// ------------------------------------------------------------------------------------------------------
// host-side scene helpers
// ------------------------------------------------------------------------------------------------------
int vpt_texture_create_3d(const float* host, int channels, int dx, int dy, int dz, vpt_tex_t* tex_out, void** array_out) {
    if (!host || !tex_out || !array_out || (channels != 1 && channels != 4) || dx < 1 || dy < 1 || dz < 1)
        return fail(nullptr, VPT_ERR_INVALID, "vpt_texture_create_3d: bad arguments");
    cudaChannelFormatDesc desc = channels == 1 ? cudaCreateChannelDesc<float>() : cudaCreateChannelDesc<float4>();
    cudaExtent ext = make_cudaExtent((size_t)dx, (size_t)dy, (size_t)dz);
    cudaArray_t arr = nullptr;
    VPT_CUDA(nullptr, cudaMalloc3DArray(&arr, &desc, ext));
    cudaMemcpy3DParms cp; memset(&cp, 0, sizeof(cp));
    const size_t esz = sizeof(float) * (size_t)channels;
    cp.srcPtr = make_cudaPitchedPtr((void*)host, (size_t)dx * esz, (size_t)dx, (size_t)dy);
    cp.dstArray = arr; cp.extent = ext; cp.kind = cudaMemcpyHostToDevice;
    VPT_CUDA(nullptr, cudaMemcpy3D(&cp));
    cudaResourceDesc res; memset(&res, 0, sizeof(res));
    res.resType = cudaResourceTypeArray; res.res.array.array = arr;
    cudaTextureDesc td; memset(&td, 0, sizeof(td));
    td.normalizedCoords = 1; td.filterMode = cudaFilterModeLinear;
    td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
    td.readMode = cudaReadModeElementType;
    cudaTextureObject_t tex = 0;
    VPT_CUDA(nullptr, cudaCreateTextureObject(&tex, &res, &td, NULL));
    *tex_out = (vpt_tex_t)tex; *array_out = (void*)arr;
    return VPT_OK;
}

int vpt_texture_create_3d_from_device(const float* d_data, int channels, int dx, int dy, int dz, vpt_tex_t* tex_out, void** array_out) {
    if (!d_data || !tex_out || !array_out || (channels != 1 && channels != 4) || dx < 1 || dy < 1 || dz < 1)
        return fail(nullptr, VPT_ERR_INVALID, "vpt_texture_create_3d_from_device: bad arguments");
    cudaChannelFormatDesc desc = channels == 1 ? cudaCreateChannelDesc<float>() : cudaCreateChannelDesc<float4>();
    cudaExtent ext = make_cudaExtent((size_t)dx, (size_t)dy, (size_t)dz);
    cudaArray_t arr = nullptr;
    VPT_CUDA(nullptr, cudaMalloc3DArray(&arr, &desc, ext));
    cudaMemcpy3DParms cp; memset(&cp, 0, sizeof(cp));
    const size_t esz = sizeof(float) * (size_t)channels;
    cp.srcPtr = make_cudaPitchedPtr((void*)d_data, (size_t)dx * esz, (size_t)dx, (size_t)dy);
    cp.dstArray = arr; cp.extent = ext; cp.kind = cudaMemcpyDeviceToDevice;
    cudaError_t e = cudaMemcpy3D(&cp);
    cudaResourceDesc res; memset(&res, 0, sizeof(res));
    res.resType = cudaResourceTypeArray; res.res.array.array = arr;
    cudaTextureDesc td; memset(&td, 0, sizeof(td));
    td.normalizedCoords = 1; td.filterMode = cudaFilterModeLinear;
    td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
    td.readMode = cudaReadModeElementType;
    cudaTextureObject_t tex = 0;
    if (e == cudaSuccess) e = cudaCreateTextureObject(&tex, &res, &td, NULL);
    if (e != cudaSuccess) { cudaFreeArray(arr); return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_texture_create_3d_from_device: ") + cudaGetErrorString(e)); }
    *tex_out = (vpt_tex_t)tex; *array_out = (void*)arr;
    return VPT_OK;
}

int vpt_procedural_fill(float* d_buffer, int dx, int dy, int dz, int noise_type, float scale, int seed, void* stream) {
    if (!d_buffer || dx < 1 || dy < 1 || dz < 1) return fail(nullptr, VPT_ERR_INVALID, "vpt_procedural_fill: bad arguments");
    if (noise_type != 0) return fail(nullptr, VPT_ERR_UNSUPPORTED, "vpt_procedural_fill: only noise type 0 (Perlin gradient noise, the reference's default) is built");
    VPT_CUDA(nullptr, vpt::launch_fill_perlin(d_buffer, dx, dy, dz, scale, seed, (cudaStream_t)stream));
    return VPT_OK;
}

int vpt_bricks_create(const float* d_dense, int dx, int dy, int dz, vpt_devptr_t* d_pool_out, unsigned long long* bytes_out) {
    if (!d_dense || !d_pool_out || dx < 1 || dy < 1 || dz < 1) return fail(nullptr, VPT_ERR_INVALID, "vpt_bricks_create: bad arguments");
    const size_t nb = (size_t)((dx + 3) / 4) * ((dy + 3) / 4) * ((dz + 3) / 4);
    if (nb > (size_t)0x7fffffff) return fail(nullptr, VPT_ERR_UNSUPPORTED, "vpt_bricks_create: more than 2^31 bricks");
    float* pool = nullptr;
    VPT_CUDA(nullptr, cudaMalloc(&pool, nb * 512));
    cudaError_t e = vpt::launch_build_bricks(d_dense, dx, dy, dz, pool, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaFree(pool); return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_bricks_create: ") + cudaGetErrorString(e)); }
    *d_pool_out = (vpt_devptr_t)(uintptr_t)pool;
    if (bytes_out) *bytes_out = (unsigned long long)nb * 512ull;
    return VPT_OK;
}

int vpt_bricks_read(vpt_devptr_t d_pool, unsigned long long first_brick, unsigned long long n_bricks, float* h_out) {
    if (!d_pool || !h_out) return fail(nullptr, VPT_ERR_INVALID, "vpt_bricks_read: null argument");
    VPT_CUDA(nullptr, cudaMemcpy(h_out, reinterpret_cast<const char*>((uintptr_t)d_pool) + first_brick * 512ull, n_bricks * 512ull, cudaMemcpyDeviceToHost));
    return VPT_OK;
}

int vpt_debug_sampler_compare(vpt_tex_t tex, vpt_devptr_t d_pool, int dx, int dy, int dz, int n_points, unsigned seed, double out12[12]) {
    if (!tex || !d_pool || !out12 || n_points < 1) return fail(nullptr, VPT_ERR_INVALID, "vpt_debug_sampler_compare: bad arguments");
    double* d_out = nullptr;
    VPT_CUDA(nullptr, cudaMalloc(&d_out, sizeof(double) * 12));
    cudaError_t e = cudaMemset(d_out, 0, sizeof(double) * 12);
    const int dims[3] = { dx, dy, dz };
    if (e == cudaSuccess) e = vpt::launch_sampler_compare(tex, reinterpret_cast<const float*>((uintptr_t)d_pool), dims, n_points, seed, d_out, 0);
    if (e == cudaSuccess) e = cudaMemcpy(out12, d_out, sizeof(double) * 12, cudaMemcpyDeviceToHost);
    cudaFree(d_out);
    if (e != cudaSuccess) return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_debug_sampler_compare: ") + cudaGetErrorString(e));
    for (int m = 0; m < 3; ++m) out12[m * 4 + 3] = (double)n_points;
    return VPT_OK;
}

int vpt_debug_software_sample(vpt_devptr_t d_pool, vpt_devptr_t d_cells, int dx, int dy, int dz, const float* uvw, int n, float* out2) {
    if ((!d_pool && !d_cells) || dx < 1 || dy < 1 || dz < 1 || !uvw || n < 1 || !out2)
        return fail(nullptr, VPT_ERR_INVALID, "vpt_debug_software_sample: bad arguments");
    // the samplers' cell arithmetic is defined on [0, 1] (what volume_coord hands them); NaN fails this test too
    for (size_t i = 0; i < 3 * (size_t)n; ++i)
        if (!(uvw[i] >= 0.0f && uvw[i] <= 1.0f))
            return fail(nullptr, VPT_ERR_INVALID, "vpt_debug_software_sample: coordinate " + std::to_string(i) + " is not in [0, 1]");
    float *d_in = nullptr, *d_out = nullptr;
    cudaError_t e = cudaMalloc(&d_in, sizeof(float) * 3 * (size_t)n);
    if (e == cudaSuccess) e = cudaMalloc(&d_out, sizeof(float) * 2 * (size_t)n);
    if (e == cudaSuccess) e = cudaMemcpy(d_in, uvw, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice);
    const int dims[3] = { dx, dy, dz };
    if (e == cudaSuccess) e = vpt::launch_software_sample(reinterpret_cast<const float*>((uintptr_t)d_pool), reinterpret_cast<const float4*>((uintptr_t)d_cells),
                                                          dims, d_in, n, d_out, 0);
    if (e == cudaSuccess) e = cudaMemcpy(out2, d_out, sizeof(float) * 2 * (size_t)n, cudaMemcpyDeviceToHost);
    cudaFree(d_in); cudaFree(d_out);
    if (e != cudaSuccess) return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_debug_software_sample: ") + cudaGetErrorString(e));
    return VPT_OK;
}

int vpt_cells_create(const float* d_dense, int dx, int dy, int dz, vpt_devptr_t* d_cells_out, unsigned long long* bytes_out) {
    if (!d_dense || !d_cells_out || dx < 1 || dy < 1 || dz < 1) return fail(nullptr, VPT_ERR_INVALID, "vpt_cells_create: bad arguments");
    const size_t n = (size_t)dx * dy * dz;
    float4* cells = nullptr;
    cudaError_t e = cudaMalloc(&cells, n * 32);
    if (e != cudaSuccess) return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_cells_create: ") + std::to_string(n * 32 >> 20) + " MiB: " + cudaGetErrorString(e));
    e = vpt::launch_build_cells(d_dense, dx, dy, dz, cells, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaFree(cells); return fail(nullptr, VPT_ERR_CUDA, std::string("vpt_cells_create: ") + cudaGetErrorString(e)); }
    *d_cells_out = (vpt_devptr_t)(uintptr_t)cells;
    if (bytes_out) *bytes_out = (unsigned long long)n * 32ull;
    return VPT_OK;
}

int vpt_cells_read(vpt_devptr_t d_cells, unsigned long long first_cell, unsigned long long n_cells, float* h_out) {
    if (!d_cells || !h_out) return fail(nullptr, VPT_ERR_INVALID, "vpt_cells_read: null argument");
    VPT_CUDA(nullptr, cudaMemcpy(h_out, reinterpret_cast<const char*>((uintptr_t)d_cells) + first_cell * 32ull, n_cells * 32ull, cudaMemcpyDeviceToHost));
    return VPT_OK;
}

int vpt_cells_destroy(vpt_devptr_t d_cells) { if (d_cells) cudaFree((void*)(uintptr_t)d_cells); return VPT_OK; }

int vpt_set_cell_volume(vpt_context* c, vpt_devptr_t d_cells, int dx, int dy, int dz) {
    if (!c) return VPT_ERR_INVALID;
    if (d_cells && (dx < 1 || dy < 1 || dz < 1)) return fail(c, VPT_ERR_INVALID, "vpt_set_cell_volume: bad dimensions");
    c->cell_table = reinterpret_cast<const float4*>((uintptr_t)d_cells);
    c->cell_dims[0] = dx; c->cell_dims[1] = dy; c->cell_dims[2] = dz;
    // a cell is one 32-byte sector: option "l2_sector_fetch" asks the L2 not to widen a miss to a larger DRAM fetch while this mode is on
    // (cudaLimitMaxL2FetchGranularity, a DEVICE-wide hint: the streaming kernels lose ~4 % with it, so it is not the default)
    if (d_cells && c->l2_sector_fetch) {
        if (!c->l2_fetch_default) cudaDeviceGetLimit(&c->l2_fetch_default, cudaLimitMaxL2FetchGranularity);
        cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
    } else if (c->l2_fetch_default) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, c->l2_fetch_default);
    cudaGetLastError();
    return VPT_OK;
}

int vpt_bricks_destroy(vpt_devptr_t d_pool) { if (d_pool) cudaFree((void*)(uintptr_t)d_pool); return VPT_OK; }

int vpt_set_brick_volume(vpt_context* c, vpt_devptr_t d_pool, int dx, int dy, int dz) {
    if (!c) return VPT_ERR_INVALID;
    if (d_pool && (dx < 1 || dy < 1 || dz < 1)) return fail(c, VPT_ERR_INVALID, "vpt_set_brick_volume: bad dimensions");
    c->brick_pool = reinterpret_cast<const float*>((uintptr_t)d_pool);
    c->brick_dims[0] = dx; c->brick_dims[1] = dy; c->brick_dims[2] = dz;
    return VPT_OK;
}

int vpt_texture_create_env(const float* rgba, unsigned w, unsigned h, vpt_tex_t* tex_out, void** array_out) {
    if (!rgba || !tex_out || !array_out || !w || !h) return fail(nullptr, VPT_ERR_INVALID, "vpt_texture_create_env: bad arguments");
    const cudaChannelFormatDesc desc = cudaCreateChannelDesc<float4>();
    cudaArray_t arr = nullptr;
    VPT_CUDA(nullptr, cudaMallocArray(&arr, &desc, w, h));
    VPT_CUDA(nullptr, cudaMemcpy2DToArray(arr, 0, 0, rgba, (size_t)w * sizeof(float4), (size_t)w * sizeof(float4), h, cudaMemcpyHostToDevice));
    cudaResourceDesc res; memset(&res, 0, sizeof(res));
    res.resType = cudaResourceTypeArray; res.res.array.array = arr;
    cudaTextureDesc td; memset(&td, 0, sizeof(td));
    td.addressMode[0] = cudaAddressModeWrap; td.addressMode[1] = cudaAddressModeClamp; td.addressMode[2] = cudaAddressModeWrap;
    td.filterMode = cudaFilterModeLinear; td.readMode = cudaReadModeElementType; td.normalizedCoords = 1;
    cudaTextureObject_t tex = 0;
    VPT_CUDA(nullptr, cudaCreateTextureObject(&tex, &res, &td, NULL));
    *tex_out = (vpt_tex_t)tex; *array_out = (void*)arr;
    return VPT_OK;
}

// point-sampled, unnormalised float table (h == 0: 1-D array), the descriptor main.cpp:788-867 uses for the env sampling tables
static int create_table_texture(const float* data, unsigned w, unsigned h, vpt_tex_t* tex_out, void** array_out) {
    const cudaChannelFormatDesc desc = cudaCreateChannelDesc<float>();
    cudaArray_t arr = nullptr;
    VPT_CUDA(nullptr, cudaMallocArray(&arr, &desc, w, h));
    VPT_CUDA(nullptr, cudaMemcpy2DToArray(arr, 0, 0, data, (size_t)w * sizeof(float), (size_t)w * sizeof(float), h ? h : 1, cudaMemcpyHostToDevice));
    cudaResourceDesc res; memset(&res, 0, sizeof(res));
    res.resType = cudaResourceTypeArray; res.res.array.array = arr;
    cudaTextureDesc td; memset(&td, 0, sizeof(td));
    td.addressMode[0] = cudaAddressModeWrap; td.addressMode[1] = h ? cudaAddressModeClamp : cudaAddressModeWrap; td.addressMode[2] = cudaAddressModeWrap;
    td.filterMode = cudaFilterModePoint; td.readMode = cudaReadModeElementType; td.normalizedCoords = 0;
    cudaTextureObject_t tex = 0;
    VPT_CUDA(nullptr, cudaCreateTextureObject(&tex, &res, &td, NULL));
    *tex_out = (vpt_tex_t)tex; *array_out = (void*)arr;
    return VPT_OK;
}

// Host arithmetic of create_cdf (main.cpp:681-757), pointer walk restated with indices.  The reference reads one element
// BEFORE two of its arrays (quirk Q20): `*(func_p - 1)` at y == 0, x == 0 and `*(marginal_cdf_p - 1)` at y == 0; those two reads
// are taken as 0 here (in the reference they hit the allocator's bookkeeping word: a denormal).  Everything else is literal:
//   * row y > 0 starts from func[y-1][res-1] / res, because `*(func_p - 1)` at x == 0 is the LAST element of the previous row
//     (in range), and that offset is carried through the row's cdf and into marginal_func[y];
//   * `*(cdf_p - 1) = 0` at each row start zeroes the previous row's last cdf entry, which the normalisation then sets to 1;
//   * the "total" that selects the uniform fallback is res x marginal_func[0] (the loop never advances its pointer).
int vpt_env_tables_compute(const float* func, unsigned res, float* cdf, float* marginal_func, float* marginal_cdf, float* marginal_int_out) {
    if (!func || res < 2 || !cdf || !marginal_func || !marginal_cdf || !marginal_int_out) return fail(nullptr, VPT_ERR_INVALID, "vpt_env_tables_compute: bad arguments");
    const float fres = (float)res;
    for (unsigned y = 0; y < res; ++y) {
        float prev_cdf = 0.0f;                                          // *(cdf_p - 1) = .0f
        if (y > 0) cdf[(size_t)y * res - 1] = 0.0f;
        for (unsigned x = 0; x < res; ++x) {
            const float prev_func = (x == 0 && y == 0) ? 0.0f : func[(size_t)y * res + x - 1];
            prev_cdf = prev_cdf + prev_func / fres;
            cdf[(size_t)y * res + x] = prev_cdf;
        }
        marginal_func[y] = prev_cdf;
    }
    float total_int = 0.0f;
    for (unsigned j = 0; j < res; ++j) total_int += marginal_func[0];
    if (total_int == 0.0f) {
        for (unsigned y = 0; y < res; ++y) for (unsigned x = 0; x < res; ++x) cdf[(size_t)y * res + x] = ((float)x / fres) * ((float)y / fres);
    } else {
        for (unsigned y = 0; y < res; ++y) for (unsigned x = 0; x < res; ++x) {
            float& c = cdf[(size_t)y * res + x];
            c /= marginal_func[y];
            if (x == res - 1) c = 1.0f;
        }
    }
    float run = 0.0f;                                                   // *(marginal_cdf_p - 1) at y == 0: out of range, taken as 0
    for (unsigned y = 0; y < res; ++y) { run = run + marginal_func[y] / fres; marginal_cdf[y] = run; }
    const float marginal_int = run;
    if (marginal_int > 0.0f) for (unsigned y = 0; y < res; ++y) marginal_cdf[y] /= std::max(.000001f, marginal_int);
    else marginal_cdf[0] = 1.0f;                                        // the reference's trailing `*marginal_cdf_p = 1.0f` lands here when the loop is skipped
    *marginal_int_out = marginal_int;
    return VPT_OK;
}

int vpt_env_tables_create(const float* func, unsigned res, vpt_tex_t tex_out[4], void* arrays_out[4], float* marginal_int_out) {
    if (!func || res < 2 || !tex_out || !arrays_out || !marginal_int_out) return fail(nullptr, VPT_ERR_INVALID, "vpt_env_tables_create: bad arguments");
    const size_t n = (size_t)res * res;
    std::vector<float> cdf(n), mfunc(res), mcdf(res);
    int rc0 = vpt_env_tables_compute(func, res, cdf.data(), mfunc.data(), mcdf.data(), marginal_int_out);
    if (rc0 != VPT_OK) return rc0;
    const float* src[4] = { func, cdf.data(), mfunc.data(), mcdf.data() };
    const unsigned heights[4] = { res, res, 0u, 0u };
    for (int i = 0; i < 4; ++i) { tex_out[i] = 0; arrays_out[i] = nullptr; }
    for (int i = 0; i < 4; ++i) {
        const int rc = create_table_texture(src[i], res, heights[i], &tex_out[i], &arrays_out[i]);
        if (rc != VPT_OK) {                                       // leave nothing half-built behind
            for (int j = 0; j < i; ++j) { vpt_texture_destroy(tex_out[j], arrays_out[j]); tex_out[j] = 0; arrays_out[j] = nullptr; }
            return rc;
        }
    }
    return VPT_OK;
}

int vpt_texture_destroy(vpt_tex_t tex, void* array) {
    if (tex) cudaDestroyTextureObject((cudaTextureObject_t)tex);
    if (array) cudaFreeArray((cudaArray_t)array);
    return VPT_OK;
}

void vpt_free(void* p) { free(p); }

int vpt_ins_load(const char* path, vpt_ins_header** out) {
    if (!path || !out) return fail(nullptr, VPT_ERR_INVALID, "vpt_ins_load: null argument");
    *out = nullptr;
    std::ifstream f(path);
    if (!f) return fail(nullptr, VPT_ERR_IO, std::string("vpt_ins_load: cannot open ") + path);
    auto bad = [&](const std::string& what) { return fail(nullptr, VPT_ERR_IO, std::string("vpt_ins_load: ") + path + ": " + what); };
    auto numbers = [](const std::string& line, double* v, int n) { std::istringstream is(line); for (int i = 0; i < n; ++i) if (!(is >> v[i])) return false; return true; };
    std::string line;
    if (!std::getline(f, line)) return bad("empty file");
    while (!line.empty() && (line.back() == '\r' || line.back() == ' ' || line.back() == '\t')) line.pop_back();
    std::vector<vpt_ins_file_entry> files;
    std::vector<double> recs;
    int kind = 0;
    if (line == "light") {
        kind = 1;
        double n = 0;
        if (!std::getline(f, line) || !numbers(line, &n, 1) || n < 0 || n > 1e7) return bad("light count missing");
        for (int i = 0; i < (int)n; ++i) {
            double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (!std::getline(f, line) || !numbers(line, v, 7)) return bad("light record " + std::to_string(i) + " needs 7 numbers: px py pz r g b power");
            recs.insert(recs.end(), v, v + 8);
        }
    } else {
        double n = 0;
        if (!numbers(line, &n, 1) || n < 0 || n > 1e6) return bad("first line must be \"light\" or the number of .vdb entries");
        for (int i = 0; i < (int)n; ++i) {
            vpt_ins_file_entry e; memset(&e, 0, sizeof(e));
            if (!std::getline(f, line)) return bad("missing .vdb path of entry " + std::to_string(i));
            while (!line.empty() && (line.back() == '\r')) line.pop_back();
            if (line.size() >= sizeof(e.path)) return bad("path too long");
            memcpy(e.path, line.c_str(), line.size());
            double cnt = 0;
            if (!std::getline(f, line) || !numbers(line, &cnt, 1) || cnt < 0 || cnt > 1e7) return bad("missing instance count of entry " + std::to_string(i));
            e.first_record = (int32_t)(recs.size() / 8); e.n_instances = (int32_t)cnt;
            for (int x = 0; x < (int)cnt; ++x) {
                double v[8];
                if (!std::getline(f, line) || !numbers(line, v, 8)) return bad("instance " + std::to_string(x) + " of entry " + std::to_string(i) + " needs 8 numbers: px py pz qx qy qz qw scale");
                recs.insert(recs.end(), v, v + 8);
            }
            files.push_back(e);
        }
    }
    const size_t bytes = sizeof(vpt_ins_header) + files.size() * sizeof(vpt_ins_file_entry) + recs.size() * sizeof(double);
    char* blk = (char*)malloc(bytes);
    if (!blk) return fail(nullptr, VPT_ERR_IO, "vpt_ins_load: out of memory");
    vpt_ins_header h; h.kind = kind; h.n_files = (int32_t)files.size(); h.n_records = (int32_t)(recs.size() / 8); h.reserved = 0;
    memcpy(blk, &h, sizeof(h));
    if (!files.empty()) memcpy(blk + sizeof(h), files.data(), files.size() * sizeof(vpt_ins_file_entry));
    if (!recs.empty()) memcpy(blk + sizeof(h) + files.size() * sizeof(vpt_ins_file_entry), recs.data(), recs.size() * sizeof(double));
    *out = reinterpret_cast<vpt_ins_header*>(blk);
    return VPT_OK;
}

int vpt_vdb_load(const char* path, const char* grid_name, float** values_out, int info[13], float xform16[16], float stats[4]) {
    if (!path || !grid_name || !values_out) return fail(nullptr, VPT_ERR_INVALID, "vpt_vdb_load: null argument");
    *values_out = nullptr;
    std::ifstream f(path, std::ios::binary);
    if (!f) return fail(nullptr, VPT_ERR_IO, std::string("vpt_vdb_load: cannot open ") + path);
    std::vector<uint8_t> data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    vpt::VdbDenseGrid g;
    try {
        if (!vpt::vdb_read_dense(data.data(), data.size(), grid_name, g)) return 1;
    } catch (const std::exception& e) { return fail(nullptr, VPT_ERR_IO, std::string("vpt_vdb_load: ") + e.what()); }
    // cross-check against the file's own metadata (the only pin the format offers)
    if (g.meta.has_file_bbox)
        for (int a = 0; a < 3; ++a)
            if (g.meta.file_bbox_min[a] != g.bbox_min[a] || g.meta.file_bbox_max[a] != g.bbox_max[a])
                return fail(nullptr, VPT_ERR_IO, "vpt_vdb_load: decoded active bbox disagrees with file_bbox metadata");
    if (g.meta.file_voxel_count >= 0 && (uint64_t)g.meta.file_voxel_count != g.active_leaf_voxels + g.active_tile_voxels)
        return fail(nullptr, VPT_ERR_IO, "vpt_vdb_load: decoded active voxel count disagrees with file_voxel_count metadata");
    const size_t nfl = g.values.size();
    float* out = (float*)malloc(nfl * sizeof(float));
    if (!out) return fail(nullptr, VPT_ERR_IO, "vpt_vdb_load: out of memory");
    memcpy(out, g.values.data(), nfl * sizeof(float));
    *values_out = out;
    if (info) {
        for (int a = 0; a < 3; ++a) { info[a] = g.dim[a]; info[3 + a] = g.bbox_min[a]; info[6 + a] = g.bbox_max[a]; }
        info[9] = g.channels; info[10] = (int)g.leaf_count;
        const uint64_t act = g.active_leaf_voxels + g.active_tile_voxels;
        info[11] = (int)(act & 0xffffffffu); info[12] = (int)(act >> 32);
    }
    if (xform16) {
        // convert_to_mat4: xform[i][j] = float(M(j, i)) with M the OpenVDB row-vector Mat4 => memory image m[c][r] = M[r][c]
        for (int j = 0; j < 4; ++j) for (int i = 0; i < 4; ++i) xform16[i * 4 + j] = float(g.index_to_world[j * 4 + i]);
    }
    if (stats) {
        float mx = 0.0f, mn = FLT_MAX;                      // VDB_INFO defaults then the scan of gpu_vdb.cpp:206-207 (first channel)
        const size_t ch = (size_t)g.channels;
        for (size_t i = 0; i < nfl; i += ch) { const float v = g.values[i]; mx = fmaxf(mx, v); mn = fminf(fmaxf(FLT_EPSILON, v), mn); }
        stats[0] = mx; stats[1] = mn; stats[2] = (float)g.voxel_size[0]; stats[3] = g.background[0];
    }
    return VPT_OK;
}

int vpt_hdr_load(const char* path, float** rgba_out, unsigned* w, unsigned* h) {
    if (!path || !rgba_out || !w || !h) return fail(nullptr, VPT_ERR_INVALID, "vpt_hdr_load: null argument");
    std::vector<float> px; std::string err;
    if (!vpt::load_hdr_float4(path, px, *w, *h, err)) return fail(nullptr, VPT_ERR_IO, "vpt_hdr_load: " + err);
    *rgba_out = (float*)malloc(px.size() * sizeof(float)); memcpy(*rgba_out, px.data(), px.size() * sizeof(float));
    return VPT_OK;
}

int vpt_bmp_load_rbg(const char* path, float** xyz_out, int* w, int* h) {
    if (!path || !xyz_out || !w || !h) return fail(nullptr, VPT_ERR_INVALID, "vpt_bmp_load_rbg: null argument");
    std::vector<float> px; std::string err;
    if (!vpt::load_bmp_float3_rbg(path, px, *w, *h, err)) return fail(nullptr, VPT_ERR_IO, "vpt_bmp_load_rbg: " + err);
    *xyz_out = (float*)malloc(px.size() * sizeof(float)); memcpy(*xyz_out, px.data(), px.size() * sizeof(float));
    return VPT_OK;
}

int vpt_exr_load_rgb(const char* path, float** rgb_out, int* w, int* h) {
    if (!path || !rgb_out || !w || !h) return fail(nullptr, VPT_ERR_INVALID, "vpt_exr_load_rgb: null argument");
    std::vector<float> px; std::string err;
    if (!vpt::load_exr_float3(path, px, *w, *h, err)) return fail(nullptr, VPT_ERR_IO, "vpt_exr_load_rgb: " + err);
    *rgb_out = (float*)malloc(px.size() * sizeof(float)); memcpy(*rgb_out, px.data(), px.size() * sizeof(float));
    return VPT_OK;
}

void vpt_camera_look_at(vpt_camera* cam, const float lookfrom[3], const float lookat[3], const float vup[3], float vfov, float aspect, float aperture) {
    auto sub = [](const float* a, const float* b, float* o) { o[0] = a[0] - b[0]; o[1] = a[1] - b[1]; o[2] = a[2] - b[2]; };
    auto len = [](const float* a) { return sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); };
    auto norm = [&](float* a) { const float inv = 1.0f / sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); a[0] *= inv; a[1] *= inv; a[2] *= inv; };
    auto cross = [](const float* a, const float* b, float* o) { o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0]; };
    memset(cam, 0, sizeof(*cam));
    cam->time0 = .0f; cam->time1 = 1.0f;
    float d[3]; sub(lookfrom, lookat, d);
    const float focus = len(d);
    cam->focus_dist = focus;
    cam->lens_radius = aperture / 2.0f;
    const float theta = vfov * float(M_PI) / 180.0f;
    const float half_height = (float)tan(theta / 2.0f);
    const float half_width = aspect * half_height;
    float w[3] = { d[0], d[1], d[2] }; norm(w);
    float u[3]; cross(vup, w, u); norm(u);
    float v[3]; cross(w, u, v);
    for (int a = 0; a < 3; ++a) {
        (&cam->origin.x)[a] = lookfrom[a];
        (&cam->u.x)[a] = u[a]; (&cam->v.x)[a] = v[a]; (&cam->w.x)[a] = w[a];
        (&cam->lower_left_corner.x)[a] = lookfrom[a] - half_width * focus * u[a] - half_height * focus * v[a] - focus * w[a];
        (&cam->horizontal.x)[a] = 2.0f * half_width * focus * u[a];
        (&cam->vertical.x)[a] = 2.0f * half_height * focus * v[a];
    }
    cam->viz_dof = 0;
}

void vpt_kernel_params_defaults(vpt_kernel_params* kp) {
    memset(kp, 0, sizeof(*kp));
    kp->render = 1; kp->iteration = 0; kp->max_interactions = 100; kp->exposure_scale = 1.0f;
    kp->environment_type = 0; kp->ray_depth = 50; kp->volume_depth = 1;
    kp->phase_g1 = 0.0f; kp->phase_g2 = 0.0f; kp->phase_f = 1.0f; kp->tr_depth = 1.0f; kp->density_mult = 1.0f;
    kp->albedo = {1.0f, 1.0f, 1.0f}; kp->extinction = {1.0f, 1.0f, 1.0f};
    kp->azimuth = 120.0f; kp->elevation = 30.0f;            // ImGui values that overwrite 150/30 every frame (main.cpp:1420-1421, 1538-1539)
    kp->sun_color = {1.0f, 1.0f, 1.0f}; kp->sun_mult = 1.0f;
    kp->energy_inject = 1.0;                                 // main.cpp:1543 (energy == 0)
    kp->sky_color = {1.0f, 1.0f, 1.0f}; kp->sky_mult = 1.0f;
    kp->env_sample_tex_res = 360; kp->integrator = 0; kp->emission_scale = 0.0f; kp->emission_pivot = 1.0f;
}

} // extern "C"
