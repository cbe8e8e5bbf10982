// vpt_kernels.h -- launch interface between the host context (csrc/host) and the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/vpt_abi.h"
#include "vpt_scene.cuh"

namespace vpt {

constexpr int kTraceThreads = 128;                    // CTA size of the trace kernels but the lean ones at 2 rays per lane (trace_threads)
#ifndef VPT_TRACE_MIN_CTAS
#define VPT_TRACE_MIN_CTAS 4
#endif
constexpr int kTraceMinCtas = VPT_TRACE_MIN_CTAS;     // __launch_bounds__ hint: 4 CTAs x (51 KB ray slots + 4 KB tables) and <= 128 registers per thread

// The shape of a k_trace instantiation (DESIGN.md section 4): CTA size, CTAs per SM (the __launch_bounds__ minimum, which sets the
// register budget) and the words each parked ray takes in shared memory.  The lean kernels at 2 rays per lane park a 29-word record
// (vpt_trace.cuh, PoolLean) and run one of three shapes, VPT_LEAN2_SHAPE (DESIGN.md section 4 has the timings): 2, the default = 4 CTAs
// of 224 threads (28 warps, <= 72 registers); 0 = 3 CTAs of 256 threads (24 warps, <= 80 registers) under the driver's carveout (228 KB:
// 28 KB of L1); 1 = the same CTAs under the 196 KB carveout, which leaves the L1 60 KB.  The cell-table kernel keeps 3 CTAs of 256 threads
// in every shape: at 72 registers its stepping loop spills.
#ifndef VPT_LEAN2_SHAPE
#define VPT_LEAN2_SHAPE 2
#endif
constexpr int kRayWords = 34;                         // 32-bit words per parked ray (every kernel but the lean ones at 2 rays per lane)
constexpr int kLeanRayWords = 29;                     // ... and in the lean kernels at 2 rays per lane
constexpr int kTraceTablesBytes = 4352;               // static shared memory of k_trace: FrameShared and the empty-ahead table (asserted)
constexpr int kSmemPerSm = 233472;                    // shared memory an SM offers to its CTAs (228 KB), and the 1 KB reserved per CTA
constexpr int kSmemReservePerCta = 1024;
constexpr bool trace_28_warps(bool lean, int slots, bool cells) { return lean && slots == 2 && !cells && VPT_LEAN2_SHAPE == 2; }
constexpr int trace_threads(bool lean, int slots, bool cells = false) { return lean && slots == 2 ? (trace_28_warps(lean, slots, cells) ? 224 : 256) : kTraceThreads; }
constexpr int trace_min_ctas(bool lean, int slots, bool cells = false) { return slots != 2 ? kTraceMinCtas : lean ? (trace_28_warps(lean, slots, cells) ? 4 : 3) : 5; }
constexpr int trace_ray_words(bool lean, int slots) { return lean && slots == 2 ? kLeanRayWords : kRayWords; }
// the opt-in dynamic shared memory of an instantiation: its warps' parked rays
constexpr size_t trace_smem_bytes(bool lean, int slots, bool cells = false) { return (size_t)(trace_threads(lean, slots, cells) / 32) * trace_ray_words(lean, slots) * 32 * slots * sizeof(float); }
// the shared memory trace_min_ctas CTAs take on an SM, and the carveout (percent of kSmemPerSm) the lean kernels at 2 rays per lane ask
// for under VPT_LEAN2_SHAPE 1: the least that holds them.  The driver rounds a carveout up to the next capacity the SM supports (..., 164, 196, 228 KB).
constexpr size_t trace_sm_smem_bytes(bool lean, int slots, bool cells = false) { return (size_t)trace_min_ctas(lean, slots, cells) * (trace_smem_bytes(lean, slots, cells) + kTraceTablesBytes + kSmemReservePerCta); }
constexpr int trace_carveout_percent(bool lean, int slots, bool cells = false) { return (int)((trace_sm_smem_bytes(lean, slots, cells) * 100 + kSmemPerSm - 1) / kSmemPerSm); }

// Which pixels this rank renders: rows are dealt to ranks in interleaved stripes of `stripe_h` rows
// (rank r owns stripes r, r+R, r+2R, ...).  One rank: identity mapping, local == global indices.
struct FrameGeom {
    int width, height;      // full frame
    int local_rows;         // rows stored locally (padded so every rank holds the same count)
    int n_local;            // local_rows * width
    int stripe_h, n_ranks, rank;
};

// Everything a per-frame kernel needs, passed by value (about 600 B of kernel parameter space).
struct FrameArgs {
    vpt_camera        cam;
    vpt_light_list    lights;
    vpt_kernel_params kp;          // buffers inside are indexed by LOCAL pixel
    const vpt_sphere* sphere;
    const SceneTables* scene;
    FrameGeom         geom;
    // ray queue (hits), SoA: direction + entry distance | (local pixel, pass | draws<<6 | obj<<16) | origin (thin lens only)
    float4*   queue_dir;
    uint2*    queue_id;
    float4*   queue_aux;           // per-ray origin (thin lens or camera motion); pre-stepped ray (pinhole only): position where stepping starts
    int       thin_lens;           // per-ray origin: thin lens or camera motion (cam.lens_radius != 0 or a CameraMotion)
    // vpt_set_sample_offset: pass p of the call draws the Philox stream of iteration sample_offset + kp.iteration + p (everything else keeps
    // kp.iteration).  Read by the motion-vector kernels, which need both; k_generate* and k_trace* read kp.iteration only as the stream key,
    // so the host hands them the stream iteration in kp.iteration instead (stream_args in vpt_context.cpp) and their code stays as it was.
    // In the 4-byte hole after thin_lens: the block has no tail padding, so a field at its end would move the kernel parameters that follow
    // FrameArgs in every kernel, while the hole moves no offset at all.
    uint32_t  sample_offset;
    // (option "empty_ahead" reaches the kernels through the table behind `scene`: SceneAlloc, launch_empty_ahead)
    const float2* bn_table;       // [pass][65536] blue-noise jitter of the chunk
    int       n_passes;            // passes in this chunk (k_generate loops over them; k_trace keeps tr of the last one)
    int       passes_per_block;    // k_generate: passes handled by one block (blockIdx.z selects the run)
    int       debug_flags;         // development switches (0 in production)
    int       sched_min_lanes;     // trace scheduler: lanes an operation must gather before it pre-empts stepping
    unsigned* queue_count;
    unsigned* queue_head;
    // sample planes, [pass][local pixel].  Wide records (the frame ends on the precomputed sky: k_resolve<1/2>): A = final direction + tr,
    // B = L + depth, C = beta, D = env_pos.  Compact records (HDRI frames traced by a lean kernel; planeB/C/D null): A = the finished radiance
    // + depth, and plane_tr (below) holds tr of the hit samples of the chunk's last pass.  A miss is always A = direction + kMissSentinel.
    float4 *planeA, *planeB, *planeC, *planeD;
    // optional statistics: [0] volume lookups, [1] lane-steps, [2] warp step iterations, [3] lane transitions, [4] warp transition rounds,
    // [5] rays, [6] brick fetches, [8..10] k_trace hops of delta / ratio / emission walks, [11] k_trace walks ended by "empty ahead",
    // [12..14] k_generate pre-step rays / hops / rays ended by "empty ahead" (16 counters)
    unsigned long long* counters;
    // cell table of volume 0 (vpt_cells_create; null = texture path): per texel cell its eight corner values, 32 bytes = ONE sector per look-up
    const float4* cell_table;
    int       cell_nx, cell_ny, cell_nz;
    int       tiles_per_block;     // k_generate: consecutive 32x4 tiles handled by one block (blockIdx.x selects the run)
    float*    plane_tr;            // compact records: [local pixel] tr of the hit samples of pass n_passes - 1 (k_resolve writes it to raw.w)
    // [local pixel] 1 = k_miss_cull proved that every jitter of the pixel misses the root box and the sphere: k_generate samples nothing
    // there and k_resolve<0> (k_resolve_equirect) rebuilds the pinhole (equirectangular) miss samples.  Null = nothing culled (option
    // "miss_cull" 0, thin lens, sky frames).
    const uint8_t* miss_mask;
};

// Adaptive sampling (vpt_render_adaptive): pixels are grouped in the 32x4 tiles k_generate works on; a chunk only visits the tiles that
// still hold an active pixel.  Per pixel the context keeps a float32 Welford state of the sample luminance {n, mean, M2, err}.
constexpr float kAdaptMeanFloor = 1e-3f;   // err = sqrt(M2 / (n (n-1))) / max(mean, kAdaptMeanFloor): dark pixels are judged on absolute error
struct AdaptArgs {
    const unsigned* tiles;         // active tiles of this chunk (tile = tile_y * tiles_x + tile_x), `n_tiles` entries
    int       n_tiles;
    uint8_t*  stopped;             // [local pixel] 1 once the pixel has stopped
    float4*   stat;                // [local pixel] n, mean, M2, err
    unsigned* pass_count;          // [local pixel] passes taken (the caller's buffer)
    float*    rel_error;           // [local pixel] last err (the caller's buffer, may be null)
    unsigned* next_tiles;          // k_adapt: tiles still active after the test, appended in any order
    unsigned* next_count;          //          their number (zeroed by the host before the launch)
    float     threshold;
};

// Render region (vpt_set_render_region): a call samples and writes only the global pixels [x0, x1) x [y0, y1).  global_row increases with
// the local row, so R and this rank's stripes meet in the local rows [lr0, lr1) (lr0 == lr1: none), and the 32x4 tiles of the local frame
// that hold a pixel of R are the rectangle [tx0, tx1) x [ty0, ty1) -- every tile of it holds at least one.  A kernel argument of the region
// kernels only (k_generate_region, k_miss_cull_region, k_resolve_region, k_adapt_init_region, k_adapt_region), as AovBuffers is.
struct RenderRegion {
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    int lr0 = 0, lr1 = 0;
    int tx0 = 0, ty0 = 0, tx1 = 0, ty1 = 0;
};
// the number of local rows whose global row is below y (0 <= y <= height): the first local row at or past global row y
inline int region_local_row(const FrameGeom& g, int y)
{
    const int s = y / g.stripe_h, own = s % g.n_ranks;                 // the stripe of row y and the rank that owns it
    const int lr = own == g.rank ? (s / g.n_ranks) * g.stripe_h + (y - s * g.stripe_h)
                                 : ((s + (g.rank - own + g.n_ranks) % g.n_ranks) / g.n_ranks) * g.stripe_h;   // next stripe of this rank
    return lr < g.local_rows ? lr : g.local_rows;
}
// R's local rows and tile rectangle on this rank; the caller has checked x0 < x1 <= width and y0 < y1 <= height
inline RenderRegion region_geometry(const FrameGeom& g, int x0, int y0, int x1, int y1)
{
    RenderRegion r;
    r.x0 = x0; r.y0 = y0; r.x1 = x1; r.y1 = y1;
    r.lr0 = region_local_row(g, y0); r.lr1 = region_local_row(g, y1);
    if (r.lr0 < r.lr1) { r.tx0 = x0 / 32; r.tx1 = (x1 + 31) / 32; r.ty0 = r.lr0 / 4; r.ty1 = (r.lr1 + 3) / 4; }
    return r;
}
inline long long region_tiles(const RenderRegion& r) { return (long long)(r.tx1 - r.tx0) * (r.ty1 - r.ty0); }
inline long long region_pixels(const RenderRegion& r) { return (long long)(r.x1 - r.x0) * (r.lr1 - r.lr0); }

// Camera projection (vpt_set_projection).  kind: kProjPerspective (the reference camera) or kProjEquirect, whose ray through pixel (x, y)
// at jitter (jx, jy) has the direction pano_b0 (vpt_frame.cuh); hfov / vfov in radians.  A kernel argument of the equirectangular kernels
// only (k_generate_equirect, k_miss_cull_equirect, k_resolve_equirect, ...: the launchers below pick them for kProjEquirect), as
// RenderRegion is, so every other kernel keeps its parameter block.
constexpr int kProjPerspective = 0, kProjEquirect = 1;          // VPT_PROJECTION_PERSPECTIVE, VPT_PROJECTION_EQUIRECT of vpt_b200.h
struct Projection { int kind = kProjPerspective; float hfov = 0.f, vfov = 0.f; };
inline bool equirect(const Projection& p) { return p.kind == kProjEquirect; }

// Camera motion (vpt_set_camera_motion): the camera's pose at shutter close.  A sample with shutter draw xi uses the camera whose six
// fields below are motion_camera's lerp (vpt_frame.cuh) from the frame camera (the pose at shutter open) towards these.  A kernel argument
// of the motion kernels only (k_generate_motion, k_generate_adaptive_motion, k_generate_region_motion, k_motion_cameras: the launchers below
// pick them for a non-null CameraMotion), as Projection is.
struct CameraMotion { vpt_f3 origin, lower_left_corner, horizontal, vertical, u, v; };

// Omni-directional stereo (vpt_set_projection_ods): Projection::kind is kProjOds, and these are the rest of the projection.  Each sample's
// camera is ods_camera's (vpt_frame.cuh): the panorama of (hfov, vfov) per eye, its origin moved by +-half_ipd * k along the viewer's
// right, k the pole merge (1 up to |theta| = merge_from, 0 from merge_to on, (merge_to - |theta|) * inv_span in between; angles in
// radians).  A kernel argument of the ODS kernels only (k_generate_ods, k_generate_adaptive_ods, k_generate_region_ods, k_ods_cameras: the
// launchers below pick them for a non-null OdsParams), as Projection is.
constexpr int kProjOds = 2;                                       // VPT_PROJECTION_ODS of vpt_b200.h
constexpr int kOdsLeft = 0, kOdsRight = 1, kOdsOverUnder = 2;     // VPT_ODS_LEFT, VPT_ODS_RIGHT, VPT_ODS_OVER_UNDER
struct OdsParams { float hfov = 0.f, vfov = 0.f, half_ipd = 0.f; int layout = kOdsOverUnder; float merge_from = 0.f, merge_to = 0.f, inv_span = 0.f; };
inline bool ods(const Projection& p) { return p.kind == kProjOds; }

cudaError_t launch_prepare_scene(const vpt_gpu_vdb* vols, const vpt_octnode* root, SceneTables* out, OctInternal* internal,
                                 uint2* leaf_list, int* leaf_indices, VolumeRec* vrec, int max_volumes, cudaStream_t s);
cudaError_t launch_prepare_volumes(const vpt_gpu_vdb* vols, const SceneTables& hdr, SceneTables* out, VolumeRec* vrec, cudaStream_t s);
// pj: the frame's projection -- the launchers below run the equirectangular kernels when equirect(pj); mo: the frame's shutter-close pose
// (null: no motion) -- the generate launchers run the motion kernels when it is set (never together with equirect(pj): the host refuses that);
// od: the frame's ODS projection (null unless ods(pj)) -- the generate, cull and resolve launchers run the ODS kernels when it is set (never
// with motion)
cudaError_t launch_generate(const FrameArgs& fa, int n_passes, const Projection& pj, const CameraMotion* mo, const OdsParams* od, cudaStream_t s);
// once per render call, after the scene tables: the empty-ahead table of option "empty_ahead" (enable) into the context's SceneAlloc,
// whose first member `scene` is
cudaError_t launch_empty_ahead(SceneTables* scene, int enable, cudaStream_t s);
// once per render call, before the first chunk: mask[local pixel] = 1 where every jitter misses the root box and the sphere (pinhole
// and equirectangular cameras; a thin lens or a root box that is empty or not finite culls nothing)
// od: the frame's ODS projection (null unless ods(pj)) -- the cull and resolve launchers below run the ODS kernels when it is set
cudaError_t launch_miss_cull(const FrameArgs& fa, uint8_t* mask, const Projection& pj, cudaStream_t s, const OdsParams* od = nullptr);
struct LightGroups;
// The trace kernels, with their instantiations in trace_kernel (vpt_kernels.cu): generic / lean / volumetric path at 3 rays per lane,
// k_trace_brick, generic / lean at 2, lean at 2 on the cell table, generic / volumetric path keeping the light-group planes.
// kTraceKernels counts those; the *_MATTES kernels after them are the same with the id plane of the instance mattes and the Cryptomatte (MatteIds, below), and
// kTraceKernelsAll counts every trace kernel.
enum TraceKernel : int { TK_GENERIC_3, TK_LEAN_3, TK_VOL_3, TK_BRICK, TK_GENERIC_2, TK_LEAN_2, TK_LEAN_2_CELLS, TK_GENERIC_3_GROUPS,
                         TK_VOL_3_GROUPS, kTraceKernels,
                         TK_LEAN_3_MATTES = kTraceKernels, TK_LEAN_2_MATTES, TK_GENERIC_3_MATTES, TK_VOL_3_MATTES, TK_GENERIC_3_GROUPS_MATTES,
                         TK_VOL_3_GROUPS_MATTES, TK_GENERIC_2_MATTES, kTraceKernelsAll };
// The trace kernel of a frame.  brick / cells: volume 0 is read from a brick pool / a cell table (lean scenes only); vol_integ: the volumetric
// path integrator; group_planes: a generic kernel keeps the light-group planes; slots: rays per lane, 2 or 3 (the group kernels run 3);
// mattes: the kernel writes the instance mattes' id plane (never with brick or cell mode: the host refuses that), at the rays per lane of
// the same frame without mattes.
inline TraceKernel pick_trace_kernel(bool brick, bool cells, bool vol_integ, bool lean, bool group_planes, int slots, bool mattes = false)
{
    if (mattes) {
        if (group_planes) return vol_integ ? TK_VOL_3_GROUPS_MATTES : TK_GENERIC_3_GROUPS_MATTES;
        if (vol_integ) return TK_VOL_3_MATTES;
        if (slots == 2) return lean ? TK_LEAN_2_MATTES : TK_GENERIC_2_MATTES;
        return lean ? TK_LEAN_3_MATTES : TK_GENERIC_3_MATTES;
    }
    if (group_planes) return vol_integ ? TK_VOL_3_GROUPS : TK_GENERIC_3_GROUPS;
    if (brick) return TK_BRICK;
    if (cells) return TK_LEAN_2_CELLS;
    if (vol_integ) return TK_VOL_3;
    if (slots == 2) return lean ? TK_LEAN_2 : TK_GENERIC_2;
    return lean ? TK_LEAN_3 : TK_GENERIC_3;
}
// rays per lane of a k_trace instantiation (2 or 3); 0 for k_trace_brick, which parks no rays per lane
inline int trace_rays_per_lane(TraceKernel k)
{
    switch (k) {
    case TK_BRICK: return 0;
    case TK_GENERIC_2: case TK_LEAN_2: case TK_LEAN_2_CELLS: case TK_LEAN_2_MATTES: case TK_GENERIC_2_MATTES: return 2;
    default: return 3;
    }
}
// default of option "sched_min_lanes": lanes an operation must gather before it pre-empts stepping (26 helps only the lean kernel at 3)
inline int trace_sched_min_lanes(TraceKernel k) { return k == TK_LEAN_3 || k == TK_LEAN_3_MATTES ? 26 : 20; }
// per device: dynamic shared memory opt-in of every trace kernel, and how many CTAs of each fit on an SM
cudaError_t trace_kernels_init(int max_ctas[kTraceKernelsAll]);
// Instance mattes, trace side (vpt_set_instance_mattes): id[pass * n_local + local pixel] = the id of a sample whose camera ray collided
// (depth > 0): kMatteSphereId when the camera ray hit the sphere before the volume box, else the volume instance of the first walk's
// accepted collision (the first leaf-list entry whose density prefix passes the acceptance test).  Written only where depth > 0 will hold.
// A kernel argument of the matte instantiations of k_trace only (the last of the pack), as LightGroups is.
constexpr uint32_t kMatteSphereId = 0xffffffffu;
struct MatteIds { uint32_t* id = nullptr; };
// kernel k on n_ctas persistent CTAs.  atm: the caller's AtmosphereParameters (volumetric path kernels); lg: the light groups (group
// kernels); mi: the id plane (matte kernels); brick_pool / brick_dims: the brick pool of volume 0 and its voxels per axis (k_trace_brick)
cudaError_t launch_trace(const FrameArgs& fa, TraceKernel k, const vpt_atmosphere& atm, const LightGroups& lg, const MatteIds& mi,
                         const float* brick_pool, const int brick_dims[3], int n_ctas, cudaStream_t s);
cudaError_t launch_sampler_compare(unsigned long long tex, const float* pool, const int dims[3], int n, unsigned seed, double* d_out12, cudaStream_t s);
// brick_sample / cell_sample at n points d_uvw [n][3] in [0, 1]: d_out2 [n][2] (k_software_sample); pool or cells may be null
cudaError_t launch_software_sample(const float* pool, const float4* cells, const int dims[3], const float* d_uvw, int n, float* d_out2, cudaStream_t s);
cudaError_t launch_fill_perlin(float* d_buffer, int dx, int dy, int dz, float scale, int seed, cudaStream_t s);
cudaError_t launch_build_bricks(const float* d_dense, int dx, int dy, int dz, float* d_bricks, cudaStream_t s);
cudaError_t launch_build_cells(const float* d_dense, int dx, int dy, int dz, float4* d_cells, cudaStream_t s);
// Peer-memory exchange (multi-GPU, csrc/host/vpt_comm.cpp): the call's LAST resolve kernel stores every finished pixel straight into the
// full-frame buffer of every rank (its own included) at the pixel's global position, over NVLink peer mappings -- the all-gather and
// the stripe un-permutation fused into the kernel that produces the values.
constexpr int kMaxPeers = 8;
struct PeerFrames { int n = 0; float* accum[kMaxPeers] = {}; unsigned int* display[kMaxPeers] = {}; };
// Compositing AOVs (vpt_set_aov_buffers): [local pixel] running means of the coverage indicator [depth > 0] and of the sample's volume
// share, next to accum.  Either may be null.  A kernel argument of the AOV instantiations of k_resolve / k_resolve_adaptive only (not in
// FrameArgs, so every other kernel keeps its parameter block); aov == null or both pointers null selects the instantiations without them.
struct AovBuffers { float* alpha = nullptr; float3* volume = nullptr; };
// Light groups (vpt_set_light_group_buffers): [local pixel] running means of the radiance each light class added to the sample -- sun,
// point lights, emission, environment -- next to accum.  Any output may be null.  `planes`: the per-sample group sums of the generic trace
// kernels, float plane (group * 3 + channel) at planes + plane * stride, indexed by the sample slot pass * n_local + local pixel like the
// records; null when a lean kernel traced the frame (its path radiance L is the sun group).  A kernel argument of the light-group
// instantiations of k_trace / k_resolve / k_resolve_adaptive only, as AovBuffers is.
enum LightGroup : int { LG_SUN = 0, LG_POINT = 1, LG_EMISSION = 2, LG_ENVIRONMENT = 3, kLightGroups = 4 };
struct LightGroups { float3* out[kLightGroups] = {}; float* planes = nullptr; unsigned long long stride = 0; };
// Deep slices (vpt_set_deep_buffers): out[k * n_local + local pixel] = slice k's running means {premultiplied colour, coverage} of the
// samples whose depth d has z[k] <= d < z[k + 1] (z[n] may be +inf), d > 0.  n = 1..kDeepMaxSlices, z strictly increasing.  A kernel
// argument of the deep instantiations of k_resolve / k_resolve_adaptive / k_resolve_region only (the last of the pack), as AovBuffers is.
constexpr int kDeepMaxSlices = 32;                    // VPT_DEEP_MAX_SLICES of vpt_b200.h
struct DeepSlices { float4* out = nullptr; int n = 0; float z[kDeepMaxSlices + 1] = {}; };
// Instance mattes, resolve side (vpt_set_instance_mattes): out[k * n_local + local pixel] = matte k's running means {premultiplied colour,
// coverage}, defined as a deep slice's with "its id maps to matte k" for "its depth falls in slice k": a sample with d > 0 and id i lands in
// map[i] (i < n_ids) or `sphere` (i == kMatteSphereId), none where that is -1.  id: the trace's id plane (MatteIds); map: device memory.
// A kernel argument of the matte instantiations of the resolve kernels only (the last of the pack, in place of a DeepSlices).
constexpr int kMatteMax = 32;                         // VPT_MATTE_MAX of vpt_b200.h
struct Mattes { float4* out = nullptr; int n = 0; const uint32_t* id = nullptr; const int8_t* map = nullptr; uint32_t n_ids = 0; int sphere = -1; };
// Which k_resolve / k_resolve_adaptive a frame runs (instantiations: resolve_kernels in vpt_kernels.cu).  sky: 0 HDRI, 1 the precomputed
// sky, 2 the volumetric path integrator (ends on that sky; atm: the caller's AtmosphereParameters); with the AOVs; with the light groups;
// with the deep slices; with the instance mattes.
struct ResolveKey { int sky = 0; bool aov = false, groups = false, deep = false, mattes = false; };
cudaError_t launch_resolve(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, int sampled, int write_display,
                           const PeerFrames* peers, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                           const Projection& pj, cudaStream_t s, const OdsParams* od = nullptr);
// Motion vectors (vpt_set_motion_vectors): out[local pixel] = running means of (c vx, c vy, c), c = [depth > 0] of the pass sample and
// (vx, vy) = pi_B(P) - pi_A(P), P the sample's first collision on its camera ray, pi_K the film position (s W, t H) of camera K, A the frame
// camera and B the pose below (origin, lower_left_corner, horizontal, vertical: the only fields pi reads).  Kept by k_motion_vectors* in a
// launch of their own next to the frame's resolve (launch_motion_vectors), so no other kernel's parameter block changes.
struct MotionVectors { float3* out = nullptr; vpt_f3 origin, lower_left_corner, horizontal, vertical; };
// one chunk of n_passes passes (sampled 0: passes that sample nothing, every sample c = 0).  rg: the frame's render region (R's pixels only);
// ad: an adaptive frame (the active tiles, stopped pixels keep their vectors); mo: the frame's camera motion (each sample's camera is
// motion_camera's at its shutter draw).  At most one of rg and ad.
cudaError_t launch_motion_vectors(const FrameArgs& fa, const MotionVectors& mv, int n_passes, int sampled, const RenderRegion* rg,
                                  const AdaptArgs* ad, const CameraMotion* mo, cudaStream_t s);
// Collision AOVs (vpt_set_collision_aovs): position[local pixel] = running means of (c Px, c Py, c Pz, c), normal and albedo those of c n and
// c a, c = [depth > 0] of the pass sample and P = org + depth dir its first collision on its camera ray; n and a the sphere's or the volume's
// there (collision_surface in vpt_kernels.cu).  Any output may be null.  step: the central differences' world step h (normal only).
// brick_pool / brick_dims: volume 0's brick pool in brick mode (null otherwise; the cell table comes with FrameArgs).  Kept by
// k_collision_aovs* in a launch of their own next to the frame's resolve (launch_collision_aovs), so no other kernel's parameter block changes.
struct CollisionAovs { float4* position = nullptr; float3* normal = nullptr; float3* albedo = nullptr; float step = 0.f;
                       const float* brick_pool = nullptr; int brick_dims[3] = {}; };
// as launch_motion_vectors: one chunk of n_passes passes (sampled 0: every sample c = 0), rg / ad / mo as there
cudaError_t launch_collision_aovs(const FrameArgs& fa, const CollisionAovs& ca, int n_passes, int sampled, const RenderRegion* rg,
                                  const AdaptArgs* ad, const CameraMotion* mo, cudaStream_t s);
// Cryptomatte (vpt_set_cryptomatte): the uint32 state of 2 + 2 cap planes of n_local words, plane-major: n (passes counted), overflow, then
// (id_j, count_j) for j < cap.  Per pass under accum's gate (iteration < max_interactions; iteration 0 clears the pixel first): n += 1, and a
// sample with c = [depth > 0] adds its id (the trace's id plane, MatteIds) to the entry that holds it, else to the first entry with count 0,
// else to overflow.  Kept by k_cryptomatte* in a launch of their own next to the frame's resolve, so no other kernel's parameter block changes.
constexpr int kCryptoMaxEntries = 32;                 // VPT_CRYPTO_MAX_ENTRIES of vpt_b200.h
struct Cryptomatte { uint32_t* state = nullptr; int cap = 0; const uint32_t* id = nullptr; };
// as launch_motion_vectors: one chunk of n_passes passes (sampled 0: every sample c = 0), rg / ad as there (no camera ray is rebuilt)
cudaError_t launch_cryptomatte(const FrameArgs& fa, const Cryptomatte& cm, int n_passes, int sampled, const RenderRegion* rg, const AdaptArgs* ad,
                               cudaStream_t s);
// vpt_cryptomatte_rank: per pixel of n_px, the non-empty entries of the state by count descending, then id ascending (the sphere,
// kMatteSphereId, last); rank r = (id float, count / n) in float4 plane r / 2 of out, components 2 (r % 2) and 2 (r % 2) + 1; (0, 0) past the
// last entry and where n == 0.  id float: id_of_instance[id] (id < n_instances), sphere_id (the sphere), else 0.  out_overflow (may be null):
// overflow / n.
struct CryptoRank { const uint32_t* state = nullptr; int cap = 0; long long n_px = 0; const float* id_of_instance = nullptr; uint32_t n_instances = 0;
                    float sphere_id = 0.f; int n_ranks = 0; float2* out = nullptr; float* out_overflow = nullptr; };
cudaError_t launch_cryptomatte_rank(const CryptoRank& a, cudaStream_t s);
// flags: 64-bit epoch counters in peer-mapped memory.  signal: store `epoch` into slot `rank` of flag array `which` (0 ready, 1 done) of every
// peer; wait: spin until slots 0..n-1 of the LOCAL array have all reached `epoch` (gives up after ~10 s and raises the block's error word).
cudaError_t launch_peer_signal(unsigned long long* const peer_flags[kMaxPeers], int n, int rank, int which, unsigned long long epoch, cudaStream_t s);
cudaError_t launch_peer_wait(unsigned long long* local_flags, int n, int which, unsigned long long epoch, cudaStream_t s);
// loads every kernel a render call may issue (lazy module loading): no first launch may have to wait behind a peer's spinning flag wait
cudaError_t exchange_kernels_preload();
constexpr int kPeerFlagStride = 16;                   // u64 slots per flag array; layout of a block header: ready[16] done[16] error[1] layout[1] binned[1] (+13 unused) adapt[16]
constexpr int kPeerFlagsAdapt = 3;                    // flag array of the two barriers of every convergence test of a sharded adaptive frame
// Exchange layers (vpt_comm_p2p_export_layers): full-frame planes [H][W] of depth and the compositing layers in every rank's block, in the
// order of the VPT_LAYER_* bits (bit l = 1 << l).  Depth and alpha are float, the others float3.
enum ExchangeLayer : int { XL_DEPTH = 0, XL_ALPHA = 1, XL_VOLUME = 2, XL_SUN = 3, XL_POINT = 4, XL_EMISSION = 5, XL_ENVIRONMENT = 6, kExchangeLayers = 7 };
// src: this rank's [local pixel] buffer of each layer, null where the layer is not active on the context.  plane: every rank's full-frame
// plane of each layer as mapped here, null where the block was exported without it.  A kernel argument of k_layers_publish only.
struct LayerSources { const float* src[kExchangeLayers] = {}; };
struct LayerPlanes { int n = 0; float* plane[kExchangeLayers][kMaxPeers] = {}; };
// after the call's last resolve (or k_adapt_publish): every active, exported layer of every local pixel at its global position in every rank's
// planes; rg: the frame's render region (null: the whole frame).  Padding rows and pixels outside R are not written.
cudaError_t launch_layers_publish(const FrameGeom& g, const RenderRegion* rg, const LayerSources& src, const LayerPlanes& dst, cudaStream_t s);
// Binned exchange layers (vpt_comm_p2p_export_binned): the deep slices and the instance mattes, one [K][H][W] float4 array each in every
// rank's block after the layer planes.  plane[p]: rank p's array of one binned layer as mapped here.  A kernel argument of k_binned_publish only.
struct BinnedPlanes { int n = 0; float4* plane[kMaxPeers] = {}; };
// right after launch_layers_publish: src[k * n_local + local pixel] (a deep-slice or matte buffer, k < n_bins) of every local pixel at
// plane[p][k * W * H + global pixel] in every rank's array; rg as for launch_layers_publish.  Padding rows and pixels outside R are not written.
cudaError_t launch_binned_publish(const FrameGeom& g, const RenderRegion* rg, const float4* src, int n_bins, const BinnedPlanes& dst, cudaStream_t s);
// limit = min(W*H, 65536) entries are advanced (the reference updates entry y*W + x from pixel (x, y))
cudaError_t launch_bn_prepare(void* bn, float2* table, int np, int limit, unsigned* queue_counters, cudaStream_t s);   // also zeroes queue_counters[0..1]
cudaError_t launch_bn_advance(void* bn, int n, int limit, cudaStream_t s);
cudaError_t launch_unpermute(const void* gathered, void* full, const FrameGeom& g, int elem_bytes, cudaStream_t s);
// vpt_debug_camera_rays: out[local pixel] = (b0, 0), the ray direction before normalize of the next render call's first pass: pano_b0 or
// camera_b0 at the jitter the blue-noise buffer `bn` holds now (read only)
cudaError_t launch_camera_rays(const vpt_camera& cam, const vpt_u2 res, const FrameGeom& g, const Projection& pj, const void* bn, float4* out,
                               cudaStream_t s);
// vpt_debug_motion_cameras: out[local pixel * 20 ..] = xi, then origin, lower_left_corner, horizontal, vertical, u, v of motion_camera at the
// shutter draw of the pixel's first pass at `iteration` (19 floats, padded with 0; padding rows all 0)
cudaError_t launch_motion_cameras(const vpt_camera& cam, const CameraMotion& mo, const FrameGeom& g, uint32_t iteration, float* out, cudaStream_t s);
// vpt_debug_ods_cameras (rays == 0): out[local pixel * 8 ..] = origin', lower_left_corner', e, k of ods_camera for the next render call's
// first pass; vpt_debug_camera_rays on an ODS frame (rays == 1): out[local pixel * 4 ..] = (camera_b0 of that camera, 0).  Both at the jitter
// the blue-noise buffer `bn` holds now (read only); padding rows all 0
cudaError_t launch_ods_cameras(const vpt_camera& cam, const OdsParams& od, const vpt_u2 res, const FrameGeom& g, const void* bn, int rays, float* out,
                               cudaStream_t s);
// adaptive frame: k_generate / k_resolve over the tiles of ad.tiles only (stopped pixels sample nothing and keep their buffers); the resolve
// also updates the Welford state and writes pass_count, rel_error, display and raw of the pixels it visits
cudaError_t launch_generate_adaptive(const FrameArgs& fa, int n_passes, const AdaptArgs& ad, const Projection& pj, const CameraMotion* mo,
                                     const OdsParams* od, cudaStream_t s);
cudaError_t launch_resolve_adaptive(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, const AdaptArgs& ad,
                                    const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt, const Projection& pj,
                                    cudaStream_t s, const OdsParams* od = nullptr);
// convergence test over ad.tiles: stops every active pixel whose 3x3 neighbourhood (global rows) has err < threshold, lists the tiles still
// active.  halo: the local exchange block's full-frame err plane, read for neighbour rows of other ranks (null for one rank)
cudaError_t launch_adapt(const FrameGeom& g, const AdaptArgs& ad, const float* halo, cudaStream_t s);
// start of an adaptive frame: no pixel stopped, tile list = every tile
cudaError_t launch_adapt_init(const FrameGeom& g, uint8_t* stopped, unsigned* tiles, int n_tiles, cudaStream_t s);
// Region frames (RenderRegion above): the same kernels over R only.  k_generate_region samples the pixels of R in R's tiles;
// k_miss_cull_region tests the strips that hold a pixel of R; k_resolve_region resolves R's pixels (the peer stores as launch_resolve).
// Adaptive, one rank: the tile list starts as R's tiles with every pixel outside R stopped, and k_adapt_region clips the 3x3 neighbourhood
// at R's edge.
cudaError_t launch_generate_region(const FrameArgs& fa, int n_passes, const RenderRegion& rg, const Projection& pj, const CameraMotion* mo,
                                   const OdsParams* od, cudaStream_t s);
cudaError_t launch_miss_cull_region(const FrameArgs& fa, uint8_t* mask, const RenderRegion& rg, const Projection& pj, cudaStream_t s,
                                    const OdsParams* od = nullptr);
cudaError_t launch_resolve_region(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, int sampled, int write_display,
                                  const PeerFrames* peers, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                                  const RenderRegion& rg, const Projection& pj, cudaStream_t s, const OdsParams* od = nullptr);
cudaError_t launch_adapt_init_region(const FrameGeom& g, uint8_t* stopped, unsigned* tiles, const RenderRegion& rg, cudaStream_t s);
cudaError_t launch_adapt_region(const FrameGeom& g, const AdaptArgs& ad, const RenderRegion& rg, cudaStream_t s);
// vpt_debug_adapt_rule: passes [p0, p0 + n_passes) of `samples` ([pass][local pixel]) through the adaptive Welford state of the active
// pixels of ad.tiles, ending with k_resolve_adaptive's stat / pass_count / rel_error stores
cudaError_t launch_debug_adapt_pass(const FrameGeom& g, const AdaptArgs& ad, const float3* samples, int p0, int n_passes, cudaStream_t s);

// Sharded adaptive frame over the peer-memory exchange: every rank's block as mapped here, full-frame planes [H][W] at global pixels.
struct AdaptPeers {
    int n = 0;
    float* accum[kMaxPeers] = {}; unsigned int* display[kMaxPeers] = {};   // display null when the block was exported without it
    unsigned* count[kMaxPeers] = {}; float* err[kMaxPeers] = {};           // pass counts, relative errors (err doubles as the 3x3 halo)
    unsigned* tiles[kMaxPeers] = {};                                       // [rank] active-tile count of every rank after a test
};
// at a test chunk: the err of every active pixel whose global row borders another rank's stripe, into every rank's err plane
cudaError_t launch_adapt_halo(const FrameGeom& g, const AdaptArgs& ad, const AdaptPeers& pp, cudaStream_t s);
// after k_adapt: this rank's active-tile count (*next_count) into slot `rank` of every rank's count array; out[2] = the local error word
cudaError_t launch_adapt_count_publish(const AdaptPeers& pp, int rank, const unsigned* next_count, const unsigned long long* err_word,
                                       unsigned* out, cudaStream_t s);
// out[1] = sum of the n local count slots (n > 0), out[at] = the local error word (abandoned flag waits so far)
cudaError_t launch_adapt_tally(const unsigned* slots, int n, const unsigned long long* err_word, unsigned* out, int at, cudaStream_t s);
// end of the frame: accum, display, pass count and err of every local pixel into every rank's planes; padding rows get count 0 / err 0
cudaError_t launch_adapt_publish(const FrameGeom& g, const vpt_kernel_params& kp, const AdaptArgs& ad, const AdaptPeers& pp, cudaStream_t s);

// Denoiser (vpt_denoise, csrc/device/vpt_denoise.cu): k_denoise_prep fills plane pair 0, then one k_denoise_atrous per level ping-pongs
// the pairs; the last level reads the planes only and writes out_f3 / out_display, so out_f3 may be the colour input itself.
// vpt_denoise_layers adds layers: k_denoise_layer_gather copies each into its float4 planes of lp[0] (in order, count planes each) before
// the first level, and after each k_denoise_atrous the planes take the same level, the last one scattering into each layer's dst.
struct DenoiseLayer {
    const float* src;                    // [count][H][W][channels]
    float*       dst;                    // same shape, may equal src
    unsigned     channels, count;        // 1..4, >= 1
};
struct DenoiseArgs {
    int          width, height, iterations;
    float        sigma_l, sigma_z, exposure_scale;
    const float* color;                  // [H][W] float3
    const float* depth;                  // [H][W], null: no depth term
    const float* rel_error;              // [H][W], null: spatial variance estimate
    float*       out_f3;                 // [H][W] float3
    unsigned*    out_display;            // [H][W], may be null
    float4*      cv[2];                  // scratch planes {r, g, b, v}, width * height each
    float2*      yz[2];                  // scratch planes {Y, z}
    const DenoiseLayer* layers = nullptr; // host array of n_layers
    int          n_layers = 0;
    float4*      lp[2] = {};             // layer scratch planes, sum of the counts * width * height each
};
// launches of the layer planes per level: groups of 8, 4, 2 or 1 planes
inline int denoise_layer_groups(size_t n_planes) { return (int)(n_planes / 8) + __builtin_popcountll(n_planes % 8); }
cudaError_t launch_denoise(const DenoiseArgs& a, cudaStream_t s);

// Temporal filter (vpt_temporal, csrc/device/vpt_temporal.cu): k_temporal, one thread per pixel of full [H][W] frames.  history and
// history_len are both null (no history) or both set; out_display may be null; no output overlaps an input or another output.
// vpt_temporal_layers adds up to kTemporalMaxLayers layers, carried in the parameter block and blended with the beauty's taps and L_new;
// a layer's history is null exactly when `history` is.
constexpr int kTemporalMaxLayers = 16;                // VPT_TEMPORAL_MAX_LAYERS of vpt_b200.h
struct TemporalLayer {
    const float* src;                    // [count][H][W][channels]
    const float* history;                // same shape
    float*       dst;                    // same shape
    unsigned     channels, count;        // 1..4, >= 1
};
struct TemporalArgs {
    int          width, height;
    unsigned     max_history;
    float        clip_sigma, exposure_scale;       // clip_sigma +inf: no clip
    vpt_f3       a_origin, a_llc, a_horizontal, a_vertical;   // A, the frame camera
    vpt_f3       b_origin, b_llc, b_horizontal, b_vertical;   // B, the camera of the history
    const float* color;                  // [H][W] float3
    const float* vectors;                // [H][W] float3, vpt_set_motion_vectors' (c vx, c vy, c) towards B
    const float* history;                // [H][W] float3
    const float* history_len;            // [H][W]
    float*       out;                    // [H][W] float3
    float*       out_len;                // [H][W]
    unsigned*    out_display;            // [H][W]
    int          n_layers = 0;
    TemporalLayer layers[kTemporalMaxLayers] = {};
};
cudaError_t launch_temporal(const TemporalArgs& a, cudaStream_t s);

} // namespace vpt
