// vpt_host.h -- declarations shared by the host translation units of libvpt_b200.so (not part of the public ABI).
#pragma once
#include "../../../include/vpt_b200.h"
#include "../device/vpt_kernels.h"

#include <cuda_runtime.h>
#include <string>

#include <vector>

struct vpt_context {
    int device = 0;
    int num_sms = 0;
    std::string err;
    // options
    int passes_per_chunk = 32;
    int ctas_per_sm = 0;
    // partition
    int rank = 0, n_ranks = 1, stripe_rows = 16;
    // scene cache: keyed by the two device pointers AND the registry generation of the octree (a rebuilt octree that got the
    // same address back is a different scene); the cheap per-volume records are refreshed whenever a new frame starts
    vpt_devptr_t cached_volumes = 0, cached_root = 0;
    unsigned long long cached_generation = 0;
    bool   scene_single_volume = false;
    size_t cap_vrec = 0;              // VolumeRec capacity (grows with the instance count)
    int*   h_pinned = nullptr;        // eight pinned words: the read-back a foreign octree needs, the tile counts of an adaptive test
    int    max_ctas[vpt::kTraceKernelsAll] = {};   // trace kernel occupancy (CTAs per SM), by vpt::TraceKernel
    size_t l2_fetch_default = 0; int l2_sector_fetch = 0;     // option "l2_sector_fetch" (cell mode)
    const float4* cell_table = nullptr; int cell_dims[3] = {0, 0, 0};   // vpt_set_cell_volume
    int    trace_slots = 0;              // option "trace_slots": rays per lane of k_trace, 0 = by scene (2 for lean frames, grids larger than twice the L2, >= 64 instances)
    size_t l2_bytes = 0;
    const float* brick_pool = nullptr; int brick_dims[3] = {0, 0, 0};   // fast mode: density of volume 0 as a brick pool (vpt_set_brick_volume)
    int    force_generic = 0;        // option "generic_kernel": 1 = never use the lean trace instantiation (A/B and tests)
    vpt::SceneTables* d_scene = nullptr;
    vpt::OctInternal* d_internal = nullptr;
    uint2* d_leaf_list = nullptr;
    int* d_leaf_indices = nullptr;
    vpt::VolumeRec* d_vrec = nullptr;
    // frame buffers
    size_t cap_samples = 0;           // n_local * chunk
    bool   cap_wide = false;          // planes B, C allocated (wide sample records) rather than the tr plane
    bool   cap_planeD = false;
    size_t cap_tr = 0;                // pixels of d_plane_tr
    float* d_plane_tr = nullptr;
    uint2* d_queue_id = nullptr; float4* d_queue_org = nullptr; float2* d_bn_table = nullptr; int cap_chunk = 0;
    int sched_min_lanes = 0;          // option "sched_min_lanes": 0 = by kernel (26 for the lean kernel at 3 rays per lane, else 20)
    int debug_flags = 0;
    float4 *d_queue = nullptr, *d_planeA = nullptr, *d_planeB = nullptr, *d_planeC = nullptr, *d_planeD = nullptr;
    unsigned* d_counters = nullptr;   // [0] queue_count, [1] queue_head
    int      miss_cull = 1;           // option "miss_cull": k_miss_cull marks the pixels no jitter can take to the volume or the sphere
    uint8_t* d_miss_mask = nullptr;   // [local pixel] its mask, rebuilt by every render call of a pinhole frame
    size_t   cap_miss_mask = 0;
    // stats
    unsigned long long launches = 0;
    int count_stats = 0;              // option "count_stats": accumulate trace counters
    int empty_ahead = 1;              // option "empty_ahead": walks end at the first empty node with no populated leaf ahead (same result)
    unsigned long long* d_stats = nullptr;   // 16 counters (vpt_kernels.h FrameArgs::counters)
    int    last_trace_rays = 0;              // rays per lane of the last render call's trace kernel (vpt_get_counters out[7])
    int profile = 0;                  // option "profile": CUDA-event timing of every kernel (debug / bench breakdown)
    struct Ev { int kind; cudaEvent_t a, b; };
    std::vector<Ev> events;
    // multi-GPU (vpt_comm.cpp): NCCL communicator + gather targets; null for a single rank
    void*  nccl_comm = nullptr;
    void*  d_gathered = nullptr; size_t cap_gathered = 0;      // [rank][local pixel] staging of the all-gather
    void*  d_full_accum = nullptr;                              // caller-owned full frame float3 [H][W] (gather target), may be null
    void*  d_full_display = nullptr;                            // caller-owned full frame u32 [H][W], may be null
    void*  d_gathered_disp = nullptr; size_t cap_gathered_disp = 0;
    cudaStream_t comm_stream = nullptr; cudaEvent_t ev_render_done = nullptr, ev_gather_done = nullptr;
    // peer-memory exchange (vpt_comm_p2p_*): one cudaMalloc'd block per rank {flags, full accum, full display}, IPC-mapped into every rank
    void*  p2p_block = nullptr; size_t p2p_bytes = 0; int p2p_w = 0, p2p_h = 0;
    void*  p2p_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // [rank] -> that rank's block as mapped here (own: p2p_block)
    int    p2p_n = 0; bool p2p_on = false, p2p_display = false, p2p_local = false; unsigned long long p2p_epoch = 0;
    unsigned long long p2p_adapt_epoch = 0;                     // barriers of the convergence tests of sharded adaptive frames (flag array kPeerFlagsAdapt)
    unsigned p2p_layers = 0;                                    // VPT_LAYER_* mask the block was exported with (vpt_comm_p2p_export_layers)
    unsigned p2p_slices = 0, p2p_mattes = 0;                    // deep slices / mattes the block carries, 0: none (vpt_comm_p2p_export_binned)
    int    gather_async = 0;                                    // option "gather_async": gather on the side stream (see vpt_comm_wait)
    bool   gather_pending = false;
    size_t max_scratch_bytes = (size_t)12 << 30;                // cap of the per-chunk ray queue + sample planes
    int    chunk_auto = 1;                                      // passes_per_chunk not set by the caller: pick by local frame size
    // adaptive frames (vpt_render_adaptive), allocated on first use
    float4*   d_adapt_stat = nullptr;                           // [pixel] Welford state n, mean, M2, err of the sample luminance
    uint8_t*  d_adapt_stopped = nullptr;                        // [pixel] 1 once stopped
    unsigned* d_adapt_tiles = nullptr;                          // two active-tile lists + the count of the next one
    size_t    cap_adapt_px = 0, cap_adapt_tiles = 0;
    vpt_devptr_t adaptive_accum = 0;                            // accum_buffer of the last adaptive frame: vpt_render_passes may not continue it
    // denoiser (vpt_denoise), allocated on first use: two ping-pong plane pairs {r, g, b, v} and {Y, z}
    float4*   d_dn_cv = nullptr;                                // 2 * cap_dn_px
    float2*   d_dn_yz = nullptr;                                // 2 * cap_dn_px
    size_t    cap_dn_px = 0;
    // vpt_denoise_layers, allocated on first use and only grown: two sets of float4 layer planes of cap_dn_layer (planes * pixels) each
    float4*   d_dn_layer = nullptr;
    size_t    cap_dn_layer = 0;
    // compositing AOVs (vpt_set_aov_buffers): caller-owned [local pixel] float / float3 buffers, either may be null; registered buffers
    // become active at the next render call with iteration == 0, so no running mean ever continues from what they held before
    float*    aov_alpha = nullptr;
    float*    aov_volume = nullptr;
    bool      aov_active = false;
    // light groups (vpt_set_light_group_buffers): caller-owned [local pixel] float3 buffers of the sun, point, emission and environment
    // groups, any may be null; activated like the AOVs.  d_lg_planes: the generic trace kernels' per-sample group sums (12 float planes of
    // cap_lg_samples each), allocated with the other frame buffers
    float*    lg_out[4] = {nullptr, nullptr, nullptr, nullptr};
    bool      lg_active = false;
    float*    d_lg_planes = nullptr;
    size_t    cap_lg_samples = 0;
    // deep slices (vpt_set_deep_buffers): a caller-owned [slice][local pixel] float4 buffer with its slice count and bounds, checked when set
    // (deep_req.out null: off) and activated like the AOVs
    vpt::DeepSlices deep_req;
    bool      deep_active = false;
    // instance mattes (vpt_set_instance_mattes): a caller-owned [matte][local pixel] float4 buffer, its matte count and the host copy of the
    // instance -> matte map, checked when set (matte_req.out null: off) and activated like the AOVs; the map goes to d_matte_map then.
    // d_matte_ids: the trace kernels' id plane (one uint32 per sample), allocated with the other frame buffers
    vpt::Mattes matte_req;
    std::vector<int8_t> matte_map_req;
    bool      matte_active = false;
    int8_t*   d_matte_map = nullptr;
    size_t    cap_matte_map = 0;
    uint32_t* d_matte_ids = nullptr;
    size_t    cap_matte_samples = 0;
    int       scene_instances = 0;    // instances of the cached scene
    // render region (vpt_set_render_region): global pixels [x0, x1) x [y0, y1), all 0 = the whole frame.  region_req is what the caller
    // set last; it becomes region_cur at the next render call with iteration == 0, so a running mean never continues under another region
    unsigned  region_req[4] = {0, 0, 0, 0};
    unsigned  region_cur[4] = {0, 0, 0, 0};
    // camera projection (vpt_set_projection), checked when set: proj_req is what the caller set last; it becomes proj_cur at the next render
    // call with iteration == 0, so a running mean never continues under another projection
    vpt::Projection proj_req, proj_cur;
    // the rest of an ODS projection (vpt_set_projection_ods), read where proj_req / proj_cur is of kind kProjOds, and taken over with it
    vpt::OdsParams ods_req, ods_cur;
    // camera motion (vpt_set_camera_motion), checked when set: the shutter-close pose the caller set last (motion_req false: none); it becomes
    // motion_cur at the next render call with iteration == 0, so a running mean never continues under another pose
    bool      motion_req = false, motion_cur = false;
    vpt::CameraMotion motion_close_req, motion_close_cur;
    // motion vectors (vpt_set_motion_vectors): a caller-owned [local pixel] float3 buffer and the target pose, checked when set (mv_req.out
    // null: off) and activated like the AOVs, so a frame in progress keeps the target it started with (setting clears mv_active)
    vpt::MotionVectors mv_req;
    bool      mv_active = false;
    // collision AOVs (vpt_set_collision_aovs): caller-owned [local pixel] position / normal / albedo buffers and the gradient step, checked when
    // set (all three null: off) and activated like the AOVs
    vpt::CollisionAovs ca_req;
    bool      ca_active = false;
    // Cryptomatte (vpt_set_cryptomatte): the caller-owned uint32 state and its capacity, checked when set (crypto_req.state null: off) and
    // activated like the mattes; the trace kernel writes its ids into d_matte_ids, shared with the mattes
    vpt::Cryptomatte crypto_req;
    bool      crypto_active = false;
    // sample-stream offset (vpt_set_sample_offset): the one set last becomes sample_offset_cur at the next render call with iteration == 0,
    // so the passes of one frame draw consecutive streams
    uint32_t  sample_offset_req = 0, sample_offset_cur = 0;
};


namespace vpt {

// ---- device-side builders (vpt_octree.cu) ---------------------------------------------------------------
cudaError_t octree_build_device(vpt_octnode* d_nodes, const vpt_gpu_vdb* d_vols, int n, cudaStream_t s);
void        instance_bounds_host(const vpt_gpu_vdb& g, float out6[6]);
cudaError_t octree_snapshot(const vpt_octnode* d_root, vpt_octnode* h_nodes, int* h_exists);
cudaError_t octree_flat_counts(const vpt_gpu_vdb* d_vols, int n, const float root6[6], void** d_bounds_out, int h_counts[585], cudaStream_t s);
cudaError_t octree_flat_fill(const void* d_bounds, int n, const float root6[6], const unsigned* d_offsets, int* d_indices, cudaStream_t s);
cudaError_t bvh_build_device(const vpt_gpu_vdb* d_vols, int n, vpt_bvhnode* d_nodes, vpt_bvhnode* d_leaves, float scene6[6],
                             unsigned long long* h_codes, int* h_ids, cudaStream_t s);

// ---- scene registry (vpt_scene_build.cpp) ------------------------------------------------------------------
// Every octree built by vpt_octree_build is registered under its root device pointer together with the flat
// tables the render kernels read.  vpt_render_passes looks the root pointer of params[VPT_ARG_OCTREE] up here;
// a pointer that is not registered is a foreign (reference-built, pointer-linked) octree and is flattened by
// k_prepare_scene instead.
struct SceneEntry {
    int          device = 0;
    int          n = 0;                      // instances
    unsigned long long generation = 0;       // unique per build: detects a rebuilt octree that got the same address back
    float        root6[6] = {0, 0, 0, 0, 0, 0};
    float        max_extinction = 0.f, min_extinction = 0.f;
    OctInternal* d_internal = nullptr;       // [73]
    uint2*       d_leaf_list = nullptr;      // [512] (offset, count)
    int*         d_leaf_indices = nullptr;   // CSR payload (at least 1 element)
    size_t       total_indices = 0;
    int          max_leaf_count = 0;
    unsigned     any_flags = 0;              // bit0: some instance has a colour grid, bit1: some instance has an emission grid
    unsigned long long max_grid_bytes = 0;   // density grid of the largest instance (float voxels): picks the trace kernel's rays per lane
    int          dim0[3] = {0, 0, 0};        // voxels per axis of volume 0's density grid: what a brick pool or cell table must cover
};
bool scene_registry_find(vpt_devptr_t d_root, SceneEntry* out);

int  fail_global(int code, const std::string& msg);     // records the text for vpt_last_error(NULL)
int  fail_ctx(vpt_context* ctx, int code, const std::string& msg);
FrameGeom make_frame_geom(const vpt_context* c, unsigned w, unsigned h);
// after the last resolve of a vpt_render_passes call: all-gather + un-permute into the caller's full-frame buffers (vpt_comm.cpp)
int  comm_p2p_begin(vpt_context* c, cudaStream_t stream);                                        // call start: tell the peers this rank's frame may be overwritten
int  comm_p2p_peers(vpt_context* c, cudaStream_t stream, PeerFrames* out);                       // before the call's last resolve: wait for the peers, hand out their frames
int  comm_p2p_end(vpt_context* c, cudaStream_t stream);                                          // after it: publish, and wait until every peer has published
// right before comm_p2p_end: the exported layers that src holds into every rank's planes (k_layers_publish); nothing when the exchange is
// suspended, on one rank or without layers.  rg: the frame's render region, null for the whole frame
int  comm_p2p_layers(vpt_context* c, const FrameGeom& g, const RenderRegion* rg, const LayerSources& src, cudaStream_t stream,
                     const float3* motion = nullptr);   // motion: the frame's active motion-vector buffer (VPT_LAYER_MOTION), null: none
// right after comm_p2p_layers: the frame's active deep slices and mattes (null: not active) into every rank's binned arrays
// (k_binned_publish); nothing when the exchange is suspended, on one rank, or for a layer the block does not carry.  The caller has checked
// that an active layer's count is the exported one (frame_setup)
int  comm_p2p_binned(vpt_context* c, const FrameGeom& g, const RenderRegion* rg, const float4* deep, const float4* mattes, cudaStream_t stream);
// sharded adaptive frames: every rank's planes as mapped here, and the local block's halo (err plane), count slots and error word
struct P2pAdaptLocal { const float* halo = nullptr; const unsigned* tiles = nullptr; const unsigned long long* error_word = nullptr; };
void comm_p2p_adapt_views(vpt_context* c, AdaptPeers* out, P2pAdaptLocal* local);
int  comm_p2p_adapt_barrier(vpt_context* c, cudaStream_t stream);                                // signal + wait on the adapt flags (own epoch)
int  comm_gather_frame(vpt_context* c, const FrameGeom& g, const void* d_local_accum, const void* d_local_display, cudaStream_t stream);
int  comm_before_accum_write(vpt_context* c, cudaStream_t stream);   // async mode: the previous gather must have read accum

} // namespace vpt
