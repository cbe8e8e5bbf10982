/*
 * vpt_b200.h -- C ABI of libvpt_b200.so, the H100-native (sm_90a) replacement for the reference render pass.
 *
 * Drop-in boundary.  The reference application issues one progressive pass as
 *
 *     void* params[] = { &cam, &l_list, &d_volume_ptr, &d_geo_ptr, &d_geo_list_ptr,
 *                        &bvh_builder.bvh.BVHNodes, &bvh_builder.root, atmos_params, &kernel_params };
 *     cuLaunchKernel(cuRaycastKernel, grid.x, grid.y, 1, 16, 16, 1, 0, NULL, params, NULL);   // main.cpp:1826-1827
 *
 * and the replacement is that one line:
 *
 *     vpt_render_pass(ctx, params, NULL);
 *
 * with the very same `params` array (layouts in vpt_abi.h).  All memory named by the parameters stays
 * owned by the caller, exactly as with the reference kernel; the context only owns its ray queue,
 * sample planes and the flattened scene tables it derives from GPU_VDB[] + the OCTNode tree.
 *
 * Every function returns 0 on success or a negative VPT_ERR_* code; vpt_last_error() gives the text.
 * There is no CPU fallback: without a CUDA device every entry point fails with VPT_ERR_CUDA.
 */
#ifndef VPT_B200_H_
#define VPT_B200_H_

#include "vpt_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VPT_OK                 0
#define VPT_ERR_INVALID       -1   /* bad argument */
#define VPT_ERR_CUDA          -2   /* CUDA runtime / driver failure (text in vpt_last_error) */
#define VPT_ERR_UNSUPPORTED   -3   /* parameter combination this build does not implement */
#define VPT_ERR_IO            -4   /* file could not be read / decoded */

typedef struct vpt_context vpt_context;

/* ---- lifecycle ----------------------------------------------------------------------------------- */
int  vpt_create(vpt_context** out);                    /* binds to the calling thread's current CUDA device */
void vpt_destroy(vpt_context* ctx);
const char* vpt_last_error(const vpt_context* ctx);    /* ctx may be NULL: error of the last failed vpt_create / helper */
const char* vpt_version(void);
/* sizeof() of the boundary structs: camera, light_list, GPU_VDB, sphere, geometry_list, BVHNode, OCTNode,
 * AtmosphereParameters, Kernel_params, point_light, VDB_INFO, AABB.  Returns how many entries exist. No CUDA call. */
int  vpt_abi_sizes(size_t* out, int n);

/* Tunables: "passes_per_chunk" (1..64 passes fused per generate/trace/resolve round; 0 = automatic, the default: 32, or 64 when the
 * local frame has at most 2^20 pixels), "max_scratch_mb" (cap of the per-round ray queue + sample planes, default 12288),
 * "gather_async" (see vpt_comm_*),
 * "sched_min_lanes" (1..32, lanes an operation must gather in a warp before it pre-empts stepping; 0 = by kernel, the default: 26 for the
 * lean kernel at 3 rays per lane, else 20),
 * "trace_slots" (rays per lane of the trace kernel: 0 = by scene, the default -- 2 for a frame with one volume, no emission and no point
 * lights under the direct integrator, or when the density grid is larger than twice the L2 or the scene has 64 or more instances, else 3;
 * 2 or 3 to force it),
 * "l2_sector_fetch" (0|1: while a cell table is set, ask the L2 for 32-byte DRAM fetches -- a device-wide hint, see vpt_set_cell_volume),
 * "ctas_per_sm" (trace CTAs per SM, each of the trace kernel's own size: 256 threads for the lean kernel at 2 rays per lane, whose
 * maximum is 3, and 128 for the others; 0 = occupancy maximum), "generic_kernel" (1: never pick the lean instantiation), "debug_flags" (development),
 * "miss_cull" (1, the default: a pinhole HDRI frame first marks the pixels whose every jitter misses the volume's root box and the sphere,
 * and writes and reads no sample records for them -- the miss samples are rebuilt from the camera and the jitter, the frame is bit for
 * bit the same; 0: off),
 * "empty_ahead" (1, the default: a walk that reaches an empty octree node from which no populated leaf lies in its direction of travel
 * ends there instead of hopping to the root box's exit -- bit for bit the same frame; 0: off, every walk hops),
 * "count_stats" / "profile" (0|1, see vpt_get_counters / vpt_get_kernel_times). */
int  vpt_set_option(vpt_context* ctx, const char* key, int value);

/* Multi-GPU partition of the frame: rank r of n renders the interleaved row stripes r, r+n, ... of
 * `stripe_rows` rows.  With n_ranks > 1 every buffer inside Kernel_params (accum, depth, cost, raw,
 * display) holds vpt_local_pixels() pixels in rank-local order; the blue-noise buffer stays a full
 * 256x256 replica.  Default: one rank, identity layout (bit-compatible with the reference buffers). */
int  vpt_set_partition(vpt_context* ctx, int rank, int n_ranks, int stripe_rows);
long long vpt_local_pixels(const vpt_context* ctx, unsigned width, unsigned height);
/* After an all-gather of rank-local buffers ([rank][local pixel], elem_bytes per pixel, multiple of 4)
 * scatter them back into a full row-major frame. */
int  vpt_unpermute(vpt_context* ctx, const void* d_gathered, void* d_full, unsigned width, unsigned height,
                   int elem_bytes, void* stream);

/* Multi-GPU exchange, issued by the library itself (one process per GPU, NCCL; SURVEY 8(e)).  One rank obtains an id
 * (ncclGetUniqueId) and hands the 128 bytes to every rank by whatever means the application has (MPI, torch.distributed,
 * a file); every rank then calls vpt_comm_init (collective: ncclCommInitRank; also applies vpt_set_partition).  With a
 * gather target set, every vpt_render_pass(es) call ends with ONE ncclAllGather of the rank-local accumulators (and one of
 * the display words if asked) + the stripe un-permutation into the caller's full-frame buffers -- row-major [H][W] float3 /
 * uint32, allocated by the caller on every rank -- enqueued on the caller's stream behind the last kernel.  Option
 * "gather_async" = 1 moves that exchange to a side stream so the next call's sampling kernels overlap it; the library waits
 * for it before the next call overwrites the accumulator, and vpt_comm_wait(ctx, stream) makes `stream` wait for it.
 * NCCL is bound at run time (dlopen): without it these entry points fail with VPT_ERR_UNSUPPORTED, everything else works. */
#define VPT_COMM_ID_BYTES 128
int  vpt_comm_get_unique_id(unsigned char id_out[VPT_COMM_ID_BYTES]);
int  vpt_comm_init(vpt_context* ctx, const unsigned char id[VPT_COMM_ID_BYTES], int rank, int n_ranks, int stripe_rows);
int  vpt_comm_set_gather(vpt_context* ctx, void* d_full_accum_f3, void* d_full_display_u32);   /* either may be NULL */
int  vpt_comm_wait(vpt_context* ctx, void* stream);
int  vpt_comm_info(vpt_context* ctx, int* nccl_version, int* rank, int* n_ranks);
int  vpt_comm_destroy(vpt_context* ctx);

/* Peer-memory exchange: the same result without NCCL and without a separate gather step, for up to 8 GPUs of one NVLink / NVSwitch
 * domain (one process per GPU).  Every rank allocates ONE exchange block {flags, full-frame float3 accumulators, optional display words}
 * and exports it as a CUDA IPC handle (vpt_comm_p2p_export: also applies vpt_set_partition); the application hands all handles to all
 * ranks (64 bytes each, rank order) and every rank maps its peers (vpt_comm_p2p_import).  From then on the LAST resolve kernel of every
 * vpt_render_pass(es) call stores each finished pixel straight into every rank's frame at its global position (all-gather and stripe
 * un-permutation fused into the producing kernel, over peer mappings), bracketed by two flag exchanges in peer memory: "my previous frame
 * has been consumed" at the start of the call, "my stripes are in place" at the end; the call's stream work ends with a wait for all
 * peers, so after it the frame returned by vpt_comm_p2p_frame is complete on every rank, bit-identical to a single-GPU frame.
 * vpt_comm_p2p_enable(ctx, 0) suspends the exchange for rank-local work (calls that not every rank makes); vpt_comm_p2p_status reports
 * how many flag waits gave up (a wait abandons after 10 s instead of hanging the GPU: a rank died or made fewer calls). */
#define VPT_P2P_HANDLE_BYTES 64
int  vpt_comm_p2p_export(vpt_context* ctx, int rank, int n_ranks, int stripe_rows, unsigned width, unsigned height, int with_display,
                         unsigned char handle_out[VPT_P2P_HANDLE_BYTES]);
int  vpt_comm_p2p_import(vpt_context* ctx, const unsigned char* handles /* n_ranks x VPT_P2P_HANDLE_BYTES, rank order */);
/* Same-process peers (one process driving several contexts -- several GPUs with peer access enabled, or several shards on one GPU on
 * separate streams): exchange the block addresses (vpt_comm_p2p_block) instead of IPC handles. */
int  vpt_comm_p2p_block(vpt_context* ctx, vpt_devptr_t* d_block);
int  vpt_comm_p2p_import_local(vpt_context* ctx, const vpt_devptr_t* blocks /* n_ranks addresses, rank order */);
int  vpt_comm_p2p_frame(vpt_context* ctx, vpt_devptr_t* d_full_accum_f3, vpt_devptr_t* d_full_display_u32);
/* Full-frame planes [H][W] of the block that a sharded vpt_render_adaptive fills on every rank: unsigned pass counts and float relative
 * errors, at global pixels.  A fixed-count call leaves them untouched.  Either output pointer may be NULL. */
int  vpt_comm_p2p_adaptive_frame(vpt_context* ctx, vpt_devptr_t* d_full_pass_count_u32, vpt_devptr_t* d_full_rel_error_f32);
int  vpt_comm_p2p_enable(vpt_context* ctx, int on);
int  vpt_comm_p2p_status(vpt_context* ctx, unsigned long long* abandoned_waits);

/* Exchange layers: depth, the compositing AOVs and the light groups full-frame on every rank, next to the accumulators.
 *   Export.  vpt_comm_p2p_export_layers is vpt_comm_p2p_export with `layers`, a mask of the VPT_LAYER_* bits below; each bit adds one
 *     full-frame [H][W] plane to the block (float for depth and alpha, float3 for the others: 68 B per pixel for all seven), each on a
 *     256-byte boundary after the parts vpt_comm_p2p_export allocates.  vpt_comm_p2p_export is this call with layers = 0: same block, same
 *     behaviour.  Unknown bits are refused (VPT_ERR_INVALID).  vpt_comm_p2p_block_bytes gives the size of the block for a frame (pure host
 *     code).  Every rank exports the same frame size, display flag and layers: the block header records them, and vpt_comm_p2p_import /
 *     _import_local refuse a peer whose block differs (VPT_ERR_INVALID, naming the rank) and map nothing.
 *   Calls.  Once the exchange is active, every vpt_render_pass(es) and sharded vpt_render_adaptive call ends, before the final flag exchange,
 *     with a copy of this rank's depth_buffer and of its active AOV and light-group buffers (vpt_set_aov_buffers,
 *     vpt_set_light_group_buffers) into every rank's planes at the global pixels, so after the call vpt_comm_p2p_layer's planes hold the
 *     single-context frame's buffers bit for bit on every rank, like the accumulators.  Padding rows are not stored; with a render region
 *     only R's pixels are.  A layer that is exported but not active on the context (a NULL buffer, or AOVs / groups not yet activated by an
 *     iteration-0 call) keeps its plane as it is.  Every rank activates the same AOVs and groups, like every other option of a sharded call.
 *     Nothing is copied while the exchange is suspended (vpt_comm_p2p_enable(ctx, 0)) or on one rank (n_ranks == 1: the context's own
 *     buffers are the full frame).  The NCCL exchange does not carry layers: there they stay rank-local.
 *   vpt_comm_p2p_layer returns the full-frame plane of ONE layer bit; a layer the block was exported without is refused (VPT_ERR_INVALID). */
#define VPT_LAYER_DEPTH        0x01u   /* float: depth_buffer */
#define VPT_LAYER_ALPHA        0x02u   /* float: the alpha AOV */
#define VPT_LAYER_VOLUME       0x04u   /* float3: the volume AOV */
#define VPT_LAYER_SUN          0x08u   /* float3: light group sun */
#define VPT_LAYER_POINT        0x10u   /* float3: light group point */
#define VPT_LAYER_EMISSION     0x20u   /* float3: light group emission */
#define VPT_LAYER_ENVIRONMENT  0x40u   /* float3: light group environment */
#define VPT_LAYER_MOTION      0x100u   /* float3: the motion vectors (vpt_set_motion_vectors); its plane follows the seven above, 0x80 is unused */
int  vpt_comm_p2p_export_layers(vpt_context* ctx, int rank, int n_ranks, int stripe_rows, unsigned width, unsigned height, int with_display,
                                unsigned layers, unsigned char handle_out[VPT_P2P_HANDLE_BYTES]);
int  vpt_comm_p2p_layer(vpt_context* ctx, unsigned layer, vpt_devptr_t* d_full);
int  vpt_comm_p2p_block_bytes(unsigned width, unsigned height, int with_display, unsigned layers, size_t* out);

/* Binned exchange layers: the deep slices (vpt_set_deep_buffers) and the instance mattes (vpt_set_instance_mattes) full-frame on every rank.
 *   Export.  vpt_comm_p2p_export_binned is vpt_comm_p2p_export_layers with n_slices (0 or 1..VPT_DEEP_MAX_SLICES) and n_mattes (0 or
 *     1..VPT_MATTE_MAX); 0 leaves that layer out.  vpt_comm_p2p_export_layers is this call with 0, 0: same block, same behaviour.  After the
 *     seven layer planes the block holds the deep slices [n_slices][H][W] float4, then the mattes [n_mattes][H][W] float4, each array on a
 *     256-byte boundary: slice-major and matte-major like the rank-local buffers, at global pixels.  Counts out of range are refused
 *     (VPT_ERR_INVALID).  vpt_comm_p2p_block_bytes_binned sizes the block (pure host code; with both counts 0 it is vpt_comm_p2p_block_bytes).
 *     The block header records the two counts, and vpt_comm_p2p_import / _import_local refuse a peer whose counts differ (VPT_ERR_INVALID,
 *     naming the rank and both counts) and map nothing, as for the layer mask.
 *   Layout and content.  Ranks agree on the layout (the counts, checked at import); the caller on the content: the slice bounds and the
 *     instance -> matte map are not in the block, so every rank sets the same ones, like every other option of a sharded call.
 *   Calls.  Once the exchange is active, a render call whose deep slices are active (registered, and taken over by an iteration-0 call) on a
 *     block that carries deep slices must have exactly n_slices slices, and likewise for the mattes; otherwise the call is refused
 *     (VPT_ERR_INVALID, naming both counts) before it enqueues anything, so no peer is left waiting for it.  To change K, tear the exchange
 *     down (vpt_comm_destroy) and export again.  Every vpt_render_pass(es) and sharded vpt_render_adaptive call then ends, right after the
 *     layer copy, with a copy of the active slices and mattes into every rank's arrays, so after the call vpt_comm_p2p_binned's array holds
 *     the single-context frame's buffer bit for bit on every rank.  Padding rows are not stored; with a render region only R's pixels are.  A
 *     binned layer that is exported but not active on the call keeps its array as it is.  Nothing is copied while the exchange is suspended
 *     or on one rank.  The NCCL exchange does not carry them.
 *   vpt_comm_p2p_binned returns the full-frame array of `which` (VPT_BINNED_DEEP or VPT_BINNED_MATTES) and its count K (k may be NULL); a
 *     layer the block was exported without is refused (VPT_ERR_INVALID). */
#define VPT_BINNED_DEEP    1u   /* the deep slices: [n_slices][H][W] float4 */
#define VPT_BINNED_MATTES  2u   /* the instance mattes: [n_mattes][H][W] float4 */
int  vpt_comm_p2p_export_binned(vpt_context* ctx, int rank, int n_ranks, int stripe_rows, unsigned width, unsigned height, int with_display,
                                unsigned layers, unsigned n_slices, unsigned n_mattes, unsigned char handle_out[VPT_P2P_HANDLE_BYTES]);
int  vpt_comm_p2p_binned(vpt_context* ctx, unsigned which, vpt_devptr_t* d_full, unsigned* k);
int  vpt_comm_p2p_block_bytes_binned(unsigned width, unsigned height, int with_display, unsigned layers, unsigned n_slices, unsigned n_mattes,
                                     size_t* out);

/* ---- the hot path --------------------------------------------------------------------------------
 * vpt_render_pass   replaces ONE launch of the reference `volume_rt_kernel` (render_kernel.cu:2216):
 *                   same inputs, same buffer updates (accum/depth/cost running means, display, raw,
 *                   blue-noise advance).  The caller keeps doing `++kernel_params.iteration`.
 * vpt_render_passes is n consecutive such launches with iteration, iteration+1, ... fused into as few
 *                   kernel rounds as the chunk size allows; the buffers afterwards equal the state after
 *                   n reference launches (display/raw are written once, from the final accumulator).
 * `params` is the cuLaunchKernel argument array (VPT_ARG_* in vpt_abi.h). `stream` is a cudaStream_t.
 * Work is enqueued asynchronously; synchronise the stream (or the device) as the reference loop does. */
int  vpt_render_pass(vpt_context* ctx, void* const params[VPT_NUM_ARGS], void* stream);
int  vpt_render_passes(vpt_context* ctx, void* const params[VPT_NUM_ARGS], unsigned n_passes, void* stream);

/* ---- adaptive sampling: converged pixels stop early --------------------------------------------------
 * vpt_render_adaptive renders ONE new frame (Kernel_params.iteration must be 0; pass k of the frame is the reference launch with
 * iteration k) of at most min(max_passes, max_interactions) passes, and lets each pixel stop once it and its neighbours have converged.
 *
 *   Statistic.  Every pass a pixel takes updates a float32 Welford state of the luminance Y = 0.2126 r + 0.7152 g + 0.0722 b of its
 *     sample, taken exactly as the sample enters the running mean (after the NaN / Inf guard and the viz_dof tint):
 *         n += 1;  d = Y - mean;  mean += d / n;  M2 += d * (Y - mean)
 *     and its relative error is err = sqrt(M2 / (n (n-1))) / max(mean, 1e-3)  (the floor keeps dark pixels from never converging).
 *     The arithmetic is fixed: Y = fma(0.0722, b, fma(0.2126, r, 0.7152 g)), every operation float32 round-to-nearest with subnormal
 *     inputs and results flushed to zero, M2's update a product then a sum (DESIGN.md section 8a).
 *   Tests.  After min_passes passes, then every check_interval passes, a pixel that is still active stops if the largest err over its
 *     3x3 neighbourhood (clipped at the frame edge) is strictly below `threshold`; a neighbour that has already stopped counts with the
 *     last err it had, and a NaN err counts as +Inf, so a pixel with a NaN err and its neighbours never stop.  threshold = 0: no pixel
 *     ever stops; threshold = FLT_MAX (or +Inf): every pixel whose neighbourhood holds only finite errors stops at the first test.
 *   Outputs.  d_pass_count[p] (W*H unsigned, device, required) = the passes pixel p took, and accum, depth, cost, raw and display of p
 *     are bit for bit what vpt_render_passes(d_pass_count[p]) would leave there: the Philox stream is keyed by (pixel, iteration) and
 *     the jitter of a pass does not depend on which pixels sample it.  d_rel_error (W*H float, device, may be NULL) = each pixel's last
 *     err, a noise map of the frame.  *passes_run (host, may be NULL) = the passes issued: min(max_passes, max_interactions), or fewer
 *     when every pixel stopped earlier; the blue-noise buffer is advanced exactly that many times.
 *   Synchronisation.  The call synchronises `stream` once per convergence test, to read back how many 32x4 pixel tiles are still
 *     active; everything else is enqueued asynchronously like vpt_render_passes.
 *   An adaptive frame is final.  vpt_render_passes with iteration > 0 on the accum_buffer of the context's last adaptive frame fails
 *     with VPT_ERR_INVALID; a call with iteration == 0 on it starts a new frame as usual.
 *   Multi-GPU.  A partitioned context renders its share of the frame when its peer-memory exchange is active (vpt_comm_p2p_export, then
 *     vpt_comm_p2p_import or vpt_comm_p2p_import_local, not suspended by vpt_comm_p2p_enable(ctx, 0)).  Every rank makes the same call
 *     with the same options, and the frame is exactly the single-context adaptive frame of the whole image: the 3x3 neighbourhood is taken
 *     over global rows (clipped at the global frame edge), the same passes and tests are issued, every rank returns the same *passes_run
 *     and advances its blue-noise replica that many times, also when all of its own pixels have stopped.  d_pass_count / d_rel_error hold
 *     vpt_local_pixels() entries in rank-local order like the Kernel_params buffers; entries of padding rows (global row >= H) are 0.
 *     When the call returns, every rank's exchange block holds the whole frame: accumulators and display words (vpt_comm_p2p_frame),
 *     pass counts and relative errors (vpt_comm_p2p_adaptive_frame).  Every convergence test waits for all peers, so each rank's call
 *     must be issued by its own host thread or process.  If a peer flag wait gives up (about 10 s), the call issues no further passes and
 *     fails with VPT_ERR_CUDA naming the barrier; the exchange is then out of step and must be set up again.
 *   Refused: render == 0, max_interactions < 2, min_passes < 2, check_interval == 0, a negative or NaN threshold, a subnormal threshold
 *     (0 < threshold < FLT_MIN, which the device would flush to 0), max_passes == 0, a frame size
 *     other than the exported one (VPT_ERR_INVALID); a partitioned context without an active peer exchange -- vpt_set_partition alone, a
 *     suspended exchange -- and the NCCL exchange, whose adaptive frames are not built (VPT_ERR_UNSUPPORTED).  Brick mode and cell mode
 *     work.  opt == NULL takes the defaults. */
typedef struct vpt_adaptive_options {
    unsigned min_passes;       /* passes every pixel takes before it may stop; >= 2 (default 16) */
    unsigned check_interval;   /* passes between two convergence tests; >= 1 (default 16) */
    float    threshold;        /* stop when the relative error of the pixel and of its 8 neighbours is below this (default 0.01) */
} vpt_adaptive_options;
void vpt_adaptive_options_defaults(vpt_adaptive_options* opt);
int  vpt_render_adaptive(vpt_context* ctx, void* const params[VPT_NUM_ARGS], unsigned max_passes, const vpt_adaptive_options* opt,
                         unsigned* d_pass_count, float* d_rel_error, unsigned* passes_run, void* stream);
/* The stopping rule alone, on caller-given samples: d_samples (device, float3 [n_passes][height][width]) are the samples of each pass as
 * they enter the running mean.  Runs vpt_render_adaptive's schedule of chunks and tests on one rank, with the same Welford arithmetic, tile
 * lists and convergence-test kernels, and `region` (NULL, or {x0, y0, x1, y1}) as a render region.  Writes d_pass_count and d_rel_error
 * (device [H][W], d_rel_error may be NULL) for the pixels that sample, as vpt_render_adaptive does, and at test t < max_tests every
 * pixel's err as the test reads it into d_test_err[t] (device [max_tests][H][W]; NaN outside the region, so a test that read
 * a pixel outside the region would hold its neighbours running).  *passes_run / *n_tests (host,
 * may be NULL): the passes issued and the tests run.  Synchronises the device.  Options are refused as vpt_render_adaptive refuses them. */
int  vpt_debug_adapt_rule(const float* d_samples, unsigned width, unsigned height, unsigned n_passes, const vpt_adaptive_options* opt,
                          const unsigned* region, unsigned* d_pass_count, float* d_rel_error, float* d_test_err, unsigned max_tests,
                          unsigned* passes_run, unsigned* n_tests);

/* ---- compositing AOVs: how much of each pixel is volume, and the volume's colour without the background ----------------------
 * accum_buffer holds the volume over the environment.  With AOV buffers set, every render call also keeps, per pixel, two running
 * means next to it, so the frame can be composited over another plate and the environment swapped or graded downstream.
 *
 *   Definition.  For each pass a pixel takes, let c = (depth > 0), where depth is the pass's depth sample (the one depth_buffer
 *     averages) and a NaN depth counts as false: c is the reference's own decision that the camera ray's first walk collided in the
 *     medium, or that the ray hit the sphere before the volume box.
 *       alpha   sample: c ? 1 : 0.
 *       volume  sample (float3): the sample exactly as it enters accum (after the NaN / Inf guard and the viz_dof tint) if c, +0 otherwise
 *               (a select, not a product).  When the guard replaced the sample, the volume sample is the volume AOV's own mean so far,
 *               as the guard uses accum's (at iteration 0: the buffer's previous content, as for accum).  Alpha is not guarded.
 *     Both follow accum's rule and arithmetic: iteration == 0 assigns, iteration < max_interactions updates x + (s - x) / (iteration + 1),
 *     later passes change nothing.  So per sample, beauty = volume + the transmitted background, and alpha estimates 1 - transmittance
 *     along the camera ray under the reference's tracker; over a new plate P the frame is  volume + (1 - alpha) * P.
 *   Sphere.  The sphere seen THROUGH the volume box without a collision counts as background (c is false there): that is the
 *     reference's depth decision.
 *   Buffers.  Caller-owned device memory of vpt_local_pixels() entries like the Kernel_params buffers (rank-local order on a partitioned
 *     context): d_alpha float, d_volume_f3 float3.  Either may be NULL; both NULL turns the AOVs off at once.  Buffers registered here
 *     become active at the next render call whose Kernel_params.iteration is 0; calls before that leave them untouched, so a viewer loop
 *     that enables AOVs mid-frame never continues a mean from garbage (vpt_render_adaptive always starts at 0).
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update the active AOVs.  An adaptive frame's stopped pixels keep theirs, and every
 *     pixel's AOVs are bit for bit what a fixed-count frame of its own pass count leaves there.  Level (A) (volume_rt_kernel) has none.
 *     On a partitioned context the buffers are rank-local; the peer-memory exchange carries them full-frame to every rank when the block is
 *     exported with VPT_LAYER_ALPHA / VPT_LAYER_VOLUME (vpt_comm_p2p_export_layers).  The NCCL exchange does not carry them.
 *   Refused at render time (VPT_ERR_INVALID, naming the buffer): an AOV buffer that overlaps accum, depth, cost, raw or display, and
 *     the two AOV buffers overlapping each other. */
int  vpt_set_aov_buffers(vpt_context* ctx, float* d_alpha, float* d_volume_f3);

/* ---- light groups: the beauty split by the light class that added each radiance term ------------------------------------------
 * With group buffers set, every render call also keeps, per pixel, four running means next to accum -- the radiance the sun, the point
 * lights, the volume's emission and the environment added -- so a compositor can regrade or swap each class without re-rendering.
 *
 *   Definition.  Every radiance term the integrator adds to the path's L, and the environment term at the end of the path, belongs to
 *     exactly one group.  Direct integrator: sun NEE and the sun-lit sphere bounce -> sun; the point-light estimate -> point; the emission
 *     walk -> emission; the HDRI / precomputed-sky term -> environment.  Volumetric path integrator: each scatter's light estimate goes to
 *     the class uniform_sample_one_light chose (sun, point, or environment for both halves of the sky estimate), the emission walk to
 *     emission, the end-of-path sky to environment.  A miss sample is all environment; a pass that samples nothing (render == 0) gives its
 *     WHITE to the environment and 0 to the others.  Each group follows accum's rule and arithmetic (iteration == 0 assigns,
 *     iteration < max_interactions updates x + (s - x) / (iteration + 1)); a sample the NaN / Inf guard replaced leaves every group at its
 *     own mean (at iteration 0: the buffer's previous content, as accum takes accum_buffer's).  Groups are taken before the viz_dof tint.  So per sample sun + point + emission + environment = the beauty sample up to
 *     the rounding of the separate sums, and with the direct integrator each group is bit for bit the accum of a render in which only that
 *     class is lit (the path's draws do not depend on light intensities there).
 *   Buffers.  Caller-owned device memory, float3, vpt_local_pixels() entries each (rank-local order on a partitioned context).  Any may be
 *     NULL; all four NULL turns the groups off at once.  Activation as for the AOVs: registered buffers take over at the next render call
 *     whose Kernel_params.iteration is 0, calls before that leave them untouched.
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update the active groups; an adaptive frame's stopped pixels keep theirs.  Every
 *     other output is bit for bit what the same call gives without groups.  Level (A) has none.  On a partitioned context the buffers are
 *     rank-local; the peer-memory exchange carries them full-frame to every rank when the block is exported with VPT_LAYER_SUN, _POINT,
 *     _EMISSION, _ENVIRONMENT (vpt_comm_p2p_export_layers).  The NCCL exchange does not carry them.
 *   Cost.  Groups make the lean kernels write wide sample records and the generic kernels keep 48 B more per sample (the chunk shrinks
 *     under max_scratch_mb accordingly).
 *   Refused at render time (VPT_ERR_INVALID, naming the buffer): a group buffer that overlaps accum, depth, cost, raw or display, an AOV
 *     buffer, or another group buffer. */
int  vpt_set_light_group_buffers(vpt_context* ctx, float* d_sun_f3, float* d_point_f3, float* d_emission_f3, float* d_environment_f3);

/* ---- deep slices: the compositing AOVs binned by the camera ray's collision depth ------------------------------------------------
 * alpha and volume flatten the whole camera ray, so an element at distance z can only go in front of the volume or behind it.  With a
 * slice buffer set, every render call also keeps the two AOVs split into K depth intervals, so an element can be put INSIDE the cloud
 * (deep compositing: a holdout at z keeps the slices in front of it).
 *
 *   Slices.  K = n_slices intervals given by the host bounds z_0 < z_1 < ... < z_K (copied at the call), in the units of depth_buffer:
 *     distance along the camera ray from its origin (the lens sample for a thin lens, the camera origin for a panorama).  A pass sample
 *     of depth d (the one depth_buffer averages) falls in slice k when d > 0, z_k <= d, and d < z_{k+1} or z_{k+1} = +inf.  So a NaN, a
 *     miss and a depth outside [z_0, z_K) fall in no slice, and at most one slice takes a sample.
 *   Per slice, per pixel one float4: (r, g, b) the premultiplied colour, w the coverage.
 *       coverage sample: 1 if the sample falls in slice k, else 0 (not guarded).
 *       colour   sample: the sample exactly as it enters accum (after the NaN / Inf guard and the viz_dof tint, as for the volume AOV) if it
 *                falls in slice k, +0 otherwise (a select, not a product).  When the guard replaced the sample, every slice's colour sample
 *                is that slice's own mean so far (at iteration 0: the buffer's previous content).
 *     Both follow accum's rule and arithmetic: iteration == 0 assigns, iteration < max_interactions updates x + (s - x) / (iteration + 1),
 *     later passes change nothing.  So K = 1 with bounds {0, +inf} is (volume, alpha) bit for bit; slice k of any K is bit for bit the one
 *     slice of a K = 1 frame with bounds {z_k, z_{k+1}}; with z_0 = 0 and z_K = +inf the slices sum to the AOVs up to the rounding of the
 *     separate means.  A pass that samples nothing (render == 0, the kernel tail) gives coverage 0 and colour +0.
 *   Buffer.  Caller-owned device memory of K * vpt_local_pixels() float4, slice-major [K][local pixel] (rank-local order on a partitioned
 *     context), 16-byte aligned (cudaMalloc's memory is).  A NULL buffer turns the slices off at once (n_slices and h_bounds are then ignored).  Buffer, K and bounds take over at the
 *     next render call whose Kernel_params.iteration is 0; calls before that leave the buffer untouched.
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update the active slices.  An adaptive frame's stopped pixels keep theirs, and every
 *     pixel's slices are bit for bit what a fixed-count frame of its own pass count leaves there.  A render region writes no slice outside
 *     it.  Every other output is bit for bit what the same call gives without slices.  Level (A) has none.  On a partitioned context the
 *     buffer is rank-local; the peer-memory exchange carries the slices full-frame to every rank when the block is exported with n_slices =
 *     K (vpt_comm_p2p_export_binned, which then refuses a call with another active K).  The NCCL exchange does not carry them.
 *   Cost.  A second resolve kernel per chunk: it reads the chunk's sample records again, reads and writes each slice once per pixel
 *     (K * 32 B) plus once per sample that lands in a slice, and updates every slice once per pass (DESIGN.md section 8h).
 *   Refused when set (VPT_ERR_INVALID), with a non-NULL buffer: a buffer not 16-byte aligned, n_slices outside 1..VPT_DEEP_MAX_SLICES,
 *     NULL h_bounds, a NaN or negative bound, bounds not strictly increasing, +inf anywhere but z_K.  A refused call changes nothing.
 *   Refused at render time (VPT_ERR_INVALID, naming the buffer): a slice buffer that overlaps accum, depth, cost, raw or display, an AOV
 *     buffer or a light-group buffer. */
#define VPT_DEEP_MAX_SLICES 32
int  vpt_set_deep_buffers(vpt_context* ctx, float* d_slices_f4, unsigned n_slices, const float* h_bounds /* n_slices + 1 */);

/* ---- instance mattes: the compositing AOVs split by the volume instance of each camera ray's first collision ---------------------
 * alpha and volume flatten every instance into one coverage.  With a matte buffer set, every render call also keeps the two AOVs split by
 * WHICH volume the camera ray collided with first (an ID matte), so one cloud of a cloudscape can be isolated, graded or held out without
 * rendering it alone -- which would change the octree, the majorant walk and every draw after it.
 *
 *   Id of a sample.  A pass sample whose collision decision c = depth > 0 holds (as for the AOVs; a NaN depth is none) gets an id: the
 *     sphere when the camera ray hit the reference sphere before the volume box; otherwise the volume instance of the first walk's accepted
 *     collision (the collision depth measures).  The walk accepts where sigma_max^-1 * density > u, density the float sum over the start
 *     leaf's instance list in list order at the collision point; the instance is the first list entry i whose prefix sum over entries 0..i
 *     (the same additions, point and u) passes the same test.  The last prefix is the density itself, so an accepted collision always finds
 *     an instance (with negative densities too).  No draw is added: paths are those of a render without mattes.  Each overlapping
 *     instance takes a collision with probability density_i / density while sigma_max^-1 * density <= 1.  The root majorant is a maximum
 *     over instances, not a sum, so where overlapping instances add up past it every step is accepted and the first list entries are
 *     favoured.  A single-volume scene's id is always instance 0.
 *   Mattes.  h_matte_of_instance[i] (copied at the call) maps instance i to one of K = n_mattes mattes or to none (-1); sphere_matte maps the
 *     sphere.  Per matte and pixel one float4: (r, g, b) the premultiplied colour, w the coverage, defined exactly as a deep slice with "its
 *     id maps to matte k" for "falls in slice k": coverage sample 1 or 0 (not guarded); colour sample the sample as the volume AOV takes it,
 *     or +0 (a select); a sample the guard replaced gives every matte its own mean; accum's rule and arithmetic; a pass that samples nothing
 *     gives coverage 0 and colour +0.  So K = 1 with every instance and the sphere in matte 0 is (volume, alpha) bit for bit; matte k of
 *     any K is bit for bit the single matte of a K = 1 frame whose map selects the same set; with every id mapped the mattes sum to the AOVs
 *     up to the rounding of the separate means.
 *   Buffer.  Caller-owned device memory of K * vpt_local_pixels() float4, matte-major [K][local pixel] (rank-local order on a partitioned
 *     context), 16-byte aligned.  A NULL buffer turns the mattes off at once (the other arguments are then ignored).  Buffer, K and map take
 *     over at the next render call whose Kernel_params.iteration is 0; calls before that leave the buffer untouched.
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update the active mattes, as they do the deep slices (adaptive frames, render
 *     regions, panoramas with the miss cull).  Every other output is bit for bit what the same call gives without mattes.  Level (A) has
 *     none.  On a partitioned context the buffer is rank-local; the peer-memory exchange carries the mattes full-frame to every rank when
 *     the block is exported with n_mattes = K (vpt_comm_p2p_export_binned, which then refuses a call with another active K).  The NCCL
 *     exchange does not carry them.
 *   Cost.  The trace kernel writes 4 B per sample whose camera ray collided (generic kernels: one pass over the leaf list per first
 *     collision), and a resolve kernel more per chunk reads the records again.  The trace kernel keeps the rays per lane of
 *     the frame without mattes (DESIGN.md section 8l).
 *   Refused when set (VPT_ERR_INVALID), with a non-NULL buffer: a buffer not 16-byte aligned, n_mattes outside 1..VPT_MATTE_MAX, a NULL map
 *     with n_instances > 0, a map entry or sphere_matte outside -1..n_mattes - 1.  A refused call changes nothing.  A NULL map with
 *     n_instances == 0 is an empty map, accepted when set on purpose: every scene has at least one instance, so the first render call
 *     refuses it for its instance count.
 *   Refused at render time: n_instances other than the scene's instance count (VPT_ERR_INVALID); a matte buffer that overlaps accum, depth,
 *     cost, raw or display, an AOV, light-group or deep-slice buffer (VPT_ERR_INVALID, naming the buffer); brick or cell mode
 *     (VPT_ERR_UNSUPPORTED). */
#define VPT_MATTE_MAX 32
int  vpt_set_instance_mattes(vpt_context* ctx, float* d_mattes_f4, unsigned n_mattes, const int* h_matte_of_instance, unsigned n_instances,
                             int sphere_matte);

/* ---- render region: sample and write only a rectangle of the frame ------------------------------------------------------------
 * A viewer that tunes the density, the phase or a light on part of a volume re-renders only that part.  The region R is the half-open
 * rectangle [x0, x1) x [y0, y1) in pixels of the full frame, also on a partitioned context; (0, 0, 0, 0) clears it.
 *
 *   Activation.  A region set or cleared here takes effect at the next render call whose Kernel_params.iteration is 0; calls before that
 *     keep the old one (the rule of the AOVs and light groups).  A viewer that moves the region resets the iteration, as on every scene
 *     edit, so no pixel ever continues a running mean from another frame.
 *   vpt_render_pass(es).  Every pixel of R gets bit for bit what the same call gives without a region: accum, depth, cost, raw, display,
 *     the active AOVs and light groups -- also in the passes that sample nothing (render == 0, iteration >= max_interactions).  Outside R
 *     nothing is written, in the caller's buffers or in the peer-exchange frame.  The blue-noise buffer is advanced exactly as without a
 *     region (its limit still comes from the full resolution).  A partitioned context renders R's rows among its stripes; the peer exchange
 *     stores only R's pixels into every rank's frame, which inside R is then the single-context region frame bit for bit.  The NCCL
 *     exchange gathers the rank-local buffers as they are, so outside R the gathered frame holds whatever those buffers held.
 *   vpt_render_adaptive (one context).  Only R's pixels take passes; the 3x3 neighbourhood is clipped at R's edge, so the rule is the one
 *     above applied to R as if R were the frame.  d_pass_count and d_rel_error outside R are left untouched.  R = the whole frame gives the
 *     frame without a region.  A sharded adaptive frame with a region set is refused (VPT_ERR_UNSUPPORTED).
 *   Refused at render time (VPT_ERR_INVALID, naming the bound): x0 >= x1, y0 >= y1, x1 > resolution.x, y1 > resolution.y.  R need not be
 *     aligned to anything; 1 x 1 is legal.
 *   Cost.  The sample scratch keeps its full-frame size, and every chunk still prepares the whole blue-noise jitter table and starts the
 *     persistent trace grid, so a small region has a floor of a few tens of microseconds per chunk.  Level (A) has no regions. */
int  vpt_set_render_region(vpt_context* ctx, unsigned x0, unsigned y0, unsigned x1, unsigned y1);

/* ---- camera projection: perspective (the reference camera) or an equirectangular panorama -------------------------------------
 * A cloudscape baked into an environment map, a dome or a VR frame is a latitude-longitude panorama.  VPT_PROJECTION_EQUIRECT takes
 * the orientation of the caller's camera (vpt_camera_look_at): forward -w, right u, up v.  Pixel (x, y) at jitter (jx, jy) has
 * s = (x + jx) / W, t = (y + jy) / H, phi = (s - 1/2) hfov, theta = (t - 1/2) vfov, and its ray is (origin, normalize(b0)) with
 * b0 = cos theta (sin phi u - cos phi w) + sin theta v.  Row 0 is at the bottom, as with the reference's `vertical`; phi grows to the
 * right.  hfov_deg = 360, vfov_deg = 180 is the full sphere.
 *
 *   Activation.  A projection set here takes effect at the next render call whose Kernel_params.iteration is 0; calls before that keep
 *     the old one (the rule of the AOVs, light groups and regions).  VPT_PROJECTION_PERSPECTIVE (the default) brings the reference camera
 *     back; its fields of view are ignored.
 *   Samples.  A sample draws exactly what a pinhole sample draws (the lens rejection loop and the shutter-time draw), from the pixel's own
 *     Philox stream; from the ray on it is the reference kernel's path, to the parity a perspective frame has.  Everything else works as
 *     with a perspective camera: adaptive frames, render regions, AOVs, light groups, brick mode, both integrators, partitioned contexts
 *     and both exchanges.  The miss cull
 *     (option "miss_cull") skips the pixels of an HDRI panorama that cannot reach the volume or the sphere, with the same result bit for bit.
 *   Refused when set (VPT_ERR_INVALID): an unknown kind; for VPT_PROJECTION_EQUIRECT an hfov_deg outside (0, 360] or a vfov_deg outside
 *     (0, 180] (NaN included).  Refused at render time (VPT_ERR_UNSUPPORTED): an equirectangular frame with camera.lens_radius != 0.
 *   Level (A) has no projections. */
#define VPT_PROJECTION_PERSPECTIVE 0
#define VPT_PROJECTION_EQUIRECT    1
int  vpt_set_projection(vpt_context* ctx, int kind, double hfov_deg, double vfov_deg);
/* Diagnostic: writes, for every local pixel, float4 (b0, 0) -- the ray direction before normalize that the next render call's first pass
 * gives that pixel: pano_b0 of the projection that call takes, or the reference camera's llc + s horizontal + t vertical - origin, at the
 * jitter the blue-noise buffer holds now.  Reads params (camera, Kernel_params, blue noise); writes d_out_f4 only, on the default stream. */
int  vpt_debug_camera_rays(vpt_context* ctx, void* const params[VPT_NUM_ARGS], float* d_out_f4);

/* ---- omni-directional stereo (ODS): a stereo panorama for VR players, domes and video platforms -------------------------------------
 * A mono panorama seen in a headset has no depth.  VPT_PROJECTION_ODS renders each eye's panorama from a point on a circle of radius ipd/2
 * around the camera origin, so that every ray is tangent to that circle (the ODS construction every VR player expects).  The orientation is
 * the camera's, as for VPT_PROJECTION_EQUIRECT: forward -w, right u, up v; row 0 at the bottom.
 *
 *   The sample's camera.  For pixel (x, y) at jitter (jx, jy): the layout gives the eye e (-1 left, +1 right), the row y_e within the eye and
 *     the eye's height H_e (H, or H/2 over-under).  (phi, theta) and b0 are the equirectangular projection's at resolution (W, H_e), row y_e.
 *     The pole merge k is 1 for |theta| <= from, 0 for |theta| >= to and (to - |theta|) / (to - from) in between, so the circle shrinks to the
 *     centre near the poles (a step when from == to).  With s = (e ipd/2) k and r = cos phi u + sin phi w (the viewer's right at azimuth phi),
 *     the sample's camera has origin' = fma(s, r, origin), lower_left_corner' = origin' + b0, horizontal = vertical = 0 and the caller's
 *     u, v, w.  Its ray is the reference's camera::get_ray of that camera, bit for bit (the pinhole rule of the perspective camera), so
 *     from the ray on every sample is the reference kernel's path for it.  Depth (and with it the AOVs' and deep slices' collision depth)
 *     is measured from origin'.  The direction is llc' - origin', which is b0 only up to a rounding that grows with |origin| -- as the
 *     reference's own perspective camera, whose lower_left_corner is stored in absolute coordinates too.
 *   Layouts.  VPT_ODS_OVER_UNDER (the delivery format of VR players and video platforms): rows [H/2, H) -- the top, since row 0 is the
 *     bottom -- are the left eye, rows [0, H/2) the right eye; H must be even.  VPT_ODS_LEFT / VPT_ODS_RIGHT: the whole frame is one eye.
 *   Activation.  As vpt_set_projection: from the next render call whose Kernel_params.iteration is 0; vpt_set_projection(PERSPECTIVE or
 *     EQUIRECT) switches back.
 *   Works with vpt_render_pass(es), vpt_render_adaptive, render regions, AOVs, light groups, deep slices, brick and cell mode, both
 *     integrators, both environments, partitioned contexts and both exchanges (a sharded adaptive frame with a region stays refused).  The
 *     miss cull (option "miss_cull") skips the pixels of an HDRI frame that no ray from any point of the viewing circle can take to the
 *     volume or the sphere, with the same result bit for bit.  An ODS frame runs no octree pre-step and keeps a per-ray origin, so it costs
 *     more than an equirectangular frame of the same size.
 *   Refused when set (VPT_ERR_INVALID; the projection stays as it was): vpt_set_projection with VPT_PROJECTION_ODS (its options are
 *     missing); the field-of-view ranges of VPT_PROJECTION_EQUIRECT; a negative or non-finite ipd; an unknown layout; pole-merge angles
 *     outside 0 <= from <= to <= 90.  Refused at render time (VPT_ERR_UNSUPPORTED): camera.lens_radius != 0; camera motion;
 *     VPT_ODS_OVER_UNDER with an odd height.  Level (A) has no ODS projection. */
#define VPT_PROJECTION_ODS 2
#define VPT_ODS_LEFT       0   /* the whole frame is the left eye */
#define VPT_ODS_RIGHT      1   /* the whole frame is the right eye */
#define VPT_ODS_OVER_UNDER 2   /* rows [H/2, H) (the top: row 0 is the bottom) left eye, rows [0, H/2) right eye; H must be even */
typedef struct vpt_ods_options {
    float ipd;                  /* interocular distance in scene units; finite, >= 0 (default 0.064) */
    int   layout;               /* VPT_ODS_* (default VPT_ODS_OVER_UNDER) */
    float pole_merge_from_deg;  /* the eye separation is full up to this |elevation| ... (default 60) */
    float pole_merge_to_deg;    /* ... and 0 from this one on, linear in between; 0 <= from <= to <= 90 (default 75) */
} vpt_ods_options;
void vpt_ods_options_defaults(vpt_ods_options* opt);
int  vpt_set_projection_ods(vpt_context* ctx, double hfov_deg, double vfov_deg, const vpt_ods_options* opt);  /* opt NULL = defaults */
/* Diagnostic: writes, for every local pixel, 8 floats: origin' (3), lower_left_corner' (3), e and k of the camera of that pixel's sample in
 * the next render call's first pass, at the jitter the blue-noise buffer holds now (padding rows of a partitioned context all 0).  Reads
 * params (camera, Kernel_params, blue noise); writes d_out only, on the default stream, and leaves the blue noise as it is.  VPT_ERR_INVALID
 * when the next call has no ODS projection.  vpt_debug_camera_rays on an ODS frame writes llc' - origin' of that camera (camera_b0). */
int  vpt_debug_ods_cameras(vpt_context* ctx, void* const params[VPT_NUM_ARGS], float* d_out);

/* ---- camera motion: motion blur from a camera that moves between two poses over the shutter --------------------------------------
 * The reference draws a shutter time for every camera ray (camera::get_ray, right after the lens rejection loop) and never reads it.
 * Here that draw, xi in (0, 1] from the pixel's Philox stream, places the sample's camera between two poses: the Kernel_params camera is
 * the pose at shutter open, `shutter_close` (typically a second vpt_camera_look_at) the pose at shutter close.  The call copies it; NULL
 * clears the motion.
 *
 *   The sample's camera.  Its origin, lower_left_corner, horizontal, vertical, u and v are, per component, c == o ? o : fma(xi, c - o, o)
 *     (o the open pose's value, c the close pose's).  A component that does not move keeps the open pose's bits, -0 included, so a pure
 *     translation keeps the basis and shutter_close == the open camera is the static camera.  xi = 1 reaches the close pose only up to the
 *     rounding of c - o.  The weight is xi itself: time0 and time1 stay unread, as in the reference.  lens_radius, focus_dist and viz_dof
 *     are the open camera's; shutter_close's copies, its w, time0 and time1 are not read.  No draw of any path changes, so every sample is
 *     the reference kernel's path for the ray of the reference camera whose fields are that sample's camera.  Depth (and with it the
 *     AOVs' and deep slices' collision depth) is measured from the sample's own origin.
 *   Activation.  Motion set or cleared here takes effect at the next render call whose Kernel_params.iteration is 0; a continued frame
 *     keeps the pose it started with (the rule of the projection and regions).
 *   Works with vpt_render_pass(es), vpt_render_adaptive, render regions, AOVs, light groups, deep slices, brick mode, both integrators,
 *     both environments, partitioned contexts and both exchanges.  A motion frame runs no miss cull (option "miss_cull") and keeps every
 *     sample record, so it costs more than a static frame even when the poses are equal.
 *   Refused when set (VPT_ERR_INVALID; the motion is left as it was): a non-finite component in any of the six interpolated fields of
 *     shutter_close.  Refused at render time (VPT_ERR_UNSUPPORTED): motion with VPT_PROJECTION_EQUIRECT.  Level (A) has no motion. */
int  vpt_set_camera_motion(vpt_context* ctx, const vpt_camera* shutter_close);
/* Diagnostic: writes, for every local pixel, 20 floats: the shutter draw xi of the next render call's first pass, then origin,
 * lower_left_corner, horizontal, vertical, u and v of that sample's camera (19 floats, padded with 0; padding rows of a partitioned
 * context all 0), the same bits the generator computes.  Reads params (camera, Kernel_params); writes d_out only, on the default stream,
 * and leaves the blue noise as it is.  VPT_ERR_INVALID when the next call has no camera motion.  vpt_debug_camera_rays refuses such a
 * call (VPT_ERR_UNSUPPORTED): its rays depend on each sample's draw. */
int  vpt_debug_motion_cameras(vpt_context* ctx, void* const params[VPT_NUM_ARGS], float* d_out);

/* ---- motion vectors: each pixel's screen-space motion of the camera ray's first collision towards a second camera pose --------------
 * With a vector buffer set, every render call also keeps, per pixel, where the point each sample's camera ray first collided with moves on
 * the film when the camera goes from the frame's pose A (the Kernel_params camera; the shutter-open pose of a motion frame) to a target pose
 * B -- the input of a vector blur in post, of retiming and of temporal filtering.
 *
 *   Definition.  For each pass a pixel takes, let c = (depth > 0) as for the alpha AOV (a NaN depth counts as false).  If c holds, the
 *     sample's first collision is P = org + depth * dir, with (org, dir) the sample's camera ray exactly as the generator built it (pinhole:
 *     the camera origin and normalize(llc + s horizontal + t vertical - origin) at the pass's jitter; thin lens: origin + the lens offset and
 *     the lens loop's direction; camera motion: the ray of the sample's camera at its shutter draw).  The film projection pi_K(P) of a camera
 *     K reads only its origin, lower_left_corner, horizontal and vertical: d = P - origin, e = llc - origin, n = cross(horizontal, vertical),
 *     k = (e . n) / (d . n), q = k d - e, and (s, t) solving q = s horizontal + t vertical (the 2x2 normal equations; the dot-product form
 *     when horizontal . vertical == 0); pi_K(P) = (s W, t H), the units of the film position (x + jx, y + jy): pixels along the column and
 *     the buffer's row index.  A thin lens therefore projects through its lens centre.  The sample vector is pi_B(P) - pi_A(P), or (+0, +0)
 *     when k <= 0 or the result is not finite for A or B (the point is not in front of that camera; the sample still counts as covered).
 *   Buffer.  Per pixel one float3: the running means of (c vx, c vy, c) in accum's rule and arithmetic (iteration == 0 assigns,
 *     iteration < max_interactions updates x + (s - x) / (iteration + 1), later passes change nothing), not guarded.  So z is the alpha AOV
 *     bit for bit, xy / z is the unpremultiplied vector, B == A gives +0 in x and y everywhere, and a miss or a pass that samples nothing
 *     adds exact zeros.  Caller-owned device memory of vpt_local_pixels() float3 (rank-local order on a partitioned context).
 *   Activation.  As for the AOVs: a buffer and target set here take over at the next render call whose Kernel_params.iteration is 0; calls
 *     before that leave the buffer untouched.  A NULL buffer turns the vectors off at once (target is then ignored).  The call copies target.
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update the active vectors (an adaptive frame's stopped pixels keep theirs; a render
 *     region writes none outside it).  Every other output is bit for bit what the same call gives without vectors: a kernel of its own reads
 *     each sample's depth word next to the frame's resolve.  On a partitioned context the buffer is rank-local; the peer-memory exchange
 *     carries it full-frame to every rank when the block is exported with VPT_LAYER_MOTION.  The NCCL exchange does not carry it.  Level (A)
 *     has no vectors.
 *   Refused when set (VPT_ERR_INVALID; the vectors are left as they were): a NULL target with a buffer, a non-finite component of target's
 *     origin, lower_left_corner, horizontal or vertical.  Refused at render time: VPT_PROJECTION_EQUIRECT and VPT_PROJECTION_ODS
 *     (VPT_ERR_UNSUPPORTED); a buffer that overlaps accum, depth, cost, raw, display, an AOV, light-group, deep-slice or matte buffer
 *     (VPT_ERR_INVALID, naming the buffer). */
int  vpt_set_motion_vectors(vpt_context* ctx, float* d_vectors_f3, const vpt_camera* target);

/* ---- collision AOVs: world position, normal and albedo at each sample's first collision -------------------------------------------
 * The utility passes a compositor and a denoiser expect next to the beauty: world position P (relighting, position masks, fog, a
 * disocclusion test), the normal N (relighting, a denoiser guide) and the albedo (the second guide of OIDN and the OptiX denoiser).
 *
 *   Definition.  For each pass a pixel takes, let c = (depth > 0) as for the alpha AOV (a NaN depth counts as false).  If c holds:
 *     P = org + depth * dir, with (org, dir) the sample's camera ray exactly as the generator built it (as for vpt_set_motion_vectors:
 *     pinhole, thin lens, the camera of the shutter draw under camera motion, keyed by the sample offset + iteration).  The depth pass's own
 *     test on that ray (nearest of the octree root box and the sphere) tells what P lies on:
 *     - Sphere: n = normalize(P - centre), albedo = the sphere's colour, the reflectance the integrators' sphere branch multiplies the
 *       throughput by.
 *     - Volume: rho(X) is the density the frame's tracker reads -- volume 0 through the frame's sampler (texture, brick pool or cell table)
 *       in a single-volume scene, else the sum over the leaf list of the octree leaf that contains X (0 in no populated leaf).
 *       g_i = (rho(P + h e_i) - rho(P - h e_i)) / (2h) with h = gradient_step in world units; n = -g / |g|, or (0, 0, 0) when g . g is 0
 *       or not finite in float32.  albedo = Kernel_params.albedo * Cd(P) * density_color[index(rho(P))] / Kernel_params.extinction *
 *       energy_inject: the throughput factor an accepted collision at P applies, with Cd the leaf colour (volume 0's colour grid, clamped
 *       at 0, for one volume) and index = floor(clamp(rho / max_extinction * 255 / emission_pivot, 0, 255)).  Where P lies in no populated
 *       leaf rho and Cd are 0 and the expression is evaluated as written.
 *     Non-finite results are stored as they come (not guarded, as the motion vectors).
 *   Buffers.  Per pixel the running means in accum's rule and arithmetic (iteration == 0 assigns, iteration < max_interactions updates
 *     x + (s - x) / (iteration + 1), later passes change nothing) of: position float4 (c Px, c Py, c Pz, c) -- w is the alpha AOV bit for bit
 *     and a one-pass frame holds P exactly; normal float3 c n (premultiplied: callers normalise); albedo float3 c a (premultiplied by the
 *     coverage).  A miss or a pass that samples nothing adds exact zeros.  Caller-owned device memory of vpt_local_pixels() entries each
 *     (rank-local order on a partitioned context).  Any buffer may be NULL; all three NULL turns the layers off at once.
 *   Activation.  As for the AOVs: buffers set here take over at the next render call whose Kernel_params.iteration is 0.
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update the active layers (an adaptive frame's stopped pixels keep theirs; a render
 *     region writes nothing outside it).  Works with camera motion, thin lens, both integrators, all three environments, instanced scenes,
 *     brick and cell mode, partitioned contexts and vpt_set_sample_offset.  Every other output is bit for bit what the same call gives
 *     without them: a kernel of its own reads each sample's depth word next to the frame's resolve, and runs the look-ups (seven density
 *     and one colour fetch) only for covered samples.  Neither exchange carries the layers.  Level (A) has none.
 *   Refused when set (VPT_ERR_INVALID; the layers are left as they were): a normal buffer with a gradient_step that is not finite or <= 0.
 *     Refused at render time: VPT_PROJECTION_EQUIRECT and VPT_PROJECTION_ODS (VPT_ERR_UNSUPPORTED); a buffer that overlaps accum, depth,
 *     cost, raw, display, an AOV, light-group, deep-slice, matte or motion-vector buffer, or another of the three (VPT_ERR_INVALID, naming
 *     the buffers). */
int  vpt_set_collision_aovs(vpt_context* ctx, float* d_position_f4, float* d_normal_f3, float* d_albedo_f3, float gradient_step);

/* ---- Cryptomatte: per-pixel instance coverage ranked by id, keyed after the render ----------------------------------------------
 * The industry's ID matte (Nuke, Fusion, Houdini and Resolve key it natively): each pixel keeps how many of its camera rays collided first
 * with each volume instance (or the sphere), and the user picks the ids afterwards.  Unlike the instance mattes nothing is declared before
 * the render and there is no plane per set.
 *
 *   State.  Caller-owned device memory of uint32, 2 + 2 S planes of vpt_local_pixels() entries each, plane-major (rank-local order on a
 *     partitioned context), S = capacity in 1..VPT_CRYPTO_MAX_ENTRIES: plane 0 n (the passes counted), plane 1 overflow, plane 2 + 2j id_j,
 *     plane 3 + 2j count_j.  4-byte aligned.
 *   Per pass.  For pass p of a call at Kernel_params.iteration = i, with it = i + p, in this order:
 *     1. it >= max_interactions: nothing changes (accum's gate);
 *     2. it == 0: the pixel is cleared first (n, overflow and every id_j and count_j set to 0; accum's "iteration 0 assigns");
 *     3. n += 1;
 *     4. if c = depth > 0 (the alpha AOV's decision; a NaN depth is false), the sample's id -- the instance of its camera ray's first
 *        collision, or 0xffffffff for the sphere, exactly the id of the instance mattes -- goes to the entry that holds it (count_j > 0 and
 *        id_j == id: count_j += 1), otherwise to the first entry with count_j == 0 (it takes (id, 1)), otherwise overflow += 1.
 *     So a pass that samples nothing (Kernel_params.render == 0, a pixel the miss cull removed) counts in n and adds no id; entries fill in
 *     first-seen order and stay a prefix of the table; the state is exact integer arithmetic, so chunks, fused passes, single passes and a
 *     continued call give the same bits, and an adaptive frame's pixel holds the state of a fixed-count frame of its own pass count.  For any
 *     set of ids, sum(count_j over the set) / n estimates the coverage that set's instance matte keeps (exactly: n * matte.w rounds to it).
 *     The rules assume a state this library wrote since an iteration-0 call (as accum does).
 *   Activation.  A NULL state turns the Cryptomatte off at once (capacity is then ignored).  Otherwise state and capacity take over at the
 *     next render call whose Kernel_params.iteration is 0; calls before that leave the state untouched.
 *   Calls.  vpt_render_pass(es) and vpt_render_adaptive update it (an adaptive frame's stopped pixels keep their state; a render region
 *     writes nothing outside it; panoramas and the miss cull as the mattes).  The trace kernel writes the id plane of the instance mattes
 *     (the mattes' trace kernels, one plane shared by both); a kernel of its own reads the depth words and the ids next to the frame's
 *     resolve.  Every other output is bit for bit what the same call gives without it.  On a partitioned context the state is rank-local;
 *     neither exchange carries it.  Level (A) has none.
 *   Refused when set (VPT_ERR_INVALID; the Cryptomatte is left as it was): a non-NULL state with capacity outside 1..VPT_CRYPTO_MAX_ENTRIES
 *     or not 4-byte aligned.  Refused at render time: a state that overlaps accum, depth, cost, raw, display, an AOV, light-group, deep-slice,
 *     matte, motion-vector or collision-AOV buffer (VPT_ERR_INVALID, naming the buffer); brick or cell mode (VPT_ERR_UNSUPPORTED). */
#define VPT_CRYPTO_MAX_ENTRIES 32
int  vpt_set_cryptomatte(vpt_context* ctx, uint32_t* d_state, unsigned capacity);

/* The Cryptomatte ranks of a state (width * rows pixels, capacity S, as vpt_set_cryptomatte), for an EXR writer.  Per pixel the non-empty
 * entries (count_j > 0) are sorted by count descending, then by id ascending (instance index; the sphere, 0xffffffff, last).  Rank r goes
 * to float4 plane r / 2 of d_out_f4 ([n_ranks / 2][pixel], 16-byte aligned), components 2 (r % 2) and 2 (r % 2) + 1, as (id float,
 * coverage): id float = d_id_of_instance[id] for id < n_instances, sphere_id for the sphere, 0.0f otherwise; coverage = count / n, the
 * float32 division rounded to nearest of the two converted counts.  Ranks past the last entry, and every rank where n == 0, are (0, 0),
 * Cryptomatte's empty rank.  d_out_overflow (may be NULL): overflow / n the same way (0 where n == 0).  The kernel never hashes: the id
 * table holds the floats of vpt_cryptomatte_hash.  Asynchronous on `stream`, deterministic, no scratch.
 *   Refused (VPT_ERR_INVALID): a NULL state or output, a NULL table with n_instances > 0, capacity outside 1..VPT_CRYPTO_MAX_ENTRIES,
 *   n_ranks odd or outside 2..32, width or rows 0, more than 2^31 pixels, a misaligned buffer, an output that overlaps the state, the
 *   table or the other output. */
int  vpt_cryptomatte_rank(vpt_context* ctx, unsigned width, unsigned rows, const uint32_t* d_state, unsigned capacity,
                          const float* d_id_of_instance, unsigned n_instances, float sphere_id, unsigned n_ranks, float* d_out_f4,
                          float* d_out_overflow, void* stream);

/* MurmurHash3_x86_32 of the len bytes at name (seed 0; NULL with len 0 is the empty name), as Cryptomatte hashes its names.  id_out (may
 * be NULL): the Cryptomatte float of the name, the hash with bit 23 flipped where its exponent (h >> 23) & 0xff is 0 or 255 (so no id is a
 * denormal, an infinity or a NaN), read as float bits.  The manifest entry of a name is "%08x" of those float bits. */
uint32_t vpt_cryptomatte_hash(const char* name, size_t len, float* id_out);

/* ---- sample-stream offset: a fresh Philox stream for every frame of a restarted accumulation ----------------------------------------
 * Pass p of a render call at Kernel_params.iteration = i draws the Philox stream the reference draws at iteration offset + i + p (32-bit
 * unsigned arithmetic, wrapping as iteration * 4096 does).  Everything else keyed by the iteration keeps the caller's i: the running-mean
 * arithmetic, the iteration < max_interactions gate and the "iteration 0 assigns" rule.  So a viewer that restarts every frame at
 * iteration 0 (the reference application does on every camera move) draws new samples each frame when it advances the offset, and a
 * one-pass frame at iteration 0 and offset k is the progressive render's pass k sample.  Offset 0, the default, is the reference stream.
 *   Activation.  The offset takes effect at the next render call whose Kernel_params.iteration is 0; a continued frame keeps its own.
 *   Works with every frame kind: vpt_render_pass(es), vpt_render_adaptive, render regions, both panoramas, camera motion, brick and cell
 *     mode, both integrators, partitioned contexts and both exchanges; vpt_set_motion_vectors and vpt_debug_motion_cameras follow it.
 *     Level (A) has none (its ABI is fixed). */
int  vpt_set_sample_offset(vpt_context* ctx, uint32_t offset);

/* ---- denoising: an edge-avoiding a-trous filter of a finished frame ------------------------------------------------------
 * vpt_denoise filters an HDR float3 frame (accum_buffer, or a full frame of the exchange block) guided by the noise of each pixel and by
 * the depth buffer -- the replacement for the reference application's Denoise button, which runs OIDN in place on accum_buffer.
 *
 *   Noise.  Y = 0.2126 r + 0.7152 g + 0.0722 b.  With d_rel_error (vpt_render_adaptive's error map; threshold 0 gives a fixed-count frame
 *     with one) the variance of the pixel's mean luminance is v = (err * max(Y, 1e-3))^2, which inverts err = sigma / max(mean, 1e-3) with
 *     the colour's Y for the mean; an err that is NaN or <= 0 gives v = 0, +inf stays +inf.  Without it, v is the population variance of
 *     Y over the 5x5 window (clipped at the frame edge).
 *   Levels.  Level i = 0 .. iterations-1 has step s = 2^i.  g = the 3x3 Gaussian (1/4, 1/2, 1/4)^2 of the current v (renormalised at the
 *     frame edge); a pixel with g == 0 keeps its colour and variance bit for bit.  Otherwise its taps q at s * (-2..2)^2 with the B3-spline
 *     weights h = (1/16, 1/4, 3/8, 1/4, 1/16)^2 (taps outside the frame drop out) weigh
 *         w = exp(-|Y_p - Y_q| / (sigma_luminance sqrt(g) + 1e-10) - |z_p - z_q| / (sigma_depth max(|z_p|, |z_q|) + 1e-6))
 *     (no depth term when d_depth is NULL; the centre tap weighs 1), and c' = sum(h w c_q) / sum(h w), v' = sum((h w)^2 v_q) / sum(h w)^2.
 *   Non-finite pixels.  A pixel whose colour (or luminance) is not finite is copied unchanged and has weight 0 as a neighbour.
 *   Float32.  The filter computes in float32 with denormals flushed to zero: a v below 2^-126 is 0 (a pixel whose 3x3 window of v is all
 *     below it is copied), an h w below 2^-126 drops out and one whose square is below it adds 0 to v' (against an infinite v_q that makes
 *     v' NaN, and a pixel whose g then sees the NaN is copied); |Y_p - Y_q| is formed in float32, so luminances near FLT_MAX of opposite
 *     sign are inf apart and drop each other as taps, even where g is infinite.
 *   Outputs.  The last level writes d_out_f3 and, if d_out_display is given, the display word of each pixel exactly as k_resolve packs it
 *     (ACES, exposure_scale, gamma 2.2, BGRA).  A zero error map therefore reproduces the colour and k_resolve's display words bit for bit.
 *   Contract.  The work is enqueued asynchronously on `stream` (a cudaStream_t), with no synchronisation.  All buffers are full row-major
 *     [H][W] frames in device memory; on a partitioned context pass the full frame of the exchange block (vpt_comm_p2p_frame,
 *     vpt_comm_p2p_adaptive_frame), not the rank-local Kernel_params buffers.  Deterministic: no atomics, the same inputs give the same
 *     bits.  d_out_f3 may EQUAL d_color_f3 (in place, as the reference's Denoise button); any partial overlap of an output with an input,
 *     and any overlap of the two outputs, is refused.  The scratch planes (48 B per pixel, allocated on first use) belong to the context,
 *     so calls on one context must be ordered on one stream.  The filter touches no render state: accumulating further passes onto an
 *     accumulator denoised in place continues from the filtered mean.
 *   Refused (VPT_ERR_INVALID): a NULL ctx, colour or output; width or height 0 or above 65535; iterations outside 1..10; a sigma that is
 *     not finite and > 0; the overlaps above.  opt == NULL takes the defaults. */
typedef struct vpt_denoise_options {
    unsigned iterations;       /* a-trous levels, step 2^i for level i; 1..10 (default 5: steps 1..16) */
    float    sigma_luminance;  /* luminance edge-stopping, in units of the pixel's noise sigma; > 0 (default 4) */
    float    sigma_depth;      /* relative depth edge-stopping; > 0 (default 0.2) */
} vpt_denoise_options;
void vpt_denoise_options_defaults(vpt_denoise_options* opt);
int  vpt_denoise(vpt_context* ctx, unsigned width, unsigned height,
                 const float* d_color_f3,         /* [H][W] float3 HDR, e.g. accum_buffer or vpt_comm_p2p_frame's accumulators */
                 const float* d_depth,            /* [H][W] float, may be NULL: no depth term */
                 const float* d_rel_error,        /* [H][W] float, vpt_render_adaptive's error map, may be NULL: spatial estimate */
                 const vpt_denoise_options* opt,  /* NULL = defaults */
                 float exposure_scale,            /* only read when d_out_display != NULL */
                 float* d_out_f3,                 /* [H][W] float3; may EQUAL d_color_f3 */
                 unsigned* d_out_display,         /* [H][W] BGRA words as k_resolve writes them, may be NULL */
                 void* stream);

/* vpt_denoise_layers denoises the beauty exactly as vpt_denoise does and filters further layers (the compositing AOVs, light groups, deep
 * slices, mattes, or any other full-frame planes) with the beauty's weights, so additive identities between the layers and the beauty
 * (volume + (1 - alpha) k, the sum of the light groups, the sum of the deep slices) still hold after denoising, up to rounding.
 *   Beauty.  d_out_f3 and d_out_display are vpt_denoise's outputs for the same arguments, bit for bit; n_layers == 0 is vpt_denoise.
 *   Layers.  Each channel x of each plane of each layer is filtered at every level with the beauty's weights of that level:
 *     x' = sum(h w x_q) / sum(h w), the same taps, the same h w, in the same order, with the same copy rule.  A pixel the beauty copies
 *     (non-finite colour or luminance, or g == 0) keeps its layer values bit for bit at that level; a tap the beauty drops is dropped for
 *     every layer.  A layer carries no variance of its own and does not guide.  A non-finite layer value in a tap that is used spreads to
 *     the pixels that use it, like any other value.  A layer equal to the beauty's colour comes out equal to d_out_f3, bit for bit.
 *   Contract.  As vpt_denoise's, and: a layer's dst may EQUAL its src (in place); any partial overlap of a dst with its own src, and any
 *     overlap of a dst with another layer's src or dst, d_color_f3, d_out_f3, d_out_display, d_depth or d_rel_error, is refused.  A
 *     layer's src may be any of the beauty's inputs (d_color_f3 passed as a layer gives the beauty's output).  The layer scratch (two sets
 *     of 16 B per plane and pixel, 32 B * sum(count) per pixel, on top of vpt_denoise's 48 B) belongs to the context, is allocated on
 *     first use and only grows.
 *   Refused (VPT_ERR_INVALID, nothing enqueued): everything vpt_denoise refuses; n_layers > 0 with a NULL layers; a NULL src or dst;
 *     channels outside 1..4; count 0; the overlaps above. */
typedef struct vpt_denoise_layer {
    const float* src;       /* [count][H][W][channels] float, full row-major frames in device memory */
    float*       dst;       /* same shape; may EQUAL src (in place), no other overlap */
    unsigned     channels;  /* 1..4 */
    unsigned     count;     /* >= 1 planes of H*W pixels (K for deep slices / mattes, 1 otherwise) */
} vpt_denoise_layer;
int  vpt_denoise_layers(vpt_context* ctx, unsigned width, unsigned height,
                        const float* d_color_f3, const float* d_depth, const float* d_rel_error,
                        const vpt_denoise_options* opt, float exposure_scale,
                        float* d_out_f3, unsigned* d_out_display,
                        const vpt_denoise_layer* layers, unsigned n_layers, void* stream);

/* ---- temporal accumulation: a moving camera's frames averaged through the motion vectors ------------------------------------------
 * vpt_temporal blends the current frame C into the previous output H, carried to each pixel along the pixel's motion towards the
 * previous camera, so a viewer keeps converging while the camera moves.  For perspective frames (panoramas have no motion vectors).
 * Per pixel (x, y) of W x H (tests/temporal_ref.py restates it):
 *   1. Motion.  M = (c vx, c vy, c), the premultiplied vectors of vpt_set_motion_vectors rendered with target = `previous` (B); A is
 *      `current`, the frame camera (the shutter-open pose of a motion frame).  When M.z < 1 the uncovered share moves like the environment,
 *      a direction at infinity: d = e_A + s h_A + t v_A with s = (x + 1/2) / W, t = (y + 1/2) / H, e = llc - origin, h = horizontal,
 *      v = vertical (d = fma(t, v, fma(s, h, e)) per component), and v_env = pi_B(d) - pi_A(d), pi the film projection of
 *      vpt_set_motion_vectors with d in place of P - origin.  The pixel's motion is v = M.xy + (1 - M.z) v_env (per component
 *      fma(1 - M.z, v_env, M.xy)); with M.z >= 1 (or NaN) v = M.xy.  So B == A gives v = +0 exactly, as the vectors do.  If the
 *      projection of d fails for A or B (k <= 0 or a result not finite) while M.z < 1, the pixel has no history.
 *   2. History.  q = (x + 1/2 + v.x, y + 1/2 + v.y).  No history if v is not finite or q lies outside [0, W] x [0, H].  Otherwise the
 *      bilinear taps of H around q - 1/2, in the order (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1): taps outside the frame, of
 *      weight 0 or with a non-finite colour are dropped, the rest renormalised (sum(w h) / sum(w)); none left: no history.  L_hist is the
 *      least L among the taps used.  An integer-aligned q reads its one texel bit for bit.
 *   3. Clip.  mu and sigma are the per-channel mean and population standard deviation of C over the 3x3 window (clipped at the frame
 *      edge, non-finite neighbours dropped); h' = min(max(h, mu - clip_sigma sigma), mu + clip_sigma sigma).  clip_sigma = +inf skips it.
 *   4. Blend.  L_new = min(L_hist + 1, max_history) and out = h' + (C - h') / (float)L_new, accum's running-mean expression of k_resolve
 *      (the reference's render_kernel.cu:2284).  With no history, no history buffers, or a non-finite C: out = C bit for bit, L_new = 1.
 *      d_out_display, if given, gets the display word of out exactly as k_resolve packs it (ACES, exposure_scale, gamma 2.2, BGRA).
 *   Float32.  The footprint is float32: q = (float)x + 1/2 + v rounded, so a q that rounds onto 0, W or H keeps its history; px = q - 1/2
 *     and x0 = floorf(px) (q = 0 gives x0 = -1, fx = 1/2); a tap's weight is (1 - fx)(1 - fy) etc. each rounded, and an integer px gives
 *     weight-0 taps, which are dropped.  Lengths: the first used tap's L, then fminf with each further one, so a NaN length is ignored
 *     while another used tap has a number, and L_hist is NaN only when every used tap's is; L_new = fminf(L_hist + 1, max_history) in
 *     float32, so a NaN or +inf L_hist gives max_history, -inf gives -inf (out = h'), L_hist = -1 gives L_new = 0 (out = +-inf, or NaN
 *     where C = h'), fractional and negative lengths divide as written and L_hist + 1 rounds (2^24 + 1 is 2^24).  The library's own
 *     d_out_len is always finite and >= 1; these cases only come from caller buffers.  C - h' is formed in float32: +-inf when C and h'
 *     lie near +-FLT_MAX with opposite signs.  The weighted history sum and its division by sum(w) are float32 and can round past
 *     FLT_MAX.  The clip's window sum, mean and deviation are float32: a window sum that overflows gives mu = +-inf and mu - r NaN, which
 *     fmaxf / fminf drop, so the clip does nothing on that channel; a deviation that overflows gives r = inf and no clip either.  Denormals
 *     are flushed to zero in arithmetic (--use_fast_math): a denormal C, H, layer value or clip_sigma counts as 0 (a denormal clip_sigma
 *     clamps h to mu), and a denormal result is stored as 0; a pixel without history keeps its input bits, denormals included.
 *   Guarantee.  A still camera, clip_sigma = +inf, max_history >= F and F one-pass frames rendered at iteration 0 with sample offsets
 *     0 .. F-1 (vpt_set_sample_offset), each filtered against the previous call's outputs: out is accum of one F-pass progressive render
 *     bit for bit, and so is the display word -- unless a sample of those frames was replaced by the reference's NaN / Inf guard, which at
 *     iteration 0 keeps the buffer's previous content instead of the running mean.
 *   Contract.  Enqueued asynchronously on `stream`, no synchronisation, no scratch; touches no render state.  All buffers are full
 *     row-major [H][W] frames in device memory; on a partitioned context pass the exchange block's full frames (vpt_comm_p2p_frame, the
 *     VPT_LAYER_MOTION plane).  Deterministic: no atomics.  The fetch and the clip read neighbours, so the call cannot work in place: the
 *     caller ping-pongs two history buffers.
 *   Refused (VPT_ERR_INVALID, nothing enqueued): a NULL ctx, colour, vectors, camera, d_out_f3 or d_out_len; width or height 0 or above
 *     65535; exactly one of d_history_f3 and d_history_len NULL; max_history outside 1..2^24; clip_sigma NaN or <= 0; a non-finite
 *     component of origin, lower_left_corner, horizontal or vertical of either camera; any overlap of an output with an input or with
 *     another output.  opt == NULL takes the defaults. */
typedef struct vpt_temporal_options {
    unsigned max_history;  /* cap on the history length L, 1 .. 2^24 (default 16) */
    float    clip_sigma;   /* > 0: clip width in standard deviations of the 3x3 window; +INFINITY: no clip (default +INFINITY) */
} vpt_temporal_options;
void vpt_temporal_options_defaults(vpt_temporal_options* opt);
int  vpt_temporal(vpt_context* ctx, unsigned width, unsigned height,
                  const float* d_color_f3,        /* C: [H][W] float3, this frame (e.g. accum_buffer) */
                  const float* d_vectors_f3,      /* M: [H][W] float3, vpt_set_motion_vectors' buffer rendered with target = previous */
                  const vpt_camera* current,      /* A: the frame camera */
                  const vpt_camera* previous,     /* B: the camera of the history */
                  const float* d_history_f3,      /* H: [H][W] float3, the previous call's d_out_f3; NULL with d_history_len: no history */
                  const float* d_history_len,     /* L: [H][W] float, the previous call's d_out_len */
                  const vpt_temporal_options* opt,  /* NULL = defaults */
                  float exposure_scale,           /* only read when d_out_display != NULL */
                  float* d_out_f3,                /* [H][W] float3 */
                  float* d_out_len,               /* [H][W] float, the history length of each pixel */
                  unsigned* d_out_display,        /* [H][W] BGRA words as k_resolve writes them, may be NULL */
                  void* stream);

/* vpt_temporal_layers accumulates the beauty exactly as vpt_temporal does and blends further layers (the compositing AOVs, light groups,
 * collision AOVs, deep slices, mattes, or any other full-frame planes) with the beauty's taps and history length, so additive identities
 * between the layers and the beauty (volume + (1 - alpha) k, the sum of the light groups, the sum of the deep slices) still hold in the
 * filtered frames, up to rounding (DESIGN.md section 8r; tests/temporal_layers_ref.py restates it).
 *   Beauty.  d_out_f3, d_out_len and d_out_display are vpt_temporal's outputs for the same arguments, bit for bit; n_layers == 0 is
 *     vpt_temporal.
 *   Layers.  Each pixel uses the beauty's motion (step 1) and taps (step 2): the same taps in the same order with the same weights, and a
 *     tap the beauty drops is dropped for every layer -- also one dropped for a non-finite beauty history colour where the layer's value
 *     is finite.  Each channel x of each plane becomes
 *         h_x = sum(w H_x) / sum(w)   (fmaf in tap order, divided as the beauty divides)
 *         out_x = h_x + (x - h_x) / (float)L_new   (the beauty's L_new, accum's expression with k_resolve's flags).
 *     Where the beauty has no history (no history buffers, v not finite, q outside the frame, no tap left, a non-finite C) out_x = x bit
 *     for bit.  The clip (step 3) belongs to the beauty: layers are blended unclipped, so with a finite clip_sigma the identities hold
 *     only where the clip did not move the beauty's history (the default is no clip).  A layer carries no history length and guides
 *     nothing; a non-finite layer value in a tap that is used spreads to the pixel.  A layer whose src is d_color_f3 and whose history
 *     is d_history_f3 comes out equal to d_out_f3 bit for bit when there is no clip, and so does each of its channels passed as a
 *     1-channel layer.
 *   Guarantee.  vpt_temporal's still-camera case (B == A, no clip, max_history >= F, F one-pass frames at sample offsets 0 .. F-1): every
 *     layer k_resolve keeps with accum's running-mean rule -- alpha, volume, the light groups, the deep and matte bins, position, normal
 *     and albedo -- equals that layer of one F-pass progressive render bit for bit, with the beauty's exceptions (a sample replaced by the
 *     NaN / Inf guard) and the max_interactions gate.
 *   Contract.  As vpt_temporal's: asynchronous on `stream`, deterministic, no scratch, one launch.  The fetch reads neighbours, so
 *     nothing works in place: the caller ping-pongs each layer's two buffers as it does the beauty's.
 *   Refused (VPT_ERR_INVALID, nothing enqueued): everything vpt_temporal refuses; n_layers > 0 with a NULL layers; n_layers above
 *     VPT_TEMPORAL_MAX_LAYERS; a NULL src or dst; a layer history that is NULL while d_history_f3 is set, or set while it is NULL;
 *     channels outside 1..4; count 0; any byte overlap of a dst with any input (the beauty's or a layer's), with d_out_f3, d_out_len or
 *     d_out_display, or with another dst; any overlap of the beauty's outputs with a layer's src or history. */
#define VPT_TEMPORAL_MAX_LAYERS 16
typedef struct vpt_temporal_layer {
    const float* src;       /* [count][H][W][channels] float, this frame's layer (e.g. the alpha AOV), full row-major frames */
    const float* history;   /* same shape: the previous call's dst; NULL exactly when d_history_f3 is NULL */
    float*       dst;       /* same shape; overlaps nothing else */
    unsigned     channels;  /* 1..4 */
    unsigned     count;     /* >= 1 planes of H*W pixels (K for deep slices / mattes, 1 otherwise) */
} vpt_temporal_layer;
int  vpt_temporal_layers(vpt_context* ctx, unsigned width, unsigned height,
                         const float* d_color_f3, const float* d_vectors_f3, const vpt_camera* current, const vpt_camera* previous,
                         const float* d_history_f3, const float* d_history_len, const vpt_temporal_options* opt, float exposure_scale,
                         float* d_out_f3, float* d_out_len, unsigned* d_out_display,
                         const vpt_temporal_layer* layers, unsigned n_layers, void* stream);

/* The flattened scene tables are cached per (volumes pointer, octree root pointer, build generation of a vpt_octree_build
 * octree) and refreshed whenever a call arrives with Kernel_params.iteration == 0 (the reference application resets the
 * iteration on every scene edit, main.cpp:1667-1780).  Call this only if the GPU_VDB[] array or a foreign octree was
 * rewritten in place WITHOUT restarting the accumulation. */
int  vpt_invalidate_scene(vpt_context* ctx);

/* Counters of the last vpt_render_pass(es) call: kernels launched, and (after the stream has been
 * synchronised by the caller) rays pushed into the hit queue by the final chunk. */
int  vpt_get_stats(vpt_context* ctx, unsigned long long* kernel_launches_total, unsigned* last_queue_count);

/* Instrumentation.  Option "count_stats" = 1 makes the trace kernel accumulate out[0] volume lookups,
 * out[1] lane-steps, out[2] warp step-loop iterations, out[3] rays serviced, out[4] warp service rounds, out[5] rays
 * fetched from the queue, out[6] bricks staged by TMA (brick mode) (SIMT efficiency of the step loop = out[1] / (32 * out[2])), and
 * out[7] the rays per lane of the last render call's trace kernel (2 or 3; 0 for k_trace_brick or before any render call), which
 * unlike the warp totals out[2] and out[4] does not depend on how the warps were scheduled.  Option "profile" = 1 brackets every kernel with
 * CUDA events: ms/n[0..3] = generate, trace, resolve, blue-noise advance (in adaptive frames the convergence tests count as resolve;
 * the per-call miss cull of option "miss_cull" counts as generate).
 * Both calls synchronise the device. */
int  vpt_get_counters(vpt_context* ctx, unsigned long long out[8], int reset);
/* Hop statistics of option "count_stats" (a reset of vpt_get_counters clears them too): out[0..2] = hops over empty octree nodes of
 * the lean k_trace's delta / ratio / emission walks (the kernels that take the "empty ahead" shortcut; the lean kernel runs no emission
 * walk, so out[2] stays 0), out[3] = k_trace walks ended by "empty ahead" (option "empty_ahead"), out[4..6] = rays that
 * entered k_generate's octree pre-step / its hops / those ended at once by "empty ahead"; out[7] = 0.  Synchronises the device. */
int  vpt_get_hop_counters(vpt_context* ctx, unsigned long long out[8], int reset);
/* The "empty ahead" table of the last render call (option "empty_ahead"; built once per call from the scene's octree): out[8 * i + c] is
 * the entry of child c of internal node i (0..72), bit o set when no populated leaf lies in the orthant of the child's block for direction
 * octant o (bit 0 x < 0, bit 1 y < 0, bit 2 z < 0); the last 8 bytes are 0.  Synchronises the device. */
#define VPT_EMPTY_AHEAD_BYTES 592
int  vpt_debug_empty_ahead(vpt_context* ctx, unsigned char out[VPT_EMPTY_AHEAD_BYTES]);
int  vpt_get_kernel_times(vpt_context* ctx, float ms[4], int n[4]);

/* ---- host-side scene helpers (what the reference does in main.cpp / gpu_vdb.cpp / bvh_builder.cpp) -- */

/* Dense grid -> 3-D texture, as GPU_VDB::loadVDB builds them (gpu_vdb.cpp:215-248: cudaArray, normalised
 * coordinates, linear filter, clamp).  channels = 1 (float) or 4 (float4).  Returns the texture object and
 * an opaque array handle for vpt_texture_destroy. */
int  vpt_texture_create_3d(const float* host_data, int channels, int dim_x, int dim_y, int dim_z,
                           vpt_tex_t* tex_out, void** array_out);
/* Same texture from a dense grid that already lives in device memory (x fastest), e.g. a procedural grid of several GiB. */
int  vpt_texture_create_3d_from_device(const float* d_data, int channels, int dim_x, int dim_y, int dim_z,
                                       vpt_tex_t* tex_out, void** array_out);
/* Procedural density grid: the reference's fill_volume_buffer (texture_kernels.cu:76-128) for noise_type 0 =
 * cudaNoise::perlinNoise(pos, scale, seed) at voxel (x, y, z), x fastest -- with ZERO sub-voxel jitter (the reference draws
 * its jitter from an uninitialised generator state, quirk Q14).  d_buffer: dx*dy*dz floats in device memory.  The matching
 * VDB_INFO is what GPU_PROC_VOL::create_volume fills (gpu_vdb.cpp:529-541): bmin = box min, bmax = bmin + dim, voxelsize = res,
 * max_density 1, min_density 0, xform = scale(res). */
int  vpt_procedural_fill(float* d_buffer, int dim_x, int dim_y, int dim_z, int noise_type, float scale, int seed, void* stream);

/* ---- brick mode: brick pool + TMA-staged software sampler (the look-up without the texture unit) ---------------------
 * vpt_bricks_create re-lays a dense device grid as 4x4x4-cell bricks stored with their +1 apron (5x5x5 texels + brick max /
 * min: 512 contiguous bytes each, edge texels clamped like the reference's clamp-addressed texture).  vpt_set_brick_volume
 * makes the context trace volume 0 from that pool: k_trace_brick stages the brick under each ray into shared memory with
 * one cp.async.bulk (TMA) and filters it in software with the texture unit's own arithmetic, measured on the device:
 * coordinate truncated to 21 fractional bits, eight integer corner weights that sum to 256 (split z -> x -> y), correctly
 * rounded sum.  99.6 % of the fetches are bit-identical to tex3D, the rest one ulp off; rendered frames meet the same
 * per-pixel tolerance as the texture path (tests/test_bricks_gpu.py).  Supported: a vpt_octree_build scene of one volume
 * without colour grid, direct integrator, no emission, no point lights; anything else is refused with VPT_ERR_UNSUPPORTED.
 * dim_* must be the dimensions of volume 0's density grid (vdb_info.dim of the scene's octree build): a render whose scene differs
 * fails with VPT_ERR_INVALID, naming both, and launches nothing.  d_pool = 0 returns the context to the texture path. */
int  vpt_bricks_create(const float* d_dense, int dim_x, int dim_y, int dim_z, vpt_devptr_t* d_pool_out, unsigned long long* bytes_out);
int  vpt_bricks_read(vpt_devptr_t d_pool, unsigned long long first_brick, unsigned long long n_bricks, float* h_out);   /* 128 floats per brick */
/* Diagnostic: the software filter under three weight rules (m = 0 the texture unit's integer corner weights -- the production rule --,
 * 1 per-axis weights truncated to 1/256, 2 per-axis full fp32 fractions), reading the bricks from global memory, against tex3D on n pseudo-random points: out12[m*4 + 0..3] = max |d|, sum |d|,
 * number of bit-identical results, n. */
int  vpt_debug_sampler_compare(vpt_tex_t tex, vpt_devptr_t d_pool, int dim_x, int dim_y, int dim_z, int n_points, unsigned seed, double out12[12]);
/* Diagnostic: the production brick and cell samplers (the look-ups of k_trace_brick and of the lean k_trace in cell mode) at n chosen
 * normalised points, host arrays uvw[n][3] in [0, 1] (anything else is refused) -> out2[n][2] = { brick value, cell value }, on the default
 * stream.  d_pool (vpt_bricks_create) or d_cells (vpt_cells_create) may be 0, its value is then 0; dim_* are the grid's dimensions.  Bricks
 * are staged through a per-thread shared-memory slot exactly as in the trace, each thread taking 32 consecutive points. */
int  vpt_debug_software_sample(vpt_devptr_t d_pool, vpt_devptr_t d_cells, int dim_x, int dim_y, int dim_z, const float* uvw, int n, float* out2);
int  vpt_bricks_destroy(vpt_devptr_t d_pool);
int  vpt_set_brick_volume(vpt_context* ctx, vpt_devptr_t d_pool, int dim_x, int dim_y, int dim_z);

/* ---- cell mode: one DRAM sector per look-up for grids no cache can hold -------------------------------------------
 * vpt_cells_create re-lays a dense device grid as a CELL TABLE: for every texel cell (i, j, k) the eight corner texels a
 * trilinear look-up in that cell blends (clamped at the upper faces), 32 contiguous, 32-byte aligned bytes, x fastest.  Eight
 * times the memory of the grid (1024^3: 32 GiB -- sized for 180 GB of HBM), and ONE sector per look-up where the 2x2x2
 * footprint costs four or five in the tiled array of the texture path.  vpt_set_cell_volume makes the trace kernel read volume
 * 0 from it (lean instantiation, 2 rays per lane, the texture unit's arithmetic in software as in brick mode: same per-pixel
 * tolerance, tests/test_bricks_gpu.py); same scene restrictions as brick mode, and the same dimension rule: dim_* must be those of
 * volume 0's density grid or the render fails with VPT_ERR_INVALID and launches nothing; d_cells = 0 returns to the texture path. */
int  vpt_cells_create(const float* d_dense, int dim_x, int dim_y, int dim_z, vpt_devptr_t* d_cells_out, unsigned long long* bytes_out);
int  vpt_cells_read(vpt_devptr_t d_cells, unsigned long long first_cell, unsigned long long n_cells, float* h_out);       /* 8 floats per cell */
int  vpt_cells_destroy(vpt_devptr_t d_cells);
int  vpt_set_cell_volume(vpt_context* ctx, vpt_devptr_t d_cells, int dim_x, int dim_y, int dim_z);

/* Equirectangular environment map float4 (main.cpp:945-978: wrap / clamp, linear, normalised). */
int  vpt_texture_create_env(const float* host_rgba, unsigned width, unsigned height, vpt_tex_t* tex_out, void** array_out);
/* The four sky-sampling tables the volumetric path integrator reads when environment_type == 0 (reference create_cdf,
 * main.cpp:647-867): from a res x res table of the sky's luminous power over (azimuth = x, elevation = y) builds the
 * row-conditional cdf, the marginal function and its cdf, and wraps all four as point-sampled unnormalised float
 * textures (2-D, 2-D, 1-D, 1-D).  tex_out / arrays_out order: env_func_tex, env_cdf_tex, env_marginal_func_tex,
 * env_marginal_cdf_tex; *marginal_int_out is Kernel_params.env_marginal_int; env_sample_tex_res = res.  The arithmetic is
 * vpt_env_tables_compute's. */
int  vpt_env_tables_create(const float* func, unsigned res, vpt_tex_t tex_out[4], void* arrays_out[4], float* marginal_int_out);
/* The host arithmetic of create_cdf (main.cpp:681-757) on caller-provided arrays (cdf: res*res, marginal_func / marginal_cdf:
 * res), literally: row y > 0 of the conditional cdf starts from func[y-1][res-1] / res (the reference's `*(func_p - 1)` at x == 0
 * is the previous row's last element), the uniform fallback is selected by marginal_func[0] == 0, the last cdf entry of each
 * row is 1.  The only two reads the reference makes OUTSIDE its arrays (func[-1], marginal_cdf[-1]; quirk Q20) are taken as 0.
 * Pure host code, no device needed. */
int  vpt_env_tables_compute(const float* func, unsigned res, float* cdf, float* marginal_func, float* marginal_cdf, float* marginal_int_out);
/* The table create_cdf feeds into the above: luminous power of the reference's HOST-side analytic sky (single-scattering
 * Rayleigh + Mie march, 16 x 8 samples, main.cpp:242-301) over res x res directions, func[y*res + x] =
 * |sky(dir(az = x/(res-1)*2pi, el = y/(res-1)*pi)) * sky_color| (main.cpp:683-693; the reference uses res = 180 and
 * Kernel_params.azimuth / elevation / sky_color).  Pure host code, no device needed. */
int  vpt_env_sky_tabulate(float azimuth_deg, float elevation_deg, const float sky_color[3], unsigned res, float* func_out);
int  vpt_texture_destroy(vpt_tex_t tex, void* array);

/* Minimal OpenVDB (file format 224) reader: densify grid `grid_name` over its active-voxel bounding box
 * (gpu_vdb.cpp:133-212).  On success *values_out is malloc'd (x fastest, `channels` floats per voxel; free
 * with vpt_free) and info[] receives: dim[3], bbox_min[3], bbox_max[3], channels, leaf_count,
 * active_voxel_count (lo, hi 32 bits)  -> 13 ints; xform16 receives the reference's mat4 memory image
 * (gpu_vdb.cpp:81-92, convert_to_mat4); stats[] = { max_value, min_density per Q10, voxel_size, background }.
 * Returns 1 if the file has no such grid. */
int  vpt_vdb_load(const char* path, const char* grid_name, float** values_out, int info[13], float xform16[16], float stats[4]);
int  vpt_hdr_load(const char* path, float** rgba_out, unsigned* width, unsigned* height);   /* hdr_loader.h:249-278 */
int  vpt_bmp_load_rbg(const char* path, float** xyz_out, int* width, int* height);          /* fileIO.cpp:460-495 (Q16) */
int  vpt_exr_load_rgb(const char* path, float** rgb_out, int* width, int* height);          /* fileIO.cpp:356-390 */
void vpt_free(void* p);

/* Scene / light instance file (.ins) reader -- the text format of read_instance_file, main.cpp:980-1040, SURVEY 8(f) N4:
 *     "light" \n N \n { px py pz r g b power } x N                                  (point lights)
 *     N_vdbs \n { vdb_path \n N_inst \n { px py pz qx qy qz qw scale } x N_inst } x N_vdbs   (instanced volumes)
 * One record per line, whitespace separated, paths taken verbatim (the reference resolves them against its CWD).
 * *out is one malloc'd block (free with vpt_free): the header below, then n_files vpt_ins_file_entry, then n_records records
 * of 8 doubles each (volumes: px py pz qx qy qz qw scale; lights: px py pz r g b power 0).  Unlike the reference, a line
 * with too few numbers is an error (VPT_ERR_IO) instead of leaving the fields uninitialised.  The instance transform itself
 * (mat4 algebra of main.cpp:1059-1099) is applied by the caller; see volumetric-path-tracer_b200/scene.py:instance_xform. */
typedef struct vpt_ins_header { int32_t kind; int32_t n_files; int32_t n_records; int32_t reserved; } vpt_ins_header;   /* kind: 0 volumes, 1 lights */
typedef struct vpt_ins_file_entry { char path[1024]; int32_t first_record; int32_t n_instances; } vpt_ins_file_entry;
int  vpt_ins_load(const char* path, vpt_ins_header** out);

/* Instance acceleration build -- replaces BVH_Builder::build_bvh (bvh_builder.cpp:46-105).
 *
 * vpt_octree_build: depth-3 octree over the instance bounds (host root set-up bvh_builder.cpp:61-78, node semantics of
 * bvh_kernels.cu:204-246: child boxes by halving, inclusive overlap test, ascending instance order), built in parallel
 * with no device heap.  Any n >= 1:
 *   n <= VPT_OCT_MAX_VOLUMES  *d_root_out is node 0 of a contiguous 585-node tree in the reference's own OCTNode layout
 *                             (pointer-linked; the reference kernel can consume it as well);
 *   n >  VPT_OCT_MAX_VOLUMES  the reference layout cannot hold the lists (vol_indices[600]; the reference itself overflows
 *                             the node there, quirk Q11): *d_root_out points to the root record only (children null).
 * In both cases the octree is ALSO kept in the flat form the render kernels read (73 internal nodes + 512 leaf lists in
 * CSR form, no per-leaf limit) and registered under the returned root pointer: vpt_render_pass(es) recognises the pointer
 * in params[VPT_ARG_OCTREE] and uses those tables directly.  h_volumes: host array of n GPU_VDB; the GPU_VDB[] device
 * array passed at render time must describe the same instances.  Free with vpt_octree_destroy. */
int  vpt_octree_build(const vpt_gpu_vdb* h_volumes, int n, vpt_devptr_t* d_root_out);
int  vpt_octree_destroy(vpt_devptr_t d_root);
/* What vpt_octree_build registered for this root: instance count, whether reference-layout nodes exist (n <= 600), total
 * and largest leaf-list length.  Any output pointer may be NULL. */
int  vpt_octree_info(vpt_devptr_t d_root, int* n_instances, int* reference_layout, long long* total_leaf_entries, int* max_leaf_entries);
/* Copy any pointer-linked octree (this builder's n <= 600 tree or the reference's device-heap one) into 585 host nodes in
 * the canonical numbering 0 | 1+c1 | 9+c1*8+c2 | 73+c1*64+c2*8+c3; exists[j] = 0 for nodes never allocated. */
int  vpt_octree_read(vpt_devptr_t d_root, vpt_octnode* h_nodes585, int* h_exists585);
/* Flat leaf lists of a registered octree: leaf_offset_count[2*l] / [2*l+1] = offset / length of leaf l = c1*64+c2*8+c3 in
 * `indices` (ascending instance ids; capacity in ints, indices may be NULL to fetch the table only). */
int  vpt_octree_read_flat(vpt_devptr_t d_root, unsigned leaf_offset_count[1024], int* indices, long long capacity);

/* LBVH over the instance AABBs in the reference's BVHNode layout (BuildBVH, bvh_kernels.cu:460-580: Morton codes of the
 * centroids in the scene box, stable sort, Karras radix tree with the (code, id) tie-break, bottom-up refit).
 * *d_nodes_out: n-1 internal nodes (node 0 is the root; one zeroed node when n == 1), *d_leaves_out: n leaves in sorted
 * order; child / parent fields are device pointers into the two arrays, exactly what the reference passes as `root_node`.
 * scene_bounds6 (may be NULL): union of the instance boxes.  h_sorted_codes / h_sorted_ids (host, n entries, may be NULL):
 * the sorted 30-bit Morton codes and instance ids.  Unlike the reference the arrays are zero-initialised and n == 1 is
 * handled (quirk Q18).  The live integrators of the reference never traverse this tree (SURVEY section 0); it is built for
 * callers that pass it on. */
int  vpt_bvh_build(const vpt_gpu_vdb* h_volumes, int n, vpt_devptr_t* d_nodes_out, vpt_devptr_t* d_leaves_out, float scene_bounds6[6],
                   unsigned long long* h_sorted_codes, int* h_sorted_ids);
/* Copy a BVH in that layout (either builder's) to the host, pointer fields rewritten as indices: internal node i -> i,
 * leaf i -> (n-1)+i, anything else -> (uint64)-1. */
int  vpt_bvh_read(vpt_devptr_t d_nodes, vpt_devptr_t d_leaves, int n, vpt_bvhnode* h_nodes, vpt_bvhnode* h_leaves);
int  vpt_bvh_destroy(vpt_devptr_t d_nodes, vpt_devptr_t d_leaves);
/* AABB of one instance (GPU_VDB::Bounds, gpu_vdb.h:131-146): out6 = pmin, pmax. */
void vpt_volume_bounds(const vpt_gpu_vdb* h_volume, float out6[6]);

/* ---- Bruneton sky tables (replaces atmosphere::init, source/atmosphere/atmosphere.cpp:1177-1291 + atmosphere_kernels.cu) ------------
 * Builds the Earth model of the reference (its spectra, density profiles, radii), reduces it to the AtmosphereParameters block the
 * render path takes by value, precomputes the transmittance / irradiance / scattering / single-Mie tables on the device (own sm_90a
 * kernels, four scattering orders) and wraps them as the four look-up textures with the reference's descriptors.  *out receives the
 * complete block (scalars + texture objects; scratch buffer pointers null); free with vpt_atmosphere_destroy(handle).
 * The tables reproduce the reference's build of the model, including the places where it departs from Bruneton's paper (later
 * orders overwrite instead of accumulate because the host passes a float4 where its kernels read an int: quirk Q17; mie_extinction
 * taken from the Mie scattering spectrum), except that a table look-up whose linear index leaves the table is clamped to it where
 * the reference reads outside its buffers (atmosphere_kernels.cu:161-171, 375-395): before the delta scattering-density buffer
 * for rays just below the horizon near the ground, one past the transmittance table's end (vpt_bruneton.cu). */
typedef struct vpt_atmosphere_options {
    int   use_constant_solar_spectrum;   /* main.cpp:1433 default 1 */
    int   use_ozone;                     /* default 1 */
    int   luminance_mode;                /* 0 NONE (default), 1 APPROXIMATE, 2 PRECOMPUTED (15 wavelengths) */
    int   do_white_balance;              /* default 1 */
    float exposure;                      /* default 1 */
    int   num_scattering_orders;         /* default 4 */
} vpt_atmosphere_options;
void vpt_atmosphere_options_defaults(vpt_atmosphere_options* opt);
int  vpt_atmosphere_precompute(const vpt_atmosphere_options* opt, vpt_atmosphere* out, void** handle_out);
int  vpt_atmosphere_destroy(void* handle);
/* Texel centres of a float4 texture (w x h, or w x h x d when d > 0) into host memory, 4 floats per texel, x fastest. */
int  vpt_texture_read_f4(vpt_tex_t tex, int w, int h, int d, float* host_out);
/* Diagnostic: tex3D<float> at n arbitrary normalised coordinates (uvw: 3 floats per point). */
int  vpt_debug_texture_sample(vpt_tex_t tex, const float* uvw, int n, float* out);
/* Diagnostic: ONE launch of one of the six precompute kernels -- the launch vpt_atmosphere_precompute makes for that stage -- on
 * caller-owned device tables, then a device synchronisation.  tables[9]: float4 device buffers in the order of the reference's
 * AtmosphereParameters (definitions.h:82-90): delta irradiance, delta Rayleigh, delta Mie, delta scattering density, delta multiple
 * scattering (256x128x32 except the irradiance ones), transmittance (256x64), irradiance (256x64), scattering, single Mie.  P's own
 * buffer pointers are not read.  lfr: the luminance-from-radiance matrix, row-major (y_r = sum_c lfr[r*3+c] x_c).  blend (0 or 1) goes
 * to the kernels that take it (single scattering: both of its flags); order (2..16) to the three kernels of the later orders.
 * Anything else is refused with VPT_ERR_INVALID and nothing is launched. */
#define VPT_BRUNETON_TRANSMITTANCE        0
#define VPT_BRUNETON_DIRECT_IRRADIANCE    1
#define VPT_BRUNETON_SINGLE_SCATTERING    2
#define VPT_BRUNETON_SCATTERING_DENSITY   3
#define VPT_BRUNETON_INDIRECT_IRRADIANCE  4
#define VPT_BRUNETON_MULTIPLE_SCATTERING  5
int  vpt_debug_bruneton_stage(int stage, const vpt_atmosphere* P, const vpt_devptr_t tables[9], const float lfr[9], int blend, int order);

/* Thin-lens camera set-up (camera::update_camera, camera.h:110-129). */
void vpt_camera_look_at(vpt_camera* cam, const float lookfrom[3], const float lookat[3], const float vup[3],
                        float vfov_deg, float aspect, float aperture);
/* Kernel_params defaults of main.cpp:1350-1376 with the frame-loop overrides (:1533-1544). */
void vpt_kernel_params_defaults(vpt_kernel_params* kp);

#ifdef __cplusplus
}
#endif
#endif /* VPT_B200_H_ */
